#!/usr/bin/env python
"""How many lanes of a warp share one owner triangle in the pixel-parallel kernels, on bench.py's workload.

A warp of the tile kernels covers 16 x 2 pixels of a 16 x 16 tile (lane l: column l % 16, row 2p + l / 16).  The colour
epilogue of the z pass (and k_shade) sets up the forward owner of each lane's pixel (`face_id`); the pixel-parallel
adjoint (k_interior_bwd, the interior pass of k_raster_bwd) sets up the adjoint owner of the pixels whose owner code
has no SMALL_FLAG (medium and large triangles; exact-tie pixels are left out).  A set-up shared by the lanes of a warp
that hold the same owner would run once per (warp, owner) pair instead of once per lane: this prints the lanes per
such pair from the owner maps of one forward, read back on the host (the kernels are not touched).

    python scripts/warp_owners.py --workload c5"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SMALL_FLAG = 0x40000000  # phases.h
TRI_INDEX_MASK = 0x3FFFFFFF


def lanes_per_owner(ids: np.ndarray) -> dict:
    """ids [H, W]: the triangle a lane sets up, -1 where it sets none up.  Lanes and (warp, triangle) pairs."""
    H, W = ids.shape
    pad = np.full(((H + 1) // 2 * 2, (W + 15) // 16 * 16), -1, dtype=np.int64)
    pad[:H, :W] = ids
    Hp, Wp = pad.shape
    warp = (np.arange(Hp)[:, None] // 2) * (Wp // 16) + np.arange(Wp)[None, :] // 16
    on = pad >= 0
    pairs = np.unique(warp[on] * (int(pad.max()) + 1) + pad[on]).size
    warps = np.unique(warp[on]).size
    return {"lanes": int(on.sum()), "warps_with_a_lane": int(warps), "owners": int(pairs)}


def main():
    import torch

    import bench
    from deodr_b200.renderer import DeviceScene, Renderer

    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c5", choices=sorted(bench.WORKLOADS))
    args = ap.parse_args()

    torch.cuda.set_device(0)
    n_views = 8 if args.workload == "c4" else 1
    renderer = Renderer(0)
    total = {"epilogue": {}, "adjoint": {}}
    for v in range(n_views):
        out = renderer.render(DeviceScene(bench.build_scene(args.workload, view=v, n_views=n_views), "cuda:0"),
                              bench.SIGMA, face_id=True)
        face = out["face_id"].cpu().numpy().astype(np.int64)
        code = out["owner"].cpu().numpy().astype(np.int64)
        medium = np.where((code >= 0) & ((code & SMALL_FLAG) == 0), code & TRI_INDEX_MASK, -1)
        for name, ids in (("epilogue", face), ("adjoint", medium)):
            for k, n in lanes_per_owner(ids).items():
                total[name][k] = total[name].get(k, 0) + n
    for t in total.values():
        t["lanes_per_warp"] = round(t["lanes"] / max(t["warps_with_a_lane"], 1), 2)
        t["lanes_per_owner"] = round(t["lanes"] / max(t["owners"], 1), 2)
    print(json.dumps({"workload": args.workload, "gpu": torch.cuda.get_device_name(0), "views": n_views, **total}))


if __name__ == "__main__":
    main()
