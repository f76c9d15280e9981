#!/usr/bin/env python
"""Where a busy tile's time goes in the z pass (k_tile_z), per phase, and how many records the busy tiles hold.

Needs a measurement build of the library (the clock64() counters are compiled in only with the switch):
    scripts/build_variant.sh tilez_clocks -DDEODR_TILEZ_PHASE_CLOCKS
    DEODR_B200_LIB=$PWD/deodr_b200/libdeodr_b200_tilez_clocks.so python scripts/tilez_phases.py --workload c5
(add -DDEODR_WARP_TEST_MAX=0 to the build for the split with every chunk going through the candidate scatter).

Runs `--passes` forwards of bench.py's workload (c4: its 8 RGB + 8 depth views) and prints one JSON line: the warp
cycles spent in each phase summed over lane 0 of every warp of every busy tile (and the mean per busy tile and warp,
share of the total), and the histogram of records per busy tile.  The counters perturb the kernel a little (one
clock64() and a few adds per phase boundary): the split is the measurement, the kernel time is bench.py's."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ["copy_wait", "scatter", "barrier", "pix_test", "large", "epilogue", "tma_store"]  # kernels.cu TZ_* order
TZ_HIST = 1025
BUCKETS = [(1, 1), (2, 8), (9, 16), (17, 32), (33, 64), (65, 96), (97, 127), (128, 128), (129, 256), (257, 10 ** 9)]


def main():
    import torch

    import bench
    from deodr_b200 import _cabi
    from deodr_b200.renderer import DeviceScene, Renderer

    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c5", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--passes", type=int, default=10)
    args = ap.parse_args()

    lib = _cabi.load()
    if not hasattr(lib, "deodr_b200_tilez_phase_clocks"):
        sys.exit(f"{_cabi.LIB_PATH} was built without -DDEODR_TILEZ_PHASE_CLOCKS (see this script's docstring)")
    fn = lib.deodr_b200_tilez_phase_clocks
    fn.argtypes = [C.POINTER(C.c_ulonglong), C.POINTER(C.c_uint)]
    clocks = (C.c_ulonglong * (len(PHASES) + 1))()
    hist = (C.c_uint * TZ_HIST)()

    torch.cuda.set_device(0)
    n_views = 8 if args.workload == "c4" else 1
    scenes = [bench.build_scene(args.workload, view=v, n_views=n_views) for v in range(n_views)]
    if args.workload == "c4":  # bench.py's depth renders of the same views
        for v in range(n_views):
            d = bench.build_scene(args.workload, view=v, n_views=n_views)
            d.nb_colors, d.colors = 1, np.ascontiguousarray(d.depths[:, None])
            d.background_color = np.array([float(d.depths.max())])
            d.texture = np.zeros((2, 2, 1))
            scenes.append(d)
    renderer = Renderer(0)
    dss = [DeviceScene(s, "cuda:0") for s in scenes]
    for _ in range(2):  # plan + warm-up
        renderer.render_views(dss, bench.SIGMA)
    _cabi.check(fn(clocks, hist))  # clears the counters
    for _ in range(args.passes):
        renderer.render_views(dss, bench.SIGMA)
    _cabi.check(fn(clocks, hist))

    warps = clocks[len(PHASES)]
    total = sum(clocks[i] for i in range(len(PHASES)))
    h = np.array(hist[:], dtype=np.int64) // args.passes  # per forward of all the views
    busy = int(h.sum())
    recs = np.arange(TZ_HIST)
    out = {
        "workload": args.workload,
        "lib": os.path.basename(_cabi.LIB_PATH),
        "gpu": torch.cuda.get_device_name(0),
        "passes": args.passes,
        "busy_tiles_per_forward": busy,
        "warp_cycles_per_busy_tile_warp": {p: round(clocks[i] / max(warps, 1), 1) for i, p in enumerate(PHASES)},
        "share": {p: round(clocks[i] / max(total, 1), 4) for i, p in enumerate(PHASES)},
        "records_per_busy_tile": {
            "tiles_without_records": int(h[0]),
            "mean_over_tiles_with_records": round(float((h[1:] * recs[1:]).sum() / max(h[1:].sum(), 1)), 1),
            "median_over_tiles_with_records": int(np.searchsorted(np.cumsum(h[1:]), h[1:].sum() / 2) + 1),
            "histogram": {f"{a}-{b}" if a != b else f"{a}": int(h[a:min(b, TZ_HIST - 1) + 1].sum()) for a, b in BUCKETS},
            "last_chunk_at_most_32": int(sum(h[n] for n in range(1, TZ_HIST) if (n - 1) % 128 + 1 <= 32)),
        },
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
