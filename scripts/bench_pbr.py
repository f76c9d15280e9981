#!/usr/bin/env python
"""Time one textured DeviceMeshView step (render plus backward) in three variants, alternated in one process: the
Phong form, the metallic-roughness (GGX) form without a map and the GGX form with a metallic-roughness map, on two
scenes: the duck at 320 x 240 (its 512 x 512 texture) and the 200k-triangle
torus (torus_mesh(316), its uv split at the seam) at 1024 x 1024 with a 1024 x 1024 texture.  One JSON line per view:
  ms_per_step      CUDA events around --steps steps after --warmup steps (alternated rounds: the median and all rounds)
  shade_us         device time per step of the Phong shading kernels (k_phong_shade, k_phong_shade_b,
                   k_point_lights_pixel_b), from a torch.profiler run of --profile-steps steps of its own, by kernel
  other_us         device time per step of every other kernel (the rasters, the projection, the normals)
  shade_bytes      the bytes each shading kernel must move at least, from the shapes (reads plus writes)
The card's name, power limit and maximum SM clock are printed first, read in the same run.  Writes nothing.

    python scripts/bench_pbr.py [--steps 20] [--warmup 3] [--rounds 5] [--profile-steps 10]
"""
import argparse
import json
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.dirname(os.path.abspath(__file__))]

from bench_fitter import card  # noqa: E402
from bench_normal_map import torus_split_uv  # noqa: E402

KERNELS = re.compile(r"(k_phong_shade_b|k_phong_shade|k_point_lights_pixel_b)\b")


def shade_bytes(pixels: int, C: int, mapped: bool) -> dict:
    """The least bytes of the shading kernels, fp32 buffers: the forward reads the G-buffer (7), the albedo (C) and
    the map raster (2, with a map) and writes the image (C); the adjoint reads those and image_b (C) and writes
    channels_b (7), albedo_b (C) and the map raster's gradient (2)."""
    m = 2 if mapped else 0
    return {"k_phong_shade": pixels * 4 * (7 + C + m + C),
            "k_phong_shade_b": pixels * 4 * (7 + C + m + C + 7 + C + m)}


def scenes(dev):
    """(name, faces, vertices, camera, H, W, uv, faces_uv, texture) of the two scenes."""
    from deodr_b200.mesh_ops import CameraParams

    d = np.load(os.path.join(ROOT, "tests", "golden", "duck_textured.npz"))
    duck_cam = CameraParams(d["extrinsic_320"], d["intrinsic_320"], d["distortion"])
    yield ("duck_320x240", d["faces"].astype(np.int64), d["vertices"], duck_cam, 240, 320, d["uv"],
           d["faces_uv"].astype(np.int64), d["texture_u8"] / 255.0)
    size, texels = 1024, 1024
    vertices, faces, uv, faces_uv = torus_split_uv(316, texels)
    cam = CameraParams(np.eye(3, 4), np.array([[size, 0, size / 2], [0, size, size / 2], [0, 0, 1]]))
    texture = np.random.default_rng(0).uniform(0.2, 1.0, (texels, texels, 3))
    yield ("torus_200k_1024", faces, vertices + np.array([0.0, 0.0, 3.0]), cam, size, size, uv, faces_uv, texture)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=10)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from deodr_b200.mesh_ops import DeviceMeshView

    if not torch.cuda.is_available():
        raise SystemExit("bench_pbr.py needs a CUDA device")
    dev = "cuda:0"
    print(json.dumps({"card": card()}), flush=True)
    for name, faces, vertices, cam, H, W, uv, faces_uv, texture in scenes(dev):
        rng = np.random.default_rng(1)
        mr = np.stack((rng.uniform(0.3, 0.9, texture.shape[:2]), rng.uniform(0.0, 1.0, texture.shape[:2])), axis=2)
        common = dict(light_directional=np.array([0.3, -0.4, 0.8]), ambient=0.2,
                      background_color=np.array([0.1, 0.2, 0.3]), sigma=1.0, device=dev, uv=uv, faces_uv=faces_uv,
                      texture=texture)
        pbr = dict(common, shading="pbr_textured", metallic=1.0, roughness=1.0)
        views = {"phong": DeviceMeshView(faces, vertices.shape[0], cam, H, W, shading="phong_textured", specular=0.5,
                                         shininess=20.0, **common),
                 "pbr_no_map": DeviceMeshView(faces, vertices.shape[0], cam, H, W, **pbr),
                 "pbr_map": DeviceMeshView(faces, vertices.shape[0], cam, H, W, metallic_roughness_map=mr, **pbr)}
        v = torch.from_numpy(vertices).to(dev)
        image_b = torch.from_numpy(rng.normal(size=(H, W, 3)).astype(np.float32)).to(dev)

        def step(view):
            view.render(v)
            view.backward(image_b)

        def timed(view, steps):
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(steps):
                step(view)
            stop.record()
            torch.cuda.synchronize()
            return start.elapsed_time(stop) / steps

        for view in views.values():
            for _ in range(args.warmup):
                step(view)
        torch.cuda.synchronize()
        ms = {s: [] for s in views}
        for _ in range(args.rounds):
            for s, view in views.items():
                ms[s].append(timed(view, args.steps))
        for s, view in views.items():
            sizes = shade_bytes(H * W, 3, s == "pbr_map")
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.profile_steps):
                    step(view)
                torch.cuda.synchronize()
            us, other = {}, 0.0
            for e in prof.events():
                if e.device_type.name != "CUDA" or e.device_time <= 0:
                    continue
                m = KERNELS.search(e.name)
                if m:
                    us[m.group(1)] = us.get(m.group(1), 0.0) + e.device_time / args.profile_steps
                elif "Memcpy" not in e.name and "Memset" not in e.name:
                    other += e.device_time / args.profile_steps
            print(json.dumps({"scene": name, "view": s, "triangles": int(len(faces)), "pixels": H * W,
                              "texels": int(texture.shape[0] * texture.shape[1]),
                              "ms_per_step": float(np.median(ms[s])), "ms_rounds": [round(x, 4) for x in ms[s]],
                              "other_us": round(other, 1), "shade_us": {k: round(u, 2) for k, u in us.items()},
                              "shade_bytes": {k: sizes[k] for k in us if k in sizes},
                              "shade_GBps": {k: round(sizes[k] / (u * 1e3), 1) for k, u in us.items()
                                             if u > 0 and k in sizes}}), flush=True)


if __name__ == "__main__":
    main()
