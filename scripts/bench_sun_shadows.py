#!/usr/bin/env python
"""Time one Phong DeviceMeshView step (render plus backward) under a directional light, without shadows and with the
light's shadow map at M = 512, 1024 and 2048, and with that map beside one point light's cube maps (M = 512), the
views alternated in one process, on two workloads:

  hand           the hand of the fitting examples (526 vertices, 1048 faces) at 640 x 480, sigma 1
  torus_plane    the 200k-triangle torus (torus_mesh(316)) in front of a 64 x 64-quad plane, at 1024 x 1024, sigma 1

The light comes from beside the camera, a third of the way to the mesh off axis, so that the shadows fall on the
visible side; the map's window is the mesh's bounding sphere.  Per workload and view, one JSON line:
  ms_per_step      CUDA events around --steps steps after --warmup steps (alternated rounds: the median and all rounds)
  kernel_us        device time per step of the shadow and shading kernels, from a torch.profiler run of
                   --profile-steps steps of its own, by kernel instance
  raster_us        device time per step of every other kernel (the rasteriser's passes, the projections, normals and
                   silhouettes): the view's own raster, plus the shadow maps' rasters
The card's name, power limit and maximum SM clock are printed first, read in the same run.  Writes nothing.

    python scripts/bench_sun_shadows.py [--steps 20] [--warmup 3] [--rounds 5] [--profile-steps 10]
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
from bench_shadows import workloads  # noqa: E402

SHADING = re.compile(r"(k_sun_project_b|k_sun_project|k_sun_visibility_b|k_sun_visibility|"
                     r"k_cube_project_b<\d+>|k_cube_project|k_cube_cameras|k_shadow_visibility_b<\d+>|"
                     r"k_shadow_visibility|k_phong_shade_b<[^>]*>|k_phong_shade<[^>]*>|k_point_lights_pixel_b<[^>]*>)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=10)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from deodr_b200.mesh_ops import DeviceMeshView, camera_center

    if not torch.cuda.is_available():
        raise SystemExit("bench_sun_shadows.py needs a CUDA device")
    dev = "cuda:0"
    print(json.dumps({"card": card()}), flush=True)
    for name, (faces, V, cam, H, W) in workloads().items():
        center, mid = camera_center(cam), V.mean(axis=0)
        lo, hi = V.min(axis=0), V.max(axis=0)
        size = float(np.linalg.norm(hi - lo))
        dist = float(np.linalg.norm(center - mid))
        bounds = tuple((0.5 * (lo + hi)).tolist()) + (0.5 * size * 1.01,)
        rng = np.random.default_rng(2)
        # the light travels from beside the camera to the mesh
        src = center + (mid - center) * 0.3 + rng.uniform(-0.3, 0.3, 3) * dist
        light = (mid - src) / np.linalg.norm(mid - src) * 0.8
        p = center + (mid - center) * 0.3 + rng.uniform(-0.3, 0.3, (1, 3)) * dist
        point = torch.from_numpy(np.concatenate((p, np.sum((p - mid) ** 2, axis=1, keepdims=True) * 0.3), axis=1))
        point = point.to(dev)
        colors = np.random.default_rng(0).uniform(0.2, 1, (V.shape[0], 3))
        sun = dict(light_shadow_bias=0.01 * size, light_shadow_softness=0.02 * size, light_shadow_bounds=bounds)
        cube = dict(point_lights=point, shadow_map_size=512, shadow_bias=0.01 * size, shadow_softness=0.02 * size)
        configs = {"none": {}, "sun512": dict(light_shadow_map_size=512, **sun),
                   "sun1024": dict(light_shadow_map_size=1024, **sun), "sun2048": dict(light_shadow_map_size=2048, **sun),
                   "point512": cube, "point512_sun1024": dict(light_shadow_map_size=1024, **sun, **cube)}
        views = {s: DeviceMeshView(faces, V.shape[0], cam, H, W, light_directional=light, ambient=0.2,
                                   background_color=np.array([0.1, 0.2, 0.3]), sigma=1.0, device=dev,
                                   shading="phong", specular=0.5, shininess=20.0, **kw) for s, kw in configs.items()}
        v, c = torch.from_numpy(V).to(dev), torch.from_numpy(colors).to(dev)
        image_b = torch.from_numpy(np.random.default_rng(1).normal(size=(H, W, 3)).astype(np.float32)).to(dev)

        def step(view):
            view.render(v, c)
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
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.profile_steps):
                    step(view)
                torch.cuda.synchronize()
            us, raster = {}, 0.0
            for e in prof.events():
                if e.device_type.name != "CUDA" or e.device_time <= 0:
                    continue
                m = SHADING.search(e.name)
                if m:
                    us[m.group(1)] = us.get(m.group(1), 0.0) + e.device_time / args.profile_steps
                elif "Memcpy" not in e.name and "Memset" not in e.name:
                    raster += e.device_time / args.profile_steps
            sun_us = sum(u for k, u in us.items() if k.startswith("k_sun"))
            print(json.dumps({"workload": name, "view": s, "triangles": int(len(faces)), "pixels": H * W,
                              "ms_per_step": float(np.median(ms[s])), "ms_rounds": [round(x, 4) for x in ms[s]],
                              "raster_us": round(raster, 1), "sun_kernels_us": round(sun_us, 1),
                              "kernel_us": {k: round(u, 2) for k, u in us.items()}}), flush=True)


if __name__ == "__main__":
    main()
