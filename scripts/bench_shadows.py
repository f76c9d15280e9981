#!/usr/bin/env python
"""Time one Phong DeviceMeshView step (render plus backward) with L = 1, 2 and 4 grey point lights, without shadows
and with cube shadow maps of M = 256 and 512, the views alternated in one process, on two workloads:

  hand           the hand of the fitting examples (526 vertices, 1048 faces) at 640 x 480, sigma 1
  torus_plane    the 200k-triangle torus (torus_mesh(316)) in front of a 64 x 64-quad plane, at 1024 x 1024, sigma 1

Per workload and view, one JSON line:
  ms_per_step      CUDA events around --steps steps after --warmup steps (alternated rounds: the median and all rounds)
  kernel_us        device time per step of the shadow and shading kernels, from a torch.profiler run of
                   --profile-steps steps of its own, by kernel instance
  raster_us        device time per step of every other kernel (the rasteriser's passes, the projections, normals and
                   silhouettes): the view's own raster, plus the 6L cube faces with shadows
  kernel_bytes     the bytes each shadow kernel must move, from shapes: fp64 vertices, ij and depths, fp32 maps,
                   G-buffer position and coverage, visibility and its gradient
The card's name, power limit and maximum SM clock are printed first, read in the same run.  Writes nothing.

    python scripts/bench_shadows.py [--steps 20] [--warmup 3] [--rounds 5] [--profile-steps 10]
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

SHADING = re.compile(r"(k_cube_project_b<\d+>|k_cube_project|k_cube_cameras|k_shadow_visibility_b<\d+>|"
                     r"k_shadow_visibility|k_phong_shade_b<[^>]*>|k_phong_shade<[^>]*>|k_point_lights_pixel_b<[^>]*>)")


def kernel_bytes(name, P, V, L, M, C=3):
    K = C + 7
    if name.startswith("k_cube_project_b"):
        return V * (24 + 6 * L * (8 + 4 + 24))           # vertices, ij_b + depths_b per face, vertices_b
    if name.startswith("k_cube_project"):
        return 6 * L * V * (24 + 16 + 8)                   # vertices (from L2 after the first face), ij, depths
    if name.startswith("k_cube_cameras"):
        return 6 * L * 26 * 8
    if name.startswith("k_shadow_visibility_b"):
        return P * (16 + 4 * L + 16) + L * P * 16 + 6 * L * M * M * 4  # G-buffer slices, vis_b, taps, maps_b
    if name.startswith("k_shadow_visibility"):
        return P * (16 + 4 * L) + L * P * 16                # G-buffer slices, vis, four taps per light
    if name.startswith("k_phong_shade_b"):
        return P * (4 * C + 4 * K + 4 * K + 8 * L)
    if name.startswith("k_phong_shade"):
        return P * (4 * K + 4 * C + 4 * L)
    return P * (4 * K + 4 * C + 4 * L)                      # k_point_lights_pixel_b


def plane(z, half, n):
    g = np.linspace(-half, half, n + 1)
    x, y = np.meshgrid(g, g, indexing="ij")
    v = np.stack((x, y, np.full_like(x, z)), axis=-1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    q = (i * (n + 1) + j).ravel()
    f = np.concatenate((np.stack((q, q + n + 1, q + n + 2), 1), np.stack((q, q + n + 2, q + 1), 1)))
    tri = v[f]
    flip = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])[:, 2] > 0  # facing -z, the camera
    f[flip] = f[flip][:, ::-1]
    return v, f


def workloads():
    from deodr_b200.mesh_ops import CameraParams
    from deodr_b200.scenes import torus_mesh

    g = np.load(os.path.join(ROOT, "tests", "golden", "scene_ops.npz"))
    hand = (g["hand_faces"].astype(np.int64), g["hand_vertices"], CameraParams(g["view_extrinsic"], g["view_intrinsic"]),
            480, 640)
    tv, tf, _ = torus_mesh(316)
    tv = tv + np.array([0.0, 0.0, 3.0])
    pv, pf = plane(3.8, 2.5, 64)
    size = 1024
    tcam = CameraParams(np.eye(3, 4), np.array([[size, 0, size / 2], [0, size, size / 2], [0, 0, 1]]))
    torus = (np.concatenate((tf.astype(np.int64), pf + len(tv))), np.concatenate((tv, pv)), tcam, size, size)
    return {"hand_640x480": hand, "torus_plane_1024": torus}


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
        raise SystemExit("bench_shadows.py needs a CUDA device")
    dev = "cuda:0"
    print(json.dumps({"card": card()}), flush=True)
    for name, (faces, V, cam, H, W) in workloads().items():
        center, mid = camera_center(cam), V.mean(axis=0)
        size = float(np.linalg.norm(V.max(axis=0) - V.min(axis=0)))
        dist = float(np.linalg.norm(center - mid))
        rng = np.random.default_rng(2)
        colors = np.random.default_rng(0).uniform(0.2, 1, (V.shape[0], 3))
        views = {}
        for L in (1, 2, 4):
            # beside the camera, a third of its distance to the mesh off axis: the shadows fall on the visible side
            p = center + (mid - center) * 0.3 + rng.uniform(-0.3, 0.3, (L, 3)) * dist
            inten = np.sum((p - mid) ** 2, axis=1, keepdims=True) * rng.uniform(0.2, 0.4, (L, 1))
            lights = torch.from_numpy(np.concatenate((p, inten), axis=1)).to(dev)
            for M in (0, 256, 512):
                kw = dict(shadow_map_size=M, shadow_bias=0.01 * size, shadow_softness=0.02 * size) if M else {}
                views[f"L{L}_M{M}"] = DeviceMeshView(
                    faces, V.shape[0], cam, H, W, light_directional=None, ambient=0.2,
                    background_color=np.array([0.1, 0.2, 0.3]), sigma=1.0, device=dev, shading="phong",
                    specular=0.5, shininess=20.0, point_lights=lights, **kw)
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
        P = H * W
        for s, view in views.items():
            L, M = (int(x[1:]) for x in s.split("_"))
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
            nbytes = {k: kernel_bytes(k, P, V.shape[0], L, M) for k in us if k.startswith(("k_cube", "k_shadow"))}
            print(json.dumps({"workload": name, "view": s, "lights": L, "map_size": M, "triangles": int(len(faces)),
                              "pixels": P, "vertices": V.shape[0], "ms_per_step": float(np.median(ms[s])),
                              "ms_rounds": [round(x, 4) for x in ms[s]], "raster_us": round(raster, 1),
                              "kernel_us": {k: round(u, 2) for k, u in us.items()}, "kernel_bytes": nbytes,
                              "kernel_gb_per_s": {k: round(nbytes[k] / (us[k] * 1e3), 1) for k in nbytes
                                                  if us[k] > 0}}), flush=True)


if __name__ == "__main__":
    main()
