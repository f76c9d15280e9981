#!/usr/bin/env python
"""Time one textured Phong DeviceMeshView step (render plus backward) on the 200k-triangle torus (torus_mesh(316),
its uv split at the seam) at 1024 x 1024, without a normal map and with a 1024 x 1024 one, the two views alternated
in one process.  One JSON line per view:
  ms_per_step      CUDA events around --steps steps after --warmup steps (alternated rounds: the median and all rounds)
  kernel_us        device time per step of the tangent and normal-map kernels, from a torch.profiler run of
                   --profile-steps steps of its own, by kernel
  raster_us        device time per step of every other kernel
  kernel_bytes     the bytes each of those kernels must move at least, from the shapes (reads plus writes)
The card's name, power limit and maximum SM clock are printed first, read in the same run.  Writes nothing.

    python scripts/bench_normal_map.py [--steps 20] [--warmup 3] [--rounds 5] [--profile-steps 10]
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

KERNELS = re.compile(r"(k_face_tangents_b|k_face_tangents|k_vertex_tangents_b1|k_vertex_tangents|"
                     r"k_tangents_vertices_b|k_tangents_uv_b|k_normal_map_b|k_normal_map)\b")


def torus_split_uv(n: int, texels: int):
    """torus_mesh(n) with its uv vertices split at the seam ((n + 1)^2 of them, texel units), faces_uv to match."""
    from deodr_b200.scenes import torus_mesh

    vertices, faces, _ = torus_mesh(n)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    a, b = (i * (n + 1) + j).ravel(), ((i + 1) * (n + 1) + j).ravel()
    c, d = ((i + 1) * (n + 1) + j + 1).ravel(), (i * (n + 1) + j + 1).ravel()
    faces_uv = np.empty_like(faces)
    faces_uv[0::2] = np.stack((a, b, c), axis=1)
    faces_uv[1::2] = np.stack((a, c, d), axis=1)
    ui, vj = np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing="ij")
    uv = np.stack((ui.ravel(), vj.ravel()), axis=1) / n * (texels - 1)
    return vertices, faces.astype(np.int64), uv, faces_uv.astype(np.int64)


def kernel_bytes(V: int, T: int, U: int, pixels: int) -> dict:
    """The least bytes each kernel moves, from the shapes (fp64 vertices, uv and frames; int32 indices and CSRs; fp32
    G-buffers): every input read once and every output written once."""
    csr_v, csr_u = 4 * (V + 1 + 3 * T), 4 * (U + 1 + 3 * T)
    face_in = 12 * T + 12 * T + 24 * V + 16 * U  # faces, faces_uv, vertices, uv
    return {"k_face_tangents": face_in + 48 * T,
            "k_vertex_tangents": csr_v + 48 * T + 48 * V,
            "k_vertex_tangents_b1": csr_v + face_in + 48 * V + 48 * V,
            "k_face_tangents_b": face_in + 48 * V + 80 * T,
            "k_tangents_vertices_b": csr_v + 12 * T + 80 * T + 2 * 24 * V,
            "k_tangents_uv_b": csr_u + 12 * T + 80 * T + 16 * U,
            "k_normal_map": pixels * 4 * (13 + 3 + 7),
            "k_normal_map_b": pixels * 4 * (13 + 3 + 7 + 13 + 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=10)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from deodr_b200.mesh_ops import CameraParams, DeviceMeshView

    if not torch.cuda.is_available():
        raise SystemExit("bench_normal_map.py needs a CUDA device")
    dev = "cuda:0"
    print(json.dumps({"card": card()}), flush=True)
    size, texels = 1024, 1024
    vertices, faces, uv, faces_uv = torus_split_uv(316, texels)
    vertices = vertices + np.array([0.0, 0.0, 3.0])
    cam = CameraParams(np.eye(3, 4), np.array([[size, 0, size / 2], [0, size, size / 2], [0, 0, 1]]))
    rng = np.random.default_rng(0)
    texture = rng.uniform(0.2, 1.0, (texels, texels, 3))
    nmap = np.concatenate((rng.normal(size=(texels, texels, 2)) * 0.2, np.ones((texels, texels, 1))), axis=2)
    common = dict(light_directional=np.array([0.3, -0.4, 0.8]), ambient=0.2, background_color=np.array([0.1, 0.2, 0.3]),
                  sigma=1.0, device=dev, uv=uv, faces_uv=faces_uv, texture=texture, shading="phong_textured",
                  specular=0.5, shininess=20.0)
    views = {"no_map": DeviceMeshView(faces, vertices.shape[0], cam, size, size, **common),
             "normal_map_1024": DeviceMeshView(faces, vertices.shape[0], cam, size, size, normal_map=nmap, **common)}
    v = torch.from_numpy(vertices).to(dev)
    image_b = torch.from_numpy(np.random.default_rng(1).normal(size=(size, size, 3)).astype(np.float32)).to(dev)

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
    sizes = kernel_bytes(vertices.shape[0], faces.shape[0], uv.shape[0], size * size)
    for s, view in views.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_steps):
                step(view)
            torch.cuda.synchronize()
        us, raster = {}, 0.0
        for e in prof.events():
            if e.device_type.name != "CUDA" or e.device_time <= 0:
                continue
            m = KERNELS.search(e.name)
            if m:
                us[m.group(1)] = us.get(m.group(1), 0.0) + e.device_time / args.profile_steps
            elif "Memcpy" not in e.name and "Memset" not in e.name:
                raster += e.device_time / args.profile_steps
        print(json.dumps({"view": s, "triangles": int(len(faces)), "pixels": size * size, "texels": texels * texels,
                          "ms_per_step": float(np.median(ms[s])), "ms_rounds": [round(x, 4) for x in ms[s]],
                          "raster_us": round(raster, 1), "kernel_us": {k: round(u, 2) for k, u in us.items()},
                          "kernel_bytes": {k: sizes[k] for k in us},
                          "kernel_GBps": {k: round(sizes[k] / (u * 1e3), 1) for k, u in us.items() if u > 0}}),
              flush=True)


if __name__ == "__main__":
    main()
