#!/usr/bin/env python
"""Time the self-collision energy (csrc/collision.cu): ``DeviceSelfCollisionEnergy.evaluate`` on the hand
(526 vertices, 1048 faces, thickness 0.02, a finger pushed toward its neighbour so that pairs are in contact), on the
hand after two and three levels of Loop subdivision (8k and 33k vertices, same thickness, small noise), and on the
200k-face torus of bench config c4 (torus_mesh(316), thickness half the median edge, noise of 0.3 median edge); then
the depth fitter's step on the hand with and without the term (cself = 1000, thickness 0.02).

Per workload, one JSON line:
  pairs_vt, pairs_ee   vertex-triangle and edge-edge pairs closer than the thickness (from the fp64 restatement, where
                       it is cheap enough: the hand and its first subdivision; "not counted" elsewhere)
  us_per_call          CUDA events around --steps calls after --warmup calls (each call reads one word back)
  kernel_us_per_call   device time per call of every kernel, from a torch.profiler run of --profile-steps calls, and
                       per kernel name
The card's name and power limit are printed first, read in the same run.  Writes nothing.

    python scripts/bench_self_collision.py [--steps 200] [--warmup 20] [--profile-steps 20]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.dirname(os.path.abspath(__file__)), os.path.join(ROOT, "tests")]

from bench_fitter import card  # noqa: E402

import self_collision_ref as R  # noqa: E402


def _median_edge(faces, vertices):
    e = R.edges_of(faces, vertices.shape[0])
    return float(np.median(np.linalg.norm(vertices[e[:, 0]] - vertices[e[:, 1]], axis=1)))


def workloads():
    import torch

    from deodr_b200.mesh_ops import LoopSubdivision
    from deodr_b200.scenes import torus_mesh

    faces, rest = R.hand()
    pushed = R.pushed_finger(faces, rest, -0.01)
    out = {"hand": (faces, pushed, rest, 0.02)}
    for n in (2, 3):
        sub = LoopSubdivision(faces, rest.shape[0], n, device="cuda")
        fine = sub.apply(torch.from_numpy(pushed).cuda())[0].cpu().numpy()
        fine_rest = sub.apply(torch.from_numpy(rest).cuda())[0].cpu().numpy()
        out[f"hand_loop{n}"] = (sub.faces, fine, fine_rest, 0.02)
    tv, tf, _ = torus_mesh(316)
    tf = tf.astype(np.int64)
    h = _median_edge(tf, tv)
    noisy = tv + 0.3 * h * np.random.default_rng(0).normal(size=tv.shape)
    out["torus_200k"] = (tf, noisy, tv, 0.5 * h)
    return out


def timed(torch, fn, steps, warmup, profile_steps):
    from torch.profiler import ProfilerActivity, profile

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    stop.record()
    torch.cuda.synchronize()
    us = 1000 * start.elapsed_time(stop) / steps
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(profile_steps):
            fn()
        torch.cuda.synchronize()
    per_kernel = {}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        name = ev.name.replace("(anonymous namespace)::", "").split("(")[0].split("<")[0].replace("void ", "")
        per_kernel[name] = per_kernel.get(name, 0.0) + ev.device_time / profile_steps
    return us, sum(per_kernel.values()), {k: round(v, 2) for k, v in sorted(per_kernel.items(), key=lambda x: -x[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--profile-steps", type=int, default=20)
    args = ap.parse_args()
    import torch

    from deodr_b200.mesh_fitter import DeviceSelfCollisionEnergy, MeshDepthFitter

    assert torch.cuda.is_available(), "bench_self_collision needs a GPU"
    gpu = card()
    print("card:", gpu, flush=True)
    for name, (faces, vertices, ref, delta) in workloads().items():
        model = DeviceSelfCollisionEnergy(faces, ref, delta, 1.0)
        x = torch.from_numpy(vertices).cuda()
        us, kus, per_kernel = timed(torch, lambda: model.evaluate(x), args.steps, args.warmup, args.profile_steps)
        if vertices.shape[0] <= 10000:
            _, _, _, pairs = R.self_collision(faces, vertices, delta, 1.0)
            counts = (int(pairs["vt"]["d"].size), int(pairs["ee"]["d"].size))
        else:
            counts = ("not counted", "not counted")
        print(json.dumps({"workload": name, "vertices": int(vertices.shape[0]), "faces": int(faces.shape[0]),
                          "thickness": delta, "pairs_vt": counts[0], "pairs_ee": counts[1],
                          "energy": float(model.evaluate(x)[0]), "min_distance": float(model.min_distance),
                          "us_per_call": round(us, 2), "kernel_us_per_call": round(kus, 2),
                          "per_kernel_us": per_kernel, "card": gpu}), flush=True)

    golden = os.path.join(ROOT, "tests", "golden")
    inputs = np.load(os.path.join(golden, "hand_fitting_inputs.npz"))
    faces, rest = R.hand()
    for label, kw in (("depth_step_without", {}), ("depth_step_with", dict(cself=1000.0, self_collision_thickness=0.02))):
        f = MeshDepthFitter(rest, faces, np.array([0.1, 0.1, 0.1]), np.zeros(3), cregu=1000, **kw)
        f.set_image(inputs["depth"], focal=241, distortion=np.array([1, 0, 0, 0, 0]))
        f.set_max_depth(1)
        f.set_depth_scale(110 / 450)
        us, kus, per_kernel = timed(torch, f.step, args.steps, args.warmup, args.profile_steps)
        print(json.dumps({"workload": label, "us_per_step": round(us, 2), "kernel_us_per_step": round(kus, 2),
                          "card": gpu}), flush=True)


if __name__ == "__main__":
    main()
