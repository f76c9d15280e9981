#!/usr/bin/env python
"""Time linear blend skinning (csrc/skinning.cu): the forward (deodr_b200_skin) and the adjoint without weight
gradients, the form the fitters call (deodr_b200_skin_b), on
  tube          the articulated-fit tube of tests/test_gpu_skinning.py (658 vertices, 4 chained joints, K = 2)
  tube_2k       the same tube with 121 rings of 16 (1938 vertices)
  mesh_1m_*     1M random vertices, a random 64-joint tree, K = 4: "blocked" binds consecutive vertices to
                neighbouring joints (the order of a real mesh), "scattered" binds every vertex to 4 random joints
then the RGB fitter's step on the tube with and without its skeleton.

Per workload, one JSON line:
  fwd_kernel_us, bwd_kernel_us   device time per call of the forward and adjoint kernels, from a torch.profiler run of
                                 --profile-steps calls (per kernel name in per_kernel_us)
  fwd_bytes, bwd_bytes           bytes a call must move, computed from the shapes: forward V (24 + 12 K + 24);
                                 adjoint V (24 + 12 K + 24) for vertices_b plus V K (4 + 8 + 24 + 24) for the joint
                                 sums and 96 per chunk partial (the [J,24] table and the joint kernels are left out)
  fwd_gbps, bwd_gbps, *_of_peak  bytes over kernel time, and over NVIDIA's H100 SXM data-sheet 3.35 TB/s
  us_per_call                    CUDA events around --steps forward + adjoint pairs after --warmup pairs
The card's name and power limit are printed first, read in the same run.  Writes nothing.

    python scripts/bench_skinning.py [--steps 200] [--warmup 20] [--profile-steps 20]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.dirname(os.path.abspath(__file__)), os.path.join(ROOT, "tests")]

from bench_fitter import card  # noqa: E402
from bench_self_collision import timed  # noqa: E402

import skinning_ref as ref  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12
FWD_KERNELS = ("k_forward_kinematics", "k_skin")
BWD_KERNELS = ("k_skin_vertices_b", "k_skin_joint_partials", "k_forward_kinematics_b")


def mesh_1m(blocked: bool, V=1_000_000, J=64, K=4):
    rng = np.random.default_rng(0)
    parents = ref.random_tree(rng, J, min_depth=6)
    centres = rng.normal(size=(J, 3))
    if blocked:
        base = (np.arange(V, dtype=np.int64) * J) // V
    else:
        base = rng.integers(0, J, size=V)
    skin_index = ((base[:, None] + np.arange(K)[None, :]) % J).astype(np.int32)
    w = rng.uniform(0.1, 1.0, size=(V, K))
    return parents, centres, skin_index, w / w.sum(axis=1, keepdims=True), rng.normal(size=(V, 3))


def tube(n_along):
    vertices, faces, parents, centres, skin_index, skin_weight = ref.tube(n_along)
    return parents, centres, skin_index, skin_weight, vertices


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--profile-steps", type=int, default=20)
    args = ap.parse_args()
    import torch

    from deodr_b200.mesh_fitter import MeshRGBFitterWithPose
    from deodr_b200.mesh_ops import LinearBlendSkinning

    assert torch.cuda.is_available(), "bench_skinning needs a GPU"
    gpu = card()
    print("card:", gpu, flush=True)
    workloads = {"tube": tube(ref.N_ALONG), "tube_2k": tube(121), "mesh_1m_blocked": mesh_1m(True),
                 "mesh_1m_scattered": mesh_1m(False)}
    for name, (parents, centres, skin_index, skin_weight, vertices) in workloads.items():
        V, K = skin_index.shape
        J = len(parents)
        lbs = LinearBlendSkinning(parents, centres, skin_index, skin_weight, device="cuda")
        rng = np.random.default_rng(1)
        v = torch.from_numpy(vertices).cuda()
        r = torch.from_numpy(0.3 * rng.normal(size=(J, 3))).cuda()
        g = torch.from_numpy(rng.normal(size=(V, 3))).cuda()
        out = torch.empty_like(v)
        bout = (torch.empty_like(v), torch.empty_like(r))

        def call():
            lbs.apply(v, r, out=out)
            lbs.backward(v, r, g, out=bout)

        us, _, per_kernel = timed(torch, call, args.steps, args.warmup, args.profile_steps)
        fwd_us = sum(per_kernel.get(k, 0.0) for k in FWD_KERNELS)
        bwd_us = sum(per_kernel.get(k, 0.0) for k in BWD_KERNELS)
        fwd_bytes = V * (24 + 12 * K + 24)
        bwd_bytes = V * (24 + 12 * K + 24) + V * K * (4 + 8 + 24 + 24) + 96 * lbs.nb_chunks
        line = {"workload": name, "vertices": V, "joints": J, "influences": K,
                "levels": int(lbs.t["level_offset"].numel() - 1), "chunks": lbs.nb_chunks,
                "fwd_kernel_us": round(fwd_us, 2), "bwd_kernel_us": round(bwd_us, 2),
                "fwd_bytes": fwd_bytes, "bwd_bytes": bwd_bytes,
                "fwd_gbps": round(fwd_bytes / fwd_us / 1e3, 1), "bwd_gbps": round(bwd_bytes / bwd_us / 1e3, 1),
                "fwd_of_peak": round(fwd_bytes / (fwd_us * 1e-6) / PEAK_BYTES_PER_S, 3),
                "bwd_of_peak": round(bwd_bytes / (bwd_us * 1e-6) / PEAK_BYTES_PER_S, 3),
                "us_per_call": round(us, 2), "per_kernel_us": per_kernel, "card": gpu}
        print(json.dumps(line), flush=True)

    vertices, faces, parents, centres, skin_index, skin_weight = ref.tube()
    target = np.zeros((128, 128, 3))
    for label, skeleton in (("tube_rgb_step_without", None),
                            ("tube_rgb_step_with", (parents, centres, skin_index, skin_weight))):
        f = MeshRGBFitterWithPose(vertices, faces, np.zeros(3), np.zeros(3), [0.9, 0.6, 0.3], [0.2, -0.3, -0.7], 0.3,
                                  skeleton=skeleton)
        f.set_image(target)
        us, kus, per_kernel = timed(torch, f.step, args.steps, args.warmup, args.profile_steps)
        print(json.dumps({"workload": label, "us_per_step": round(us, 2), "kernel_us_per_step": round(kus, 2),
                          "skinning_kernel_us": round(sum(per_kernel.get(k, 0.0)
                                                          for k in FWD_KERNELS + BWD_KERNELS), 2),
                          "card": gpu}), flush=True)


if __name__ == "__main__":
    main()
