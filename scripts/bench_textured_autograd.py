#!/usr/bin/env python
"""Time and kernel launches of one textured fitting step under torch autograd, next to the hand-chained device path:

  duck_autograd      textured Scene3DPytorch.render of the duck (2108 vertices, 4212 faces, 512 x 512 x 3 texture),
                     a squared-error loss to a target image, loss.backward() to the vertices, uv, texture and light
  duck_device_view   DeviceMeshView.render / backward of the same mesh at the same size, image_b = 2 (image - target)
  eigen_faces        one step of the eigen-faces fit (tests/test_gpu_eigen_faces.py): texture = mean + coefs @
                     components, CudaRenderCompare2DTextured, loss.backward(), the two gradient steps

Step time: CUDA events around `--steps` steps after `--warmup` steps.  Launches: the CUDA kernel records of a
torch.profiler run over `--profile-steps` steps, per step (memcpy / memset records counted apart).  Prints the card
name and power limit, then one JSON line per workload, in the format of bench_pytorch_fitter.py.  Writes nothing.

    python scripts/bench_textured_autograd.py [--steps 50] [--warmup 5] [--profile-steps 20] [--size 320]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.dirname(os.path.abspath(__file__)), os.path.join(ROOT, "tests")]

from bench_fitter import card  # noqa: E402


def duck_workloads(W):
    import torch

    from deodr_b200.mesh_ops import CameraParams, DeviceMeshView
    from deodr_b200.pytorch import CameraPytorch, ColoredTriMeshPytorch, Scene3DPytorch

    H = W * 3 // 4
    d = dict(np.load(os.path.join(ROOT, "tests", "golden", "duck_textured.npz")))
    texture = d["texture_u8"] / 255
    t = lambda a, g=False: torch.tensor(np.asarray(a, dtype=np.float64), device="cuda").requires_grad_(g)  # noqa: E731
    info = {"vertices": int(d["vertices"].shape[0]), "faces": int(d["faces"].shape[0]), "image": [H, W]}

    def autograd():
        mesh = ColoredTriMeshPytorch(d["faces"], t(d["vertices"], True), faces_uv=d["faces_uv"], uv=t(d["uv"], True),
                                     texture=t(texture, True))
        scene = Scene3DPytorch()
        scene.set_mesh(mesh)
        scene.set_light(t(d["light_directional"], True), t(0.2, True))
        scene.set_background_color(d["background_color"])
        camera = CameraPytorch(d[f"extrinsic_{W}"], d[f"intrinsic_{W}"], H, W, d["distortion"])
        with torch.no_grad():
            target = scene.render(camera) * 0.9

        def step():
            loss = ((scene.render(camera) - target) ** 2).sum()
            loss.backward()
            return loss

        return step

    def device_view():
        cam = CameraParams(d[f"extrinsic_{W}"], d[f"intrinsic_{W}"], d["distortion"])
        view = DeviceMeshView(d["faces"], d["vertices"].shape[0], cam, H, W, light_directional=d["light_directional"],
                              ambient=0.2, background_color=d["background_color"], uv=d["uv"], faces_uv=d["faces_uv"],
                              texture=texture)
        v = t(d["vertices"])
        target = view.render(v).clone() * 0.9

        def step():
            diff = view.render(v) - target
            view.backward(2 * diff)
            return (diff.double() ** 2).sum()

        return step

    return {"duck_autograd": (autograd, info), "duck_device_view": (device_view, info)}


def eigen_faces_workload():
    import torch

    import eigen_faces_ref as ef
    from deodr_b200.pytorch import CudaRenderCompare2DTextured
    from deodr_b200.renderer import DeviceScene

    d = ef.load_inputs()
    K = d["components"].shape[0]

    def make():
        scene = DeviceScene(ef.scene_of(d, d["points"], ef.texture_of(d, np.zeros(K))), "cuda")
        t = lambda a: torch.tensor(np.asarray(a, dtype=np.float64), device="cuda")  # noqa: E731
        mean, components = t(d["mean"]), t(d["components"])
        obs = torch.tensor(d["image_obs"], dtype=torch.float32, device="cuda")
        uv, shade, colors = t(d["points"] * ef.SIZE + 0.5), t(np.ones(36)), t(np.ones((36, 1)))
        grid = t(d["points"])
        border = torch.tensor(ef.on_border(d["points"]), device="cuda")
        points = grid.clone().requires_grad_(True)
        coefs = torch.zeros(K, dtype=torch.float64, device="cuda", requires_grad=True)

        def step():
            texture = (mean + coefs @ components).reshape(ef.SIZE, ef.SIZE, 1)
            loss = CudaRenderCompare2DTextured(points * ef.SIZE - 0.5, colors, uv, shade, texture, obs, None, scene)
            loss.backward()
            with torch.no_grad():
                points.sub_(ef.STEP_POINTS * points.grad)
                coefs.sub_(ef.STEP_COEFS * coefs.grad)
                points[border] = grid[border]
            points.grad, coefs.grad = None, None
            return loss

        return step

    return {"eigen_faces": (make, {"vertices": 36, "faces": 50, "image": [64, 64]})}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=20)
    ap.add_argument("--size", type=int, default=320, choices=(320, 640), help="duck image width")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    assert torch.cuda.is_available(), "bench_textured_autograd needs a GPU"
    print("card:", card(), flush=True)
    for name, (make, info) in {**duck_workloads(args.size), **eigen_faces_workload()}.items():
        step = make()
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.steps):
            loss = step()
        stop.record()
        torch.cuda.synchronize()
        step_ms = start.elapsed_time(stop) / args.steps
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_steps):
                step()
            torch.cuda.synchronize()
        kernels = copies = 0
        gpu_us = copy_us = 0.0
        for ev in prof.events():
            if ev.device_type.name != "CUDA":
                continue
            gpu_us += ev.device_time
            if ev.name.startswith(("Memcpy", "Memset")):
                copies += 1
                copy_us += ev.device_time
            else:
                kernels += 1
        line = {
            "workload": name, **info, "ms_per_step": round(step_ms, 4),
            "kernel_launches_per_step": kernels / args.profile_steps,
            "copies_per_step": copies / args.profile_steps,
            "all_gpu_activity_ms_per_step": round(gpu_us / 1000 / args.profile_steps, 4),
            "copy_activity_ms_per_step": round(copy_us / 1000 / args.profile_steps, 4),
            "loss_last": float(loss), "steps": args.steps,
        }
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
