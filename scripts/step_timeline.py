#!/usr/bin/env python
"""Timeline of bench.py's graph-replayed step: where the step's time goes between and at the ends of its kernels.

    python scripts/step_timeline.py --out DIR [--workloads c5,c4,c3] [--steps 50]

For each workload the step of `bench.py` (N = 1: refresh of ij / colours, gradient clear, forward, adjoint of the
workload's views) is captured as a CUDA graph and replayed `--steps` times under torch.profiler with CUDA activities.
The kernel records of the replayed steps go to DIR/<workload>_kernels.json; one JSON line per workload is printed
(and written as DIR/<workload>_summary.json) with, as medians over the steps:
  - each kernel's start and end relative to the step's first record;
  - idle time: the part of the step during which no kernel, memset or copy runs;
  - on a single view (c5, c3), the gaps of the main chain: memset -> k_bin -> k_tile_z -> k_edge_fwd (which also
    waits for the edge lists of the side chain) -> the adjoint's first kernel.
With a library built with -DDEODR_TILEZ_TAIL_CLOCKS it also reports k_tile_z's tail, the time from the dispatch of
its last CTA to the exit of its last CTA, from %globaltimer stamps over plain (not replayed) forwards:
    scripts/build_variant.sh tail -DDEODR_TILEZ_TAIL_CLOCKS
    DEODR_B200_LIB=$PWD/deodr_b200/libdeodr_b200_tail.so python scripts/step_timeline.py --out DIR
The card's name, power limit and SM clock are read in the same process."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CHAIN = ["memset", "k_bin", "k_tile_z", "k_edge_fwd"]
SIDE = ("k_bin_edges", "k_sort_tile_edges", "k_publish")


def card():
    import torch

    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10).stdout
        p, sm, smax = [x.strip() for x in q.strip().split(",")]
        out.update({"power_limit_w": float(p), "sm_mhz": float(sm), "sm_max_mhz": float(smax)})
    except Exception as exc:  # (reported, not guessed)
        out["nvidia_smi"] = f"unavailable: {type(exc).__name__}"
    return out


def short(name):
    return name.split("<")[0].split("(")[0].replace("void ", "").strip()


def setup(workload):
    """bench.py's step at N = 1 (its `compute`), on the workload's views."""
    import torch

    import bench
    from deodr_b200.renderer import DeviceScene, Renderer

    dev = torch.device("cuda:0")
    per_gpu = 8 if workload == "c4" else 1
    scenes = [bench.build_scene(workload, view=v, n_views=per_gpu) for v in range(per_gpu)]
    if workload == "c4":  # configs[3]: an RGB and a depth render of every view
        for v in range(per_gpu):
            d = bench.build_scene(workload, view=v, n_views=per_gpu)
            d.nb_colors, d.colors = 1, np.ascontiguousarray(d.depths[:, None])
            d.background_color = np.array([float(d.depths.max())])
            d.texture = np.zeros((2, 2, 1))
            scenes.append(d)
    renderer = Renderer(0)
    dss = [DeviceScene(s, dev) for s in scenes]
    ij_dev = [ds.t["ij"].clone() for ds in dss]
    colors_dev = [ds.t["colors"].clone() for ds in dss]
    rng = np.random.default_rng(1)
    image_bs = [torch.from_numpy(rng.random((s.height, s.width, s.nb_colors), dtype=np.float32) * 2 - 1).to(dev)
                for s in scenes]
    # every gradient slot in one flat buffer, cleared by one memset per step (as bench.py does)
    names = (("colors_b", "colors"), ("uv_b", "uv"), ("shade_b", "shade"), ("texture_b", "texture"), ("ij_b", "ij"))
    flat = torch.zeros(sum(ds.t[n].numel() for ds in dss for _, n in names), dtype=torch.float32, device=dev)
    grads, off = [], 0
    for ds in dss:
        g = {}
        for k, n in names:
            g[k] = flat[off:off + ds.t[n].numel()].view(ds.t[n].shape)
            off += ds.t[n].numel()
        grads.append(g)
    state = {"outs": None}

    def compute():
        for ds, ij, col in zip(dss, ij_dev, colors_dev):
            ds.update(ij=ij, colors=col)
        flat.zero_()
        state["outs"] = renderer.render_views(dss, bench.SIGMA, out=state["outs"])
        renderer.render_b_views(dss, bench.SIGMA, state["outs"], image_bs, grads)

    return renderer, dss, compute, len(scenes)


def split_steps(records, renders):
    """Records of consecutive replays -> one list per step.  A replay starts after the previous one has ended, so a step
    ends with the last adjoint kernel that follows its `renders` binning passes."""
    bins = [r for r in records if r["name"] == "k_bin"]
    steps, start = [], 0
    for s in range(len(bins) // renders):
        first_bin = bins[s * renders]["ts"]
        next_bin = bins[(s + 1) * renders]["ts"] if (s + 1) * renders < len(bins) else float("inf")
        bwd = [r for r in records if first_bin < r["ts"] < next_bin and ("bwd" in r["name"] or "finalize" in r["name"])]
        if not bwd:
            break
        end = max(r["ts"] + r["dur"] for r in bwd)
        step = [r for r in records[start:] if r["ts"] < end]
        steps.append(step)
        start += len(step)
    return steps


def idle(step):
    t0, busy, cur_s, cur_e = step[0]["ts"], 0.0, None, None
    for r in sorted(step, key=lambda r: r["ts"]):
        s, e = r["ts"], r["ts"] + r["dur"]
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                busy += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    busy += cur_e - cur_s
    span = cur_e - t0
    return span, span - busy


def chain_gaps(step):
    """Single view: idle gaps between consecutive kernels of the main chain (us)."""
    t0 = step[0]["ts"]
    first = {}
    for r in step:
        first.setdefault(r["name"], r)
    if "k_bin" not in first or "k_edge_fwd" not in first:
        return None
    memsets = [r for r in step if r["name"] == "memset" and r["ts"] <= first["k_bin"]["ts"]]
    end = lambda r: r["ts"] + r["dur"]  # noqa: E731
    bwd = [r for r in step if "bwd" in r["name"] and r["ts"] >= first["k_edge_fwd"]["ts"]]
    gaps = {}
    if memsets:
        gaps["memset -> k_bin"] = first["k_bin"]["ts"] - end(memsets[-1])
    gaps["k_bin -> k_tile_z"] = first["k_tile_z"]["ts"] - end(first["k_bin"])
    side_end = max([end(first[n]) for n in SIDE if n in first] + [end(first["k_tile_z"])])
    gaps["k_tile_z (+ side chain) -> k_edge_fwd"] = first["k_edge_fwd"]["ts"] - side_end
    gaps["k_edge_fwd -> adjoint"] = min(r["ts"] for r in bwd) - end(first["k_edge_fwd"]) if bwd else None
    gaps["side chain end - k_tile_z end"] = side_end - end(first["k_tile_z"])
    return {k: (None if v is None else round(v, 2)) for k, v in gaps.items()}, {
        n: (round(r["ts"] - t0, 2), round(end(r) - t0, 2)) for n, r in first.items()}


def tail_stamps(renderer, dss, passes=20):
    from deodr_b200 import _cabi

    import bench

    lib = _cabi.load()
    if not hasattr(lib, "deodr_b200_tilez_tail_clocks"):
        return None
    fn = lib.deodr_b200_tilez_tail_clocks
    fn.argtypes = [C.POINTER(C.c_ulonglong)]
    st = (C.c_ulonglong * 3)()
    renderer.set_deferred(False)
    tails, durs = [], []
    for i in range(passes + 2):
        _cabi.check(fn(st))  # (also synchronises: one forward at a time)
        renderer.render_views(dss[:1], bench.SIGMA)
        _cabi.check(fn(st))
        if i >= 2:
            tails.append((st[2] - st[1]) / 1e3)
            durs.append((st[2] - st[0]) / 1e3)
    return {"tail_us_median": round(statistics.median(tails), 2), "tail_us_min": round(min(tails), 2),
            "tail_us_max": round(max(tails), 2), "first_start_to_last_exit_us_median": round(statistics.median(durs), 2),
            "passes": passes, "source": "%globaltimer stamps of thread 0 of every CTA, plain forwards of the first view"}


def run(workload, steps, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile

    renderer, dss, compute, renders = setup(workload)
    for _ in range(3):
        compute()
    torch.cuda.synchronize()
    renderer.set_deferred(True)
    cap = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(cap):
        with torch.cuda.graph(graph, stream=cap, capture_error_mode="thread_local"):
            compute()
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    renderer.status()
    trace = os.path.join(out_dir, f"{workload}.pt.trace.json")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            graph.replay()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    renderer.status()
    events = json.load(open(trace))["traceEvents"]
    records = []
    for e in events:
        cat = e.get("cat", "")
        if cat in ("kernel", "gpu_memset", "gpu_memcpy") and "dur" in e:
            records.append({"name": "memset" if cat == "gpu_memset" else "memcpy" if cat == "gpu_memcpy" else short(e["name"]),
                            "ts": float(e["ts"]), "dur": float(e["dur"])})
    records.sort(key=lambda r: r["ts"])
    os.remove(trace)
    step_list = split_steps(records, renders)
    json.dump([[dict(r, ts=round(r["ts"], 3)) for r in s] for s in step_list],
              open(os.path.join(out_dir, f"{workload}_kernels.json"), "w"))
    spans, idles, gap_rows, times = [], [], [], []
    for s in step_list:
        span, gap = idle(s)
        spans.append(span)
        idles.append(gap)
        if renders == 1:
            cg = chain_gaps(s)
            if cg:
                gap_rows.append(cg[0])
                times.append(cg[1])
    med = lambda xs: round(statistics.median(xs), 2) if xs else None  # noqa: E731
    summary = {"workload": workload, "renders_per_step": renders, "steps": len(step_list),
               "step_span_us": med(spans), "idle_us": med(idles)}
    if gap_rows:
        summary["main_chain_gaps_us"] = {k: med([g[k] for g in gap_rows if g[k] is not None]) for k in gap_rows[0]}
        summary["kernel_start_end_us"] = {n: [med([t[n][0] for t in times if n in t]), med([t[n][1] for t in times if n in t])]
                                          for n in times[0]}
    tail = tail_stamps(renderer, dss)
    summary["tile_z_tail"] = tail if tail else "not measured (library built without -DDEODR_TILEZ_TAIL_CLOCKS)"
    return summary


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--workloads", default="c5,c4,c3")
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "step_timeline.py needs a GPU"
    torch.cuda.set_device(0)
    os.makedirs(args.out, exist_ok=True)
    from deodr_b200 import _cabi

    info = {"card": card(), "lib": os.path.basename(_cabi.LIB_PATH)}
    print(json.dumps(info), flush=True)
    for wl in args.workloads.split(","):
        summary = dict(run(wl, args.steps, args.out), **info)
        json.dump(summary, open(os.path.join(args.out, f"{wl}_summary.json"), "w"), indent=1)
        print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
