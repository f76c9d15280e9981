#!/usr/bin/env python
"""Where a thread's time goes in the small-triangle adjoint (k_small_tri_bwd), per phase, and how many pixels its
triangle owns.

Needs a measurement build of the library (the clock64() counters are compiled in only with the switch):
    scripts/build_variant.sh sb_clocks -DDEODR_SMALLBWD_PHASE_CLOCKS
    DEODR_B200_LIB=$PWD/deodr_b200/libdeodr_b200_sb_clocks.so python scripts/small_bwd_phases.py --workload c5

Runs `--passes` steps of bench.py's workload (forward + adjoint of its views, as scripts/step_timeline.py sets them
up) and prints one JSON line: the thread cycles spent in each phase of small_triangle_adjoint summed over every thread
(their mean per thread and their share of the total), the threads that own no pixel (hidden triangles), and the
histogram of owned pixels per thread.  Phases (phases.h, SB_*): `walk` = vertex gather, bounds and the search for the
owned pixels (owner reads, tie lookups); `edge_mask` = clearing the pixels of tiles with silhouette edges; `setup` =
tri_attr and the colour gradients; `pixels` = the per-pixel loop; `scatter` = the atomics.  The counters perturb the
kernel a little (one clock64() per phase boundary, one warp reduction per thread): the split is the measurement, the
kernel time is bench.py's."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

PHASES = ["walk", "edge_mask", "setup", "pixels", "scatter"]  # phases.h SB_* order
SB_HIST = 65


def main():
    import torch

    import step_timeline
    from deodr_b200 import _cabi

    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c5", choices=["c3", "c4", "c5"])
    ap.add_argument("--passes", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "small_bwd_phases.py needs a GPU"

    lib = _cabi.load()
    if not hasattr(lib, "deodr_b200_small_bwd_phase_clocks"):
        sys.exit(f"{_cabi.LIB_PATH} was built without -DDEODR_SMALLBWD_PHASE_CLOCKS (see this script's docstring)")
    fn = lib.deodr_b200_small_bwd_phase_clocks
    fn.argtypes = [C.POINTER(C.c_ulonglong), C.POINTER(C.c_uint)]
    clocks = (C.c_ulonglong * (len(PHASES) + 2))()
    hist = (C.c_uint * SB_HIST)()

    torch.cuda.set_device(0)
    renderer, dss, compute, renders = step_timeline.setup(args.workload)
    for _ in range(3):  # plan + warm-up
        compute()
    _cabi.check(fn(clocks, hist))  # clears the counters
    for _ in range(args.passes):
        compute()
    _cabi.check(fn(clocks, hist))
    renderer.status()

    threads, hidden = clocks[len(PHASES)], clocks[len(PHASES) + 1]
    total = sum(clocks[i] for i in range(len(PHASES)))
    h = np.array(hist[:], dtype=np.int64)
    owners = h[1:].sum()
    out = {
        "workload": args.workload,
        "lib": os.path.basename(_cabi.LIB_PATH),
        "card": step_timeline.card(),
        "passes": args.passes,
        "renders_per_step": renders,
        "threads_per_step": int(threads // args.passes),
        "hidden_threads_per_step": int(hidden // args.passes),
        "hidden_share": round(hidden / max(threads, 1), 4),
        "cycles_per_thread": {p: round(clocks[i] / max(threads, 1), 1) for i, p in enumerate(PHASES)},
        "cycles_per_thread_total": round(total / max(threads, 1), 1),
        "share": {p: round(clocks[i] / max(total, 1), 4) for i, p in enumerate(PHASES)},
        "owned_pixels": {
            "mean_over_owners": round(float((h[1:] * np.arange(1, SB_HIST)).sum() / max(owners, 1)), 2),
            "histogram_per_step": {str(n): int(h[n] // args.passes) for n in range(SB_HIST) if h[n]},
        },
    }
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
