"""Per-kernel time of one PageRank call (RMAT-24 ef-16 by default, 100 iterations, the bench.py workload) under
torch.profiler: prints one JSON line with the time per iteration of each kernel of the pull sweep and of the PageRank
vertex pass, and the card it ran on.  A first, unprofiled call builds the graph's layouts and warms every kernel up.

The tail sweep may run beside the piece stream (CUGRAPH_B200_SWEEP_TAIL_SMS, --tail-sms), so the summed kernel times are
not the time of an iteration: "call_ms_per_iteration" is the device time of whole unprofiled calls (CUDA events on the
handle's stream, the fastest of three), per iteration.  Under CUDA_LAUNCH_BLOCKING=1 every kernel runs alone: the kernel
times of a split are then those of each side on its own share of the SMs.

    python scripts/sweep_profile.py [--scale 24] [--tail-sms K] [--trace DIR]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from cugraph_b200 import pylibcugraph as plc  # noqa: E402
from cugraph_b200.generators import rmat_edgelist  # noqa: E402

KERNELS = {  # reported name: the demangled kernel names it covers
    "k_sweep": lambda n: "k_sweep<" in n,
    "k_sweep_finish": lambda n: "k_sweep_finish<" in n,
    "k_sweep_tail": lambda n: "k_sweep_tail<" in n,
    "k_vertex_pass": lambda n: "k_vertex_pass<" in n,
    "k_finalize": lambda n: "k_finalize(" in n,
}
ITERS = 100


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = ""
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--trace", default=None, help="directory for a Chrome trace of the profiled call")
    ap.add_argument("--tail-sms", type=int, default=None, help="CUGRAPH_B200_SWEEP_TAIL_SMS for this run (default: as set)")
    args = ap.parse_args()
    if args.tail_sms is not None:  # read when the handle is made
        os.environ["CUGRAPH_B200_SWEEP_TAIL_SMS"] = str(args.tail_sms)
    src, dst = rmat_edgelist(args.scale, 16 << args.scale, seed=0)
    h = plc.ResourceHandle()
    g = plc.SGGraph(h, plc.GraphProperties(is_symmetric=False, is_multigraph=True), src.cuda(), dst.cuda(),
                    store_transposed=True, renumber=True)
    del src, dst

    def call():
        plc.pagerank(h, g, None, None, None, None, 0.85, 0.0, ITERS, False, fail_on_nonconvergence=False)
        torch.cuda.synchronize()

    call()  # layouts, out-weights, first launches
    from cugraph_b200 import _capi
    hstream = torch.cuda.ExternalStream(int(_capi.lib().cugraph_b200_handle_stream(h.ptr) or 0))
    calls = []
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(hstream)
        call()
        e1.record(hstream)
        torch.cuda.synchronize()
        calls.append(e0.elapsed_time(e1) / ITERS)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
    total = {k: 0.0 for k in KERNELS}
    count = {k: 0 for k in KERNELS}
    for ev in prof.key_averages():
        for k, match in KERNELS.items():
            if match(ev.key):
                us = getattr(ev, "self_device_time_total", None)
                total[k] += us if us is not None else ev.self_cuda_time_total
                count[k] += ev.count
    if args.trace:
        os.makedirs(args.trace, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.trace, "sweep_profile.pt.trace.json"))
    out = {"card": card(), "scale": args.scale, "iterations": ITERS,
           "tail_sms": os.environ.get("CUGRAPH_B200_SWEEP_TAIL_SMS", "default"),
           "launch_blocking": os.environ.get("CUDA_LAUNCH_BLOCKING", "0"),
           "call_ms_per_iteration": round(min(calls), 4), "call_ms_per_iteration_runs": [round(c, 4) for c in calls],
           "ms_per_iteration": {k: round(total[k] / 1e3 / ITERS, 4) for k in KERNELS},
           "launches": count}
    out["ms_per_iteration"]["sweep"] = round(sum(out["ms_per_iteration"][k] for k in ("k_sweep", "k_sweep_finish", "k_sweep_tail")), 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
