"""Per-kernel time of one PageRank call (RMAT-24 ef-16 by default, 100 iterations, the bench.py workload) under
torch.profiler: prints one JSON line with the time per iteration of each kernel of the pull sweep and of the PageRank
vertex pass, and the card it ran on.  A first, unprofiled call builds the graph's layouts and warms every kernel up.

    python scripts/sweep_profile.py [--scale 24] [--trace DIR]
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
    args = ap.parse_args()
    src, dst = rmat_edgelist(args.scale, 16 << args.scale, seed=0)
    h = plc.ResourceHandle()
    g = plc.SGGraph(h, plc.GraphProperties(is_symmetric=False, is_multigraph=True), src.cuda(), dst.cuda(),
                    store_transposed=True, renumber=True)
    del src, dst

    def call():
        plc.pagerank(h, g, None, None, None, None, 0.85, 0.0, ITERS, False, fail_on_nonconvergence=False)
        torch.cuda.synchronize()

    call()  # layouts, out-weights, first launches
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
           "ms_per_iteration": {k: round(total[k] / 1e3 / ITERS, 4) for k in KERNELS},
           "launches": count}
    out["ms_per_iteration"]["sweep"] = round(sum(out["ms_per_iteration"][k] for k in ("k_sweep", "k_sweep_finish", "k_sweep_tail")), 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
