"""Strongly connected components on one GPU: time per call on the directed RMAT graph of the PageRank benchmark (the library's
device generator, edge factor 16, as generated: multi-edges and self-loops kept), the per-phase rounds and resolved vertices
of CUGRAPH_B200_SCC_TRACE, single-GPU WCC on the symmetrised graph for comparison, and parity with
scipy.sparse.csgraph.connected_components(connection="strong") at a smaller scale (scipy's time there is the CPU figure).
    python scripts/scc_bench.py --scale 24 [--calls 5] [--parity-scale 20] [--out result.json]
Times: host clock around each call, which ends in a device synchronise (the result is copied back), after one warm-up call."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    except OSError:
        return "unknown (nvidia-smi not found)"
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, calls):
    import torch
    fn()  # warm-up (SCC: also builds the graph's in-edge view)
    torch.cuda.synchronize()
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"min_ms": min(ts), "median_ms": float(np.median(ts)), "max_ms": max(ts), "calls": calls}


def traced(graph):
    """one SCC call on a handle created with CUGRAPH_B200_SCC_TRACE set; returns the trace lines (written to stderr)"""
    from cugraph_b200 import pylibcugraph as plc
    os.environ["CUGRAPH_B200_SCC_TRACE"] = "1"
    h = plc.ResourceHandle()
    del os.environ["CUGRAPH_B200_SCC_TRACE"]
    with tempfile.TemporaryFile(mode="w+") as f:
        sys.stderr.flush()
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            plc.strongly_connected_components(h, graph, None, None, None, None, False)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        return [ln.rstrip() for ln in f if ln.startswith("scc ")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--parity-scale", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from cugraph_b200 import pylibcugraph as plc
    from cugraph_b200.generators import rmat_edgelist
    assert torch.cuda.is_available(), "scc_bench needs a GPU"
    out = {"card": card(), "scale": a.scale, "edge_factor": 16}
    print("card (name, power limit):", out["card"], flush=True)

    def directed(scale):
        src, dst = rmat_edgelist(scale, 16 << scale, seed=0)
        h = plc.ResourceHandle()
        g = plc.SGGraph(h, plc.GraphProperties(is_symmetric=False, is_multigraph=True), src, dst, store_transposed=False,
                        renumber=True)
        return src, dst, h, g

    # SCC at the benchmark scale
    src, dst, h, g = directed(a.scale)
    out["edges"] = int(src.numel())
    res = {}

    def run_scc():
        res["v"], res["l"] = plc.strongly_connected_components(h, g, None, None, None, None, False)
    out["scc"] = timed(run_scc, a.calls)
    out["scc"]["vertices"] = int(res["v"].numel())
    out["scc"]["components"] = int(torch.unique(res["l"]).numel())
    out["scc"]["largest"] = int(torch.unique(res["l"], return_counts=True)[1].max())
    out["scc_trace"] = traced(g)
    del g, h, res
    print("scc:", json.dumps(out["scc"]), flush=True)
    for ln in out["scc_trace"]:
        print("  " + ln, flush=True)

    # WCC on the symmetrised graph
    s2, d2 = torch.cat([src, dst]), torch.cat([dst, src])
    del src, dst
    h = plc.ResourceHandle()
    g = plc.SGGraph(h, plc.GraphProperties(is_symmetric=True, is_multigraph=True), s2, d2, store_transposed=False, renumber=True)
    del s2, d2
    out["wcc_symmetrised"] = timed(lambda: plc.weakly_connected_components(h, g, None, None, None, None, False), a.calls)
    del g, h
    print("wcc (symmetrised):", json.dumps(out["wcc_symmetrised"]), flush=True)
    torch.cuda.empty_cache()

    # parity with scipy at a smaller scale
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    src, dst, h, g = directed(a.parity_scale)
    t0 = time.perf_counter()
    verts, labels = plc.strongly_connected_components(h, g, None, None, None, None, False)
    torch.cuda.synchronize()
    gpu_ms = (time.perf_counter() - t0) * 1e3
    s, d = src.cpu().numpy(), dst.cpu().numpy()
    ids, inv = np.unique(np.concatenate([s, d]), return_inverse=True)
    m = sp.coo_matrix((np.ones(s.size, np.float32), (inv[:s.size], inv[s.size:])), shape=(ids.size, ids.size)).tocsr()
    t0 = time.perf_counter()
    n, lab = connected_components(m, directed=True, connection="strong")
    cpu_ms = (time.perf_counter() - t0) * 1e3
    pos = np.searchsorted(ids, verts.cpu().numpy())
    ref = lab[pos]
    got = labels.cpu().numpy()
    same = len(np.unique(got)) == n and len(set(zip(ref.tolist(), got.tolist()))) == n
    out["parity"] = {"scale": a.parity_scale, "components": int(n), "same_partition": bool(same),
                     "scipy_ms": cpu_ms, "gpu_first_call_ms": gpu_ms}
    print("parity:", json.dumps(out["parity"]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
