"""bench.py's N>1 arm: 2D-partitioned PageRank, one process per GPU (launched under torchrun)."""
from __future__ import annotations

import json
import os
import time

import torch
import torch.distributed as dist


def mg_parity(groups, alpha, scale=16, iters=30):
    """MG = SG on a small graph (the protocol of cpp/tests/link_analysis/mg_pagerank_test.cpp:158-248): RMAT-`scale` through
    MGGraph.pagerank on all ranks, the same edge list through the single-GPU C-ABI on rank 0; every vertex within 1e-6
    relative.  Returns {max_rel, ok, vertices} on rank 0 (None elsewhere).  A machine with one GPU cannot run the multi-GPU
    tests, so on several GPUs this is where the NCCL path's correctness becomes visible."""
    from cugraph_b200 import mg
    from cugraph_b200.generators import rmat_edgelist
    rank, world = dist.get_rank(), dist.get_world_size()
    E_local = (16 << scale) // world
    src, dst = rmat_edgelist(scale, E_local, seed=77 + rank)
    G = mg.MGGraph(src, dst, None, groups)
    verts, pr, _, _ = G.pagerank(alpha, 0.0, iters)
    # multi-GPU BFS from the first source of rank 0's edge list (distances must equal the single-GPU ones bit for bit); a
    # failure is reported in the line, it does not cost the PageRank measurement
    first = [int(src[0].item()) if rank == 0 else None]
    dist.broadcast_object_list(first, src=0)
    bfs_err, bv, bd = None, None, None
    try:
        bv, bd, _ = G.bfs(first[0], compute_predecessors=False)
        bv, bd = bv.cpu(), bd.cpu()
    except Exception as e:  # noqa: BLE001
        bfs_err = f"{type(e).__name__}: {e}"[:200]
    parts = [None] * world
    dist.all_gather_object(parts, (src.cpu(), dst.cpu(), verts.cpu(), pr.cpu(), bv, bd, bfs_err))
    del G
    if rank != 0:
        return None
    from cugraph_b200 import pylibcugraph as plc
    s_all = torch.cat([p[0] for p in parts]).cuda()
    d_all = torch.cat([p[1] for p in parts]).cuda()
    v_mg = torch.cat([p[2] for p in parts]).long()
    p_mg = torch.cat([p[3] for p in parts]).double()
    h = plc.ResourceHandle()
    g1 = plc.SGGraph(h, plc.GraphProperties(is_multigraph=True), s_all, d_all, store_transposed=True, renumber=True)
    v1, p1, _ = plc.pagerank(h, g1, None, None, None, None, alpha, 0.0, iters, False, fail_on_nonconvergence=False)
    n = 1 << scale
    a = torch.zeros(n, dtype=torch.float64)
    b = torch.zeros(n, dtype=torch.float64)
    a[v_mg] = p_mg
    b[v1.cpu().long()] = p1.cpu().double()
    same_set = bool(((a > 0) == (b > 0)).all())
    rel = ((a - b).abs() / b.clamp_min(1e-300))[b > 0].max().item() if bool((b > 0).any()) else 0.0
    out = {"max_rel": rel, "ok": bool(same_set and rel < 1e-6), "vertices": int((b > 0).sum()), "scale": scale, "iterations": iters}
    errs = [p[6] for p in parts if p[6]]
    if errs:
        out["bfs"] = {"ok": False, "error": errs[0]}
    else:
        try:
            g2 = plc.SGGraph(h, plc.GraphProperties(is_multigraph=True), s_all, d_all, store_transposed=False, renumber=True)
            srcs = torch.tensor([int(parts[0][0][0])], dtype=s_all.dtype, device="cuda")
            d1, _, v1b = plc.bfs(h, g2, srcs, False, -1, False, False)  # the graph is directed: no direction optimisation
            imax = torch.iinfo(torch.int32).max
            da = torch.full((n,), imax, dtype=torch.int64)
            db = torch.full((n,), imax, dtype=torch.int64)
            da[torch.cat([p[4] for p in parts]).long()] = torch.cat([p[5] for p in parts]).long()
            db[v1b.cpu().long()] = d1.cpu().long()
            reached = int((db < imax).sum())
            out["bfs"] = {"ok": bool((da == db).all()), "reached": reached, "levels": int(db[db < imax].max()) if reached else 0}
        except Exception as e:  # noqa: BLE001
            out["bfs"] = {"ok": False, "error": f"{type(e).__name__}: {e}"[:200]}
    return out


def run_mg_pagerank(args, metric_name, alpha, iters, ClockSampler, peaks):
    from cugraph_b200 import mg
    from cugraph_b200.generators import rmat_edgelist
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", str(args.gpus)))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29517")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    groups = mg.make_groups()
    parity = mg_parity(groups, alpha)
    ok = torch.tensor([1 if (rank != 0 or parity["ok"]) else 0], dtype=torch.int32, device="cuda")
    dist.broadcast(ok, src=0)
    if int(ok.item()) == 0:  # every rank leaves: a wrong multi-GPU result must not produce a bench line
        raise SystemExit(f"multi-GPU PageRank does not match the single-GPU result: {parity}")
    # weak scaling: 2^28 edge draws per GPU (= the N=1 workload); N=8 is BASELINE's scale-27 configuration
    scale = args.scale if args.scale else 24 + max(0, (world - 1).bit_length())
    E_total = 16 << scale
    E_local = E_total // world
    src, dst = rmat_edgelist(scale, E_local, seed=1000 + rank)
    h_src = h_dst = None
    if world <= 8:
        h_src = torch.empty(E_local, dtype=torch.int32).pin_memory()
        h_dst = torch.empty(E_local, dtype=torch.int32).pin_memory()
        h_src.copy_(src)
        h_dst.copy_(dst)
    G = mg.MGGraph(src, dst, None, groups)
    del src, dst
    torch.cuda.empty_cache()

    def step():
        return G.pagerank(alpha, 0.0, iters)

    def timed(fn, n):
        dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            out = fn()
        torch.cuda.synchronize()
        dt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device="cuda")
        dist.all_reduce(dt, op=dist.ReduceOp.MAX)
        return float(dt.item()), out

    for _ in range(args.warmup):
        step()
    sampler = ClockSampler(local)
    l0 = G.handle.launch_count()
    if rank == 0:
        sampler.start()
    wall, (verts, pr, _, _) = timed(step, args.steps)
    clocks = sampler.stop() if rank == 0 else None
    launches = G.handle.launch_count() - l0
    value = E_total * iters * args.steps / wall / 1e6
    # mass check: PageRank sums to 1 over all ranks
    mass = pr.double().sum().reshape(1)
    dist.all_reduce(mass)

    # multi-GPU BFS on the bench graph (pull steps on every block, frontier / visited flags all-gathered per level): a few
    # sources, time per traversal as the max over ranks; never fatal for the PageRank line
    mg_bfs = None
    try:
        from cugraph_b200.mg import vertex_owner  # noqa: F401
        srcs = [None] * 4
        if rank == 0:
            if h_src is not None:
                pick = torch.randint(0, h_src.numel(), (4,), generator=torch.Generator().manual_seed(5))
                srcs = [int(h_src[int(i)]) for i in pick]
        dist.broadcast_object_list(srcs, src=0)
        if srcs[0] is not None:
            G.bfs(srcs[0], compute_predecessors=False)  # warm-up
            times, reached = [], []
            for sv in srcs:
                tb, (bv, bd, _) = timed(lambda: G.bfs(sv, compute_predecessors=False), 1)
                r = (bd < torch.iinfo(torch.int32).max).sum().reshape(1).to(torch.int64)
                dist.all_reduce(r)
                times.append(tb)
                reached.append(int(r.item()))
            hm = len(times) / sum(t / E_total for t in times) / 1e6   # harmonic-mean MTEPS over the sources (Graph500 style)
            mg_bfs = {"sources": len(times), "ms_mean": 1e3 * sum(times) / len(times), "mteps_harmonic": hm,
                      "reached_mean": sum(reached) / len(reached), "direction": "pull on every level (flags all-gathered)"}
    except Exception as e:  # noqa: BLE001
        mg_bfs = {"error": f"{type(e).__name__}: {e}"[:200]}

    # roofline of the local sweep (no communication): CUDA events on the stream the kernels run on
    import ctypes as C
    from cugraph_b200.pylibcugraph.utils import View
    xg = torch.full((G.x_elems,), 1.0 / G.part.n_global, dtype=G.dtype, device="cuda")
    yp = torch.zeros(G.span, dtype=G.dtype, device="cuda")
    vx, vy, err = View(xg), View(yp), C.c_void_p()
    for _ in range(3):
        G.lib.cugraph_b200_block_pull_sweep(G.handle.ptr, G.block, vx.ptr, vy.ptr, alpha, C.byref(err))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    nsw = 20
    e0.record()
    for _ in range(nsw):
        G.lib.cugraph_b200_block_pull_sweep(G.handle.ptr, G.block, vx.ptr, vy.ptr, alpha, C.byref(err))
    e1.record()
    torch.cuda.synchronize()
    ms_sweep = e0.elapsed_time(e1) / nsw
    alg_bytes = G.num_edges_local * 4.0 + (G.n_rows + 1) * 4.0 + G.n_cols * 4.0 + G.n_rows * 4.0
    peak, peak_src = peaks()
    ach = alg_bytes / (ms_sweep * 1e-3) / 1e9
    t = torch.tensor([ach], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    roofline = {"bound": "hbm", "achieved": float(t.item()), "peak": peak, "unit": "GB/s", "frac": float(t.item()) / peak,
                "traffic": None, "peak_source": peak_src, "kernel": "local block pull sweep (min over ranks)",
                "ms_per_sweep": ms_sweep, "algorithmic_bytes_per_sweep": alg_bytes}

    # e2e: pinned host edge list -> H2D -> 2D partition + block build -> 100 iterations -> D2H
    e2e = None
    if h_src is not None:
        del G
        torch.cuda.empty_cache()

        def e2e_step():
            s = h_src.cuda(non_blocking=True)
            d = h_dst.cuda(non_blocking=True)
            g2 = mg.MGGraph(s, d, None, groups)
            v, p, _, _ = g2.pagerank(alpha, 0.0, iters)
            return v.cpu(), p.cpu()

        e2e_wall, (v, p) = timed(e2e_step, 1)
        e2e = {"value": E_total * iters / e2e_wall / 1e6, "unit": "MTEPS", "h2d_bytes_per_step": 2 * E_total * 4,
               "d2h_bytes_per_step": int(v.numel()) * 8 * world, "steps": 1, "ms_per_step": e2e_wall * 1e3,
               "includes": "pinned H2D of the edge list, 2D partition + block staging, 100 iterations, D2H of results"}
    if rank == 0:
        R, Cc = groups.R, groups.C
        out = {"metric": metric_name(scale, world), "value": value, "unit": "MTEPS", "n_gpus": world, "steps": args.steps,
               "warmup": args.warmup, "ms_per_step": wall / args.steps * 1e3, "higher_is_better": True, "scaling": "weak",
               "vs_baseline": None, "dtype": "f32", "data": "synthetic",
               "config": {"workload": f"pagerank_rmat{scale}_ef16_100it_2d{R}x{Cc}", "scale": scale, "edge_factor": 16,
                          "num_edges": E_total, "edges_per_gpu": E_local, "alpha": alpha, "iterations": iters,
                          "partition": f"2D {R}x{Cc} (all-gather group {R}, reduce-scatter group {Cc})",
                          "mass": float(mass.item()),
                          "mg_parity_ok": parity["ok"], "mg_parity_max_rel": parity["max_rel"],
                          "mg_parity_sample": f"RMAT-{parity['scale']} ef-16, {parity['iterations']} iterations, MG on {world} GPUs vs the single-GPU C-ABI on rank 0, {parity['vertices']} vertices",
                          "mg_bfs_parity": parity.get("bfs"), "mg_bfs": mg_bfs,
                          "l2": "inputs per sweep exceed the 50 MB L2; no explicit flush"},
               "clocks": clocks, "e2e": e2e, "gpu_launches": launches, "roofline": roofline, "cpu_baseline": None}
        print(json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()
