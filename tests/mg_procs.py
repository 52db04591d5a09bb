"""One process harness for the multi-process tests: `world` spawned ranks run a module-level worker inside one process group,
gloo on the CPU (optionally over the emulated library, tests/emu_py.py) or NCCL with one GPU per rank, and the test gets
every rank's result."""
import contextlib
import os
import socket

import pytest


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_main(rank, world, port, backend, emulated, env, worker, args, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ.update(env)
    import torch
    import torch.distributed as dist
    if backend == "nccl":
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    from tests.emu_py import emulated_python_surface
    with emulated_python_surface() if emulated else contextlib.nullcontext():
        res = [None] * world
        dist.all_gather_object(res, worker(rank, world, *args))
        if rank == 0:
            q.put(res)
        dist.barrier()
    dist.destroy_process_group()


def run(worker, world, *args, backend="gloo", emulated=False, env=None, timeout=900):
    """worker(rank, world, *args) on `world` ranks (env: variables set before the process group starts); returns the
    workers' results in rank order.  NCCL skips the test when fewer than `world` GPUs are visible."""
    import torch
    import torch.multiprocessing as mp
    if backend == "nccl" and torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, backend, emulated, env or {}, worker, args, q))
             for r in range(world)]
    for p in procs:
        p.start()
    res = q.get(timeout=timeout)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    return res
