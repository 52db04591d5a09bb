"""P ranks of torch.distributed in ONE process: run(world, fn, *args) calls fn(rank, world, *args) on one thread per rank
while cugraph_b200.mg.dist is an in-process stand-in for the NCCL collectives mg.py calls, so the one-process multi-GPU
tests run MGGraph's own drivers on one device (or on the CPU over the emulated library, tests/emu_py.py).

One rank runs at a time and hands the turn on only inside a collective or when it returns: the library and the emulator
are never entered concurrently and a run is deterministic.  The ranks share the device and torch's current stream; a
collective is torch ops on it over the members' tensors, in group-rank order.  Every collective checks that all members
made the same call (kind, op, dtypes, sizes), and a deadlock (no rank can run while some rank waits in a collective) is
seen exactly.  Either way every rank still running gets an MGWorldError naming the ranks and their calls: where NCCL
would hang, the test fails."""
import threading

import numpy as np
import torch
import torch.distributed as torch_dist


class MGWorldError(RuntimeError):
    """members of a group made different collective calls, or some rank waits in a collective that cannot complete"""


class _Group:
    def __init__(self, ranks, name=None):
        self.ranks = tuple(ranks)
        self.name = name or f"group {list(self.ranks)}"

    def __repr__(self):
        return self.name


class _Work:
    def wait(self):
        return True


_REDUCE = {"SUM": torch.sum, "MAX": torch.amax, "MIN": torch.amin}


class _Call:
    """one member's collective call; key() must be the same for every member"""

    def __init__(self, kind, out, inp, op=None, splits=None):
        self.kind, self.out, self.inp, self.op, self.splits = kind, out, inp, op, splits   # splits: (out, in)
        self.outs = out if isinstance(out, list) else [out]

    def key(self):
        sizes = () if self.splits else (self.inp.numel(), tuple(t.numel() for t in self.outs))
        return self.kind, self.op and self.op.name, self.inp.dtype, tuple(t.dtype for t in self.outs), sizes

    def __str__(self):
        t = lambda x: f"{str(x.dtype)[6:]}[{x.numel()}]"  # noqa: E731
        return (f"{self.kind}({self.op.name + ', ' if self.op else ''}in {t(self.inp)}, out {', '.join(map(t, self.outs))}"
                f"{', out/in splits %s' % (self.splits,) if self.splits else ''})")


def _size_error(calls):
    """why the members' sizes do not fit together, or None (all_reduce: equal sizes, in key())"""
    n, c = len(calls), calls[0]
    if c.kind in ("all_gather_into_tensor", "all_gather", "reduce_scatter_tensor"):
        whole = c.inp.numel() if c.kind == "reduce_scatter_tensor" else sum(t.numel() for t in c.outs)
        part = c.out.numel() if c.kind == "reduce_scatter_tensor" else c.inp.numel()
        return None if whole == n * part else f"{whole} elements for {n} members of {part}"
    for i, c in enumerate(calls if c.kind == "all_to_all_single" else []):
        for j, d in enumerate(calls):
            if c.splits[1][j] != d.splits[0][i]:
                return f"rank {i} of the group sends {c.splits[1][j]} elements to rank {j}, which expects {d.splits[0][i]}"
    return None


def _apply(calls):
    """the collective over the members' calls, in group-rank order"""
    c0 = calls[0]
    if c0.kind == "all_reduce":
        total = _REDUCE[c0.op.name](torch.stack([c.inp for c in calls]), 0)
        for c in calls:
            c.inp.copy_(total)
    elif c0.kind == "all_gather_into_tensor":
        cat = torch.cat([c.inp.reshape(-1) for c in calls])
        for c in calls:
            c.out.copy_(cat.view_as(c.out))
    elif c0.kind == "all_gather":
        for c in calls:
            for t, src in zip(c.outs, calls):
                t.copy_(src.inp)
    elif c0.kind == "reduce_scatter_tensor":
        total = _REDUCE[c0.op.name](torch.stack([c.inp.reshape(-1) for c in calls]), 0)
        m = c0.out.numel()
        for j, c in enumerate(calls):
            c.out.copy_(total[j * m:(j + 1) * m].view_as(c.out))
    else:   # all_to_all_single
        pieces = [torch.split(c.inp, c.splits[1]) for c in calls]
        for j, c in enumerate(calls):
            c.out.copy_(torch.cat([p[j] for p in pieces]))


class _World:
    """the stand-in for torch.distributed: the calls mg.py makes, on the calling thread's rank"""
    ReduceOp = torch_dist.ReduceOp

    def __init__(self, size):
        self.size = size
        self._world = _Group(range(size), "the world group")
        self._groups = {}
        self._cond = threading.Condition()
        self._tls = threading.local()
        self._running = 0                   # the one rank that runs
        self._ready = set(range(1, size))   # ranks that can run when they get the turn
        self._waiting = {}                  # rank -> (group, call) it waits in
        self._open = {}                     # group -> {rank: call}, in arrival order
        self._done = set()
        self._error = None
        self.results = [None] * size
        self.exceptions = []                # in the order the ranks raised them

    # ---- torch.distributed
    def get_world_size(self, group=None):
        return len((group or self._world).ranks)

    def get_rank(self, group=None):
        return (group or self._world).ranks.index(self._tls.rank)

    def new_group(self, ranks):
        return self._groups.setdefault(tuple(ranks), _Group(ranks))

    def get_backend(self, group=None):
        return "nccl"

    def all_reduce(self, tensor, op=torch_dist.ReduceOp.SUM, group=None, async_op=False):
        self._collective(group, _Call("all_reduce", tensor, tensor, op))
        return _Work() if async_op else None

    def all_gather(self, tensor_list, tensor, group=None):
        self._collective(group, _Call("all_gather", list(tensor_list), tensor))

    def all_gather_into_tensor(self, output_tensor, input_tensor, group=None):
        self._collective(group, _Call("all_gather_into_tensor", output_tensor, input_tensor))

    def reduce_scatter_tensor(self, output, input, op=torch_dist.ReduceOp.SUM, group=None):
        self._collective(group, _Call("reduce_scatter_tensor", output, input, op))

    def all_to_all_single(self, output, input, output_split_sizes=None, input_split_sizes=None, group=None):
        n = self.get_world_size(group)
        splits = [list(sp) if sp is not None else [t.numel() // n] * n
                  for sp, t in ((output_split_sizes, output), (input_split_sizes, input))]
        self._collective(group, _Call("all_to_all_single", output, input, splits=tuple(splits)))

    # ---- the turn
    def _main(self, rank, fn, args):
        self._tls.rank = rank
        try:
            with self._cond:
                self._cond.wait_for(lambda: self._running == rank)
                self._check_failed(rank)
            self.results[rank] = fn(rank, self.size, *args)
        except BaseException as e:  # noqa: BLE001  (re-raised by run)
            with self._cond:
                self.exceptions.append(e)
        finally:
            with self._cond:
                self._done.add(rank)
                self._pass_turn(rank)

    def _check_failed(self, rank):
        if self._error is not None:
            raise MGWorldError(f"rank {rank}: {self._error}")

    def _fail(self, rank, message):
        self._error = message
        self._check_failed(rank)

    def _pass_turn(self, rank):
        """(lock held) the next rank after `rank` that can run gets the turn.  None can while some rank waits: deadlock.
        After a failure every rank that has not returned gets the turn in order, to raise and unwind alone."""
        order = [(rank + k) % self.size for k in range(1, self.size + 1)]
        nxt = None
        if self._error is None:
            nxt = next((r for r in order if r in self._ready), None)
            if nxt is None and self._waiting:
                waits = [f"rank {r} waits in {c} on {g}" for r, (g, c) in sorted(self._waiting.items())]
                gone = [f"rank {r} returned" for r in sorted(self._done)]
                self._error = "collective deadlock: " + "; ".join(waits + gone)
        if self._error is not None:
            nxt = next((r for r in order if r not in self._done), None)
        self._running = nxt
        self._ready.discard(nxt)
        self._cond.notify_all()

    def _collective(self, group, call):
        group = group or self._world
        rank = self._tls.rank
        with self._cond:
            self._check_failed(rank)
            if rank not in group.ranks:
                self._fail(rank, f"rank {rank} calls {call} on {group}, which it is not a member of")
            members = self._open.setdefault(group, {})
            members[rank] = call
            first_rank, first = next(iter(members.items()))
            if call.key() != first.key():
                self._fail(rank, f"collective mismatch on {group}: rank {first_rank} calls {first}, rank {rank} calls {call}")
            if len(members) < len(group.ranks):
                self._waiting[rank] = (group, call)
                self._pass_turn(rank)
                self._cond.wait_for(lambda: self._running == rank)
                self._check_failed(rank)
                return
            del self._open[group]
            calls = [members[r] for r in group.ranks]
            why = _size_error(calls)
            if why is not None:
                self._fail(rank, f"collective mismatch on {group}: {why}: "
                           + "; ".join(f"rank {r} calls {members[r]}" for r in group.ranks))
            _apply(calls)
            for r in group.ranks:
                if r != rank:
                    del self._waiting[r]
                    self._ready.add(r)


def run(world, fn, *args):
    """fn(rank, world, *args) on `world` ranks, one thread each, with cugraph_b200.mg.dist the stand-in; returns the
    results in rank order, or re-raises the first exception any rank raised"""
    from cugraph_b200 import mg
    w = _World(world)
    threads = [threading.Thread(target=w._main, args=(r, fn, args), name=f"rank {r}") for r in range(world)]
    saved, mg.dist = mg.dist, w
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        mg.dist = saved
    if w.exceptions:
        raise w.exceptions[0]
    return w.results


# ---- the tests' side
def grid_world(monkeypatch, R, Cc):
    """the world size of an R x C grid, with CUGRAPH_B200_MG_GRID set so that mg.grid_shape gives that orientation"""
    from cugraph_b200 import mg
    if R < Cc:
        monkeypatch.setenv("CUGRAPH_B200_MG_GRID", "wide")
    else:
        monkeypatch.delenv("CUGRAPH_B200_MG_GRID", raising=False)
    assert mg.grid_shape(R * Cc) == (R, Cc)
    return R * Cc


def share(rank, world, *arrays):
    """rank's contiguous slice of each array (the edge list, or (ids, values) pairs)"""
    n = len(arrays[0])
    lo, hi = rank * n // world, (rank + 1) * n // world
    return tuple(a[lo:hi] for a in arrays)


def graph(rank, world, s, d, w=None, dtype=np.float32, device="cpu"):
    """rank's MGGraph built from its share of the edge list (vertex ids as given)"""
    from cugraph_b200 import mg
    s, d, *rest = share(rank, world, s, d, *([] if w is None else [w]))
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(device)  # noqa: E731
    return mg.MGGraph(t(s), t(d), t(rest[0]) if rest else None,
                      dtype=torch.float64 if np.dtype(dtype) == np.float64 else torch.float32)


def by_id(parts, V, fill=0, dtype=np.float64):
    """the ranks' (vertices, values) tensors as an array indexed by vertex id (`fill` where no rank owns the id); no id
    is owned twice"""
    out = np.full(V, fill, dtype=dtype)
    for v, x in parts:
        out[v.cpu().numpy()] = x.cpu().numpy()
    assert np.unique(np.concatenate([v.cpu().numpy() for v, _ in parts])).size == sum(v.numel() for v, _ in parts)
    return out


def present(s, d, V):
    """the ids that appear in an edge (the vertices of an MGGraph) and the map id -> index among them (-1 elsewhere)"""
    ids = np.unique(np.concatenate([s, d]))
    remap = np.full(V, -1, dtype=np.int64)
    remap[ids] = np.arange(ids.size)
    return ids, remap
