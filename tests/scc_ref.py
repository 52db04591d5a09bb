"""The CPU reference for strongly connected components (tests/test_scc_{cpu,gpu}.py, scripts/scc_bench.py's checks): the
reference test's Tarjan restated in numpy/Python."""
import numpy as np


def scc(src, dst, num_vertices):
    """component index per vertex of the directed graph src -> dst: strongly_connected_components_reference
    (cpp/tests/components/strongly_connected_components_test.cpp:32-93, Tarjan's algorithm) with an explicit stack instead of
    recursion.  Components are numbered 0, 1, ... in the order Tarjan completes them (sinks first)."""
    src = np.asarray(src, dtype=np.int64)
    dst = np.asarray(dst, dtype=np.int64)
    order = np.argsort(src, kind="stable")
    offsets = np.zeros(num_vertices + 1, dtype=np.int64)
    np.cumsum(np.bincount(src, minlength=num_vertices), out=offsets[1:])
    offsets, indices = offsets.tolist(), dst[order].tolist()
    unset = -1
    index = [unset] * num_vertices
    lowlink = [0] * num_vertices
    on_stack = [False] * num_vertices
    comp = np.full(num_vertices, -1, dtype=np.int64)
    stack, next_index, next_comp = [], 0, 0
    for root in range(num_vertices):
        if index[root] != unset:
            continue
        # call frames (v, next edge of v to consider)
        frames = [(root, offsets[root])]
        index[root] = lowlink[root] = next_index
        next_index += 1
        stack.append(root)
        on_stack[root] = True
        while frames:
            v, e = frames[-1]
            if e < offsets[v + 1]:
                frames[-1] = (v, e + 1)
                w = indices[e]
                if index[w] == unset:   # strongconnect(w)
                    index[w] = lowlink[w] = next_index
                    next_index += 1
                    stack.append(w)
                    on_stack[w] = True
                    frames.append((w, offsets[w]))
                elif on_stack[w]:
                    lowlink[v] = min(lowlink[v], index[w])
                continue
            frames.pop()
            if lowlink[v] == index[v]:  # v is a root: pop its component
                while True:
                    w = stack.pop()
                    on_stack[w] = False
                    comp[w] = next_comp
                    if w == v:
                        break
                next_comp += 1
            if frames:                  # back in the caller: lowlink[u] = min(lowlink[u], lowlink[v])
                u = frames[-1][0]
                lowlink[u] = min(lowlink[u], lowlink[v])
    return comp
