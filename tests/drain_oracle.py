"""CPU restatement of the drain simulation (ks_drain_check, include/ksched.h; DESIGN.md 5f) on the oracle's run_packed.
For each candidate: copy free[], set the nodes that are no destination (its own, and with KS_DRAIN_EXCLUDE_CANDIDATES every
candidate's) to the padding sentinel INT64_MIN, which no request >= 0 fits; then one pod at a time through run_packed,
subtracting each pod where it lands, until the first pod with no node."""
import numpy as np

SENTINEL = np.iinfo(np.int64).min


def drain_packed(orc, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, node_idx, offset, policy=0,
                 exclude=False, which=None):
    """Returns (placed[D], node_idx[P], score[P]); free_cpu / free_mem are not changed.  which: the candidates to evaluate
    (default all); the others keep placed 0 and -1 / 0."""
    N, P, D = len(free_cpu), len(req_cpu), len(node_idx)
    labels = np.ascontiguousarray(labels, np.uint64).reshape(N, -1)
    sel = np.ascontiguousarray(sel, np.uint64).reshape(P, -1)
    req_cpu, req_mem = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
    node_idx = np.asarray(node_idx, np.int64)
    placed = np.zeros(D, np.uint32)
    idx = np.full(P, -1, np.int32)
    score = np.zeros(P, np.int64)
    for d in range(D) if which is None else which:
        fc, fm = np.array(free_cpu, np.int64), np.array(free_mem, np.int64)
        gone = node_idx if exclude else node_idx[d:d + 1]
        fc[gone], fm[gone] = SENTINEL, SENTINEL
        for p in range(int(offset[d]), int(offset[d + 1])):
            i, s, _, _, _ = orc.run_packed(fc, fm, alloc_cpu, alloc_mem, labels, req_cpu[p:p + 1], req_mem[p:p + 1],
                                           sel[p:p + 1], policy, want_mask=False)
            if i[0] < 0:
                break
            idx[p], score[p] = i[0], s[0]
            fc[i[0]] -= req_cpu[p]
            fm[i[0]] -= req_mem[p]
            placed[d] += 1
    return placed, idx, score


def bound_candidates(bound_node, N):
    """Every node a candidate with its bound pods: (order, node_idx, offset), where order lists the bound pods grouped by
    node (bound order kept inside a node) and candidate n owns order[offset[n]:offset[n+1]]."""
    bound_node = np.asarray(bound_node, np.int64)
    real = np.nonzero((bound_node >= 0) & (bound_node < N))[0]  # a pod bound to an unknown node belongs to no candidate
    order = real[np.argsort(bound_node[real], kind="stable")]
    offset = np.searchsorted(bound_node[order], np.arange(N + 1)).astype(np.uint64)
    return order, np.arange(N, dtype=np.int32), offset
