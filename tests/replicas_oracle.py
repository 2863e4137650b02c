"""CPU restatements of replica placement (ks_place_replicas, include/ksched.h; DESIGN.md 5h).

sequential_packed: every copy of a spec through gang_oracle.sequential_packed, that is the oracle's own select run one
copy at a time with the earlier copies charged to a private copy of free[].
merge_packed: per node, the copies it takes on its own and their score sequence, all (node, copy) pairs sorted by
(score descending, node, copy) and the first `replicas` of them taken.
Both return (rows, node, score, offset) as Snapshot.place_replicas does."""
import numpy as np

from gang_oracle import sequential_packed as _sequential

U64_MAX = (1 << 64) - 1
PLAN_DTYPE = np.dtype([("capacity", np.uint64), ("placed", np.uint32), ("nodes", np.uint32),
                       ("feasible_cnt", np.uint32), ("max_per_node", np.uint32), ("last_score", np.int64)])


def _specs(labels, sel, N, T):
    labels = np.ascontiguousarray(labels, np.uint64).reshape(N, -1) if N else np.zeros((0, 1), np.uint64)
    sel = np.ascontiguousarray(sel, np.uint64).reshape(T, -1) if T else np.zeros((0, labels.shape[1]), np.uint64)
    return labels, sel


def node_copies(free_cpu, free_mem, labels, rc, rm, sel_row):
    """c_n for every node (int64, -1 = unbounded) and the saturating capacity as a Python int."""
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    ok = (rc <= fc) & (rm <= fm) & ((np.asarray(sel_row, np.uint64)[None, :] & ~labels) == 0).all(axis=1)
    c = np.zeros(fc.shape[0], np.int64)
    if rc == 0 and rm == 0:
        c[ok] = -1
    else:
        big = np.full_like(fc, 1 << 62)
        cc = fc // rc if rc > 0 else big
        cm = fm // rm if rm > 0 else big
        c = np.where(ok, np.minimum(cc, cm), 0)
    cap = U64_MAX if (c < 0).any() else min(U64_MAX, sum(int(x) for x in c[c > 0].tolist()))
    return c, cap


def copy_scores(fc, fm, ac, am, rc, rm, j, policy):
    """s_n(j) for arrays of node values and copy indices (free after the copy is >= 0, so floors are truncations)."""
    left_c, left_m = fc - (j + 1) * rc, fm - (j + 1) * rm
    if policy == 0:
        return (left_c << 22) + left_m
    pc = np.where(ac > 0, (left_c * 100) // np.where(ac > 0, ac, 1), 0)
    pm = np.where(am > 0, (left_m * 100) // np.where(am > 0, am, 1), 0)
    return (pc + pm) // 2


def _row(cap, feas, nodes_of_copies, last):
    r = np.zeros((), PLAN_DTYPE)
    r["capacity"], r["placed"], r["feasible_cnt"] = cap, len(nodes_of_copies), feas
    if len(nodes_of_copies):
        _, per = np.unique(nodes_of_copies, return_counts=True)
        r["nodes"], r["max_per_node"], r["last_score"] = len(per), per.max(), last
    return r


def merge_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, replicas, policy=0):
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    N, T = fc.shape[0], len(req_cpu)
    labels, sel = _specs(labels, sel, N, T)
    offset = np.zeros(T + 1, np.uint64)
    np.cumsum(np.asarray(replicas, np.uint64), out=offset[1:])
    rows = np.zeros(T, PLAN_DTYPE)
    node = np.full(int(offset[-1]), -1, np.int32)
    score = np.zeros(int(offset[-1]), np.int64)
    for t in range(T):
        rc, rm, R = int(req_cpu[t]), int(req_mem[t]), int(replicas[t])
        c, cap = node_copies(fc, fm, labels, rc, rm, sel[t])
        k = np.where(c < 0, R, np.minimum(c, R))
        nodes = np.nonzero(k)[0]
        kk = k[nodes]
        n_of = np.repeat(nodes, kk)
        j = np.arange(n_of.shape[0], dtype=np.int64) - np.repeat(np.cumsum(kk) - kk, kk)
        s = copy_scores(fc[n_of], fm[n_of], ac[n_of], am[n_of], rc, rm, j, policy)
        order = np.lexsort((j, n_of, -s))[:R]
        o = int(offset[t])
        node[o:o + len(order)], score[o:o + len(order)] = n_of[order], s[order]
        rows[t] = _row(cap, int((c != 0).sum()), n_of[order], int(s[order[-1]]) if len(order) else 0)
    return rows, node, score, offset


def sequential_packed(orc, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, replicas, policy=0):
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    N, T = fc.shape[0], len(req_cpu)
    labels, sel = _specs(labels, sel, N, T)
    offset = np.zeros(T + 1, np.uint64)
    np.cumsum(np.asarray(replicas, np.uint64), out=offset[1:])
    rows = np.zeros(T, PLAN_DTYPE)
    node = np.full(int(offset[-1]), -1, np.int32)
    score = np.zeros(int(offset[-1]), np.int64)
    for t in range(T):
        R, o = int(replicas[t]), int(offset[t])
        _, cap = node_copies(fc, fm, labels, int(req_cpu[t]), int(req_mem[t]), sel[t])
        feas = 0
        if N:
            feas = int(orc.run_packed(fc, fm, alloc_cpu, alloc_mem, labels, np.asarray(req_cpu[t:t + 1], np.int64),
                                      np.asarray(req_mem[t:t + 1], np.int64), sel[t:t + 1], policy, want_mask=False)[2][0])
        if R and N:
            i, s = _sequential(orc, fc.copy(), fm.copy(), alloc_cpu, alloc_mem, labels,
                               np.full(R, req_cpu[t], np.int64), np.full(R, req_mem[t], np.int64),
                               np.repeat(sel[t:t + 1], R, axis=0), policy)
            node[o:o + R], score[o:o + R] = i, s
        placed = node[o:o + R][node[o:o + R] >= 0]
        rows[t] = _row(cap, feas, placed, int(score[o + len(placed) - 1]) if len(placed) else 0)
    return rows, node, score, offset
