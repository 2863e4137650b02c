"""CPU restatement of pod groups (ks_gang_bind, include/ksched.h; DESIGN.md 5e) on the oracle's own streaming entry point:
for each group in order, orc_stream_bind_packed runs on copies of free[]; the copies replace free[] only when the group
placed at least min_member pods, else every pod of the group gets -1 / 0 and free[] stays as it was."""
import numpy as np


def gang_bind_packed(orc, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, offset, min_member,
                     policy=0):
    """In place on free_cpu / free_mem (int64); returns (node_idx[P], score[P], placed[G], rounds[G])."""
    N, P, G = free_cpu.shape[0], len(req_cpu), len(offset) - 1
    labels = np.ascontiguousarray(labels, np.uint64).reshape(N, -1)
    sel = np.ascontiguousarray(sel, np.uint64).reshape(P, -1)
    req_cpu, req_mem = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
    idx = np.full(P, -1, np.int32)
    score = np.zeros(P, np.int64)
    placed = np.zeros(G, np.uint32)
    rounds = np.zeros(G, np.uint32)
    for g in range(G):
        a, b = int(offset[g]), int(offset[g + 1])
        if N == 0:  # no node: the stream loop's one round in which no pod has a feasible node
            rounds[g] = 1
            continue
        fc, fm = free_cpu.copy(), free_mem.copy()
        i, s, r = orc.stream_bind_packed(fc, fm, alloc_cpu, alloc_mem, labels, req_cpu[a:b], req_mem[a:b], sel[a:b],
                                         policy)
        placed[g], rounds[g] = int((i >= 0).sum()), r
        if placed[g] >= int(min_member[g]):
            idx[a:b], score[a:b] = i, s
            free_cpu[:], free_mem[:] = fc, fm
    return idx, score, placed, rounds


def sequential_packed(orc, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, policy=0):
    """One pod at a time, each seeing the binds of all earlier pods (the reference's reconcile order, argmax select)."""
    P = len(req_cpu)
    sel = np.ascontiguousarray(sel, np.uint64).reshape(P, -1)
    idx = np.full(P, -1, np.int32)
    score = np.zeros(P, np.int64)
    for p in range(P):
        i, s, _, _, _ = orc.run_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu[p:p + 1],
                                       req_mem[p:p + 1], sel[p:p + 1], policy, want_mask=False)
        if i[0] >= 0:
            idx[p], score[p] = i[0], s[0]
            free_cpu[i[0]] -= req_cpu[p]
            free_mem[i[0]] -= req_mem[p]
    return idx, score


def groups(rng, P, lo=1, hi=1024):
    """Random group offsets over P pods, sizes in [lo, hi] (the last group takes what is left, at least 1)."""
    off = [0]
    while off[-1] < P:
        off.append(min(P, off[-1] + int(rng.integers(lo, hi + 1))))
    return np.array(off, np.uint64)
