"""CPU restatement of KS_SCORE_MOST_ALLOCATED (include/ksched.h) for the tests.

The oracle library scores LEFTOVER and LEAST_ALLOCATED only, so this module adds the bin-packing policy on top of it:
which cells are feasible (and the mask and counts) still come from orc_run_packed's cell codes, and the scores from the
definition below.  `Oracle(orc)` has orc's run_packed / stream_bind_packed / commit_claims / free_reduce and accepts
policy 3, so the existing restatements (gang_oracle, drain_oracle, replicas_oracle.sequential_packed) run under it
unchanged.  `prefix_fill_packed` is the replica plan as the library computes it under this policy: nodes filled whole,
one after another, in order of copy 0's score descending, node ascending."""
import numpy as np

from replicas_oracle import PLAN_DTYPE, _row, _specs, node_copies

MOST_ALLOCATED = 3


def term(f, a, q):
    """One resource, Python integers: clamp(A - (f - q), 0, A) * 100 / A, 0 for A <= 0."""
    if a <= 0:
        return 0
    return min(max(a - (f - q), 0), a) * 100 // a


def score(fc, fm, ac, am, rc, rm):
    return (term(int(fc), int(ac), int(rc)) + term(int(fm), int(am), int(rm))) // 2


def scores(fc, fm, ac, am, rc, rm):
    """The same on int64 arrays (broadcasting); inside the limits of ksched.h nothing overflows."""
    def t(f, a, q):
        pos = a > 0
        u = np.clip(a - (f - q), 0, np.where(pos, a, 0))
        return np.where(pos, (u * 100) // np.where(pos, a, 1), 0)
    return (t(fc, ac, rc) + t(fm, am, rm)) // 2


class Oracle:
    """orc with policy 3 added to run_packed and stream_bind_packed."""

    def __init__(self, orc):
        self.orc = orc

    def __getattr__(self, name):
        return getattr(self.orc, name)

    def run_packed(self, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, policy=0,
                   want_mask=True, want_codes=False, nthreads=0):
        if policy != MOST_ALLOCATED:
            return self.orc.run_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, policy,
                                       want_mask, want_codes, nthreads)
        _, _, cnt, mask, codes = self.orc.run_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem,
                                                     sel, 0, want_mask, True, nthreads)
        fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
        ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
        rc, rm = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
        P = rc.shape[0]
        idx = np.full(P, -1, np.int32)
        sc = np.zeros(P, np.int64)
        if P and fc.shape[0]:
            s = scores(fc[None, :], fm[None, :], ac[None, :], am[None, :], rc[:, None], rm[:, None])
            s = np.where(codes == 0, s, -1)  # every feasible score is >= 0
            best = s.argmax(axis=1)  # first maximum: ties to the lowest node index
            ok = s[np.arange(P), best] >= 0
            idx[ok] = best[ok]
            sc[ok] = s[np.arange(P), best][ok]
        return idx, sc, cnt, mask, codes if want_codes else None

    def stream_bind_packed(self, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, policy=0):
        """orc_stream_bind_packed's round loop: select the pending pods, commit the claims per node in arrival order,
        losers retry; in place on free_cpu / free_mem."""
        if policy != MOST_ALLOCATED:
            return self.orc.stream_bind_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel,
                                               policy)
        P = len(req_cpu)
        rc, rm = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
        sel = np.ascontiguousarray(sel, np.uint64).reshape(P, -1)
        idx = np.full(P, -1, np.int32)
        sc = np.zeros(P, np.int64)
        pending = np.arange(P)
        rounds = 0
        while len(pending) and rounds <= P + 1:
            i, s = self.run_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, rc[pending], rm[pending],
                                   sel[pending], policy, want_mask=False)[:2]
            acc = self.orc.commit_claims(free_cpu, free_mem, i, rc[pending], rm[pending])
            won = (i >= 0) & (acc != 0)
            idx[pending[won]], sc[pending[won]] = i[won], s[won]
            pending = pending[(i >= 0) & (acc == 0)]
            rounds += 1
        return idx, sc, rounds


def topk_packed(oracle, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, k):
    """ks_select_topk's rows under policy 3: feasible nodes by score descending, node ascending."""
    from topk_oracle import _ranked
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    rc, rm = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
    codes = oracle.orc.run_packed(fc, fm, ac, am, labels, rc, rm, sel, 0, want_mask=False, want_codes=True)[4]
    rows = []
    for p in range(len(rc)):
        n = np.nonzero(codes[p] == 0)[0]
        rows.append((n, scores(fc[n], fm[n], ac[n], am[n], rc[p], rm[p])))
    return _ranked(rows, k)


def prefix_fill_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, replicas):
    """Replica placement under policy 3 without one select per copy: s_n(j) is non-decreasing in j, so the node being
    filled never loses to one not yet touched; nodes take up to c_n copies each, in order of s_n(0) descending, node
    ascending.  Returns (rows, node, score, offset) as replicas_oracle.merge_packed does."""
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    N, T = fc.shape[0], len(req_cpu)
    labels, sel = _specs(labels, sel, N, T)
    offset = np.zeros(T + 1, np.uint64)
    np.cumsum(np.asarray(replicas, np.uint64), out=offset[1:])
    rows = np.zeros(T, PLAN_DTYPE)
    node = np.full(int(offset[-1]), -1, np.int32)
    sc = np.zeros(int(offset[-1]), np.int64)
    for t in range(T):
        rc, rm, R, o = int(req_cpu[t]), int(req_mem[t]), int(replicas[t]), int(offset[t])
        c, cap = node_copies(fc, fm, labels, rc, rm, sel[t])
        feas = np.nonzero(c != 0)[0]
        s0 = scores(fc[feas], fm[feas], ac[feas], am[feas], rc, rm)
        order = feas[np.lexsort((feas, -s0))]
        cn = np.where(c[order] < 0, R, np.minimum(c[order], R))
        take = np.clip(R - (np.cumsum(cn) - cn), 0, cn)  # each node in turn takes what it holds of what is left
        r = int(take.sum())
        n_of = np.repeat(order, take)
        j = np.arange(r, dtype=np.int64) - np.repeat(np.cumsum(take) - take, take)
        node[o:o + r] = n_of
        sc[o:o + r] = scores(fc[n_of] - j * rc, fm[n_of] - j * rm, ac[n_of], am[n_of], rc, rm)
        rows[t] = _row(cap, len(feas), node[o:o + r], int(sc[o + r - 1]) if r else 0)
    return rows, node, sc, offset
