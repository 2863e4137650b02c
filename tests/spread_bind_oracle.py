"""CPU restatement of topology spread when binding (ks_spread_bind, include/ksched.h; DESIGN.md 5m).

spread_bind_packed binds the pods one at a time in numpy, exactly as the header defines it: each group's eligible
domains, counts and minima per constrained key, then per pod the fit, selector and skew rules against the free[] and
counts every earlier pod left, the score from spread_oracle.scores_at with no earlier copy (ks_select's score), ties to
the lower node.  It charges free_cpu / free_mem in place and returns (node_idx [P], score [P], refused [P], counts) as
Snapshot.spread_bind does, counts a list of K arrays [G, D_k]."""
import numpy as np

from replicas_oracle import _specs
from spread_oracle import INT64_MIN, scores_at


def spread_bind_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, group, keys, max_skew,
                       min_domains=None, existing=None, policy=0):
    fc, fm = free_cpu, free_mem  # int64 arrays, charged in place
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    N, P, K = fc.shape[0], len(req_cpu), len(keys)
    labels, sel = _specs(labels, sel, N, P)
    group = np.asarray(group, np.int64).reshape(P)
    dom = [np.asarray(d, np.int64).reshape(N) for d, _ in keys]
    dn = [np.where(d >= 0, d, 0) for d in dom]
    D = [int(n) for _, n in keys]
    skew = np.asarray(max_skew, np.int64).reshape(-1, K)
    G = skew.shape[0]
    mind = np.zeros((G, K), np.int64) if min_domains is None else np.asarray(min_domains, np.int64).reshape(G, K)
    cnt = [[np.zeros(d, np.int64) if existing is None else np.asarray(existing[k], np.int64).reshape(G, d)[g].copy()
            for k, d in enumerate(D)] for g in range(G)]
    # 1. group state: eligible nodes and domains, each constrained key's minimum (0 under minDomains)
    in_e = [[None] * K for _ in range(G)]
    forced = np.zeros((G, K), bool)
    m = np.zeros((G, K), np.int64)
    for g in range(G):
        members = np.nonzero(group == g)[0]
        gsel = sel[members[0]] if len(members) else np.zeros(labels.shape[1], np.uint64)
        eligible = ((gsel[None, :] & ~labels) == 0).all(axis=1)
        for k in range(K):
            if skew[g, k]:
                eligible &= dom[k] >= 0
        for k in range(K):
            if not skew[g, k]:
                continue
            e = np.zeros(D[k], bool)
            e[dom[k][eligible]] = True
            in_e[g][k] = e
            forced[g, k] = int(e.sum()) < mind[g, k]
            m[g, k] = 0 if not e.any() or forced[g, k] else int(cnt[g][k][e].min())
    node = np.full(P, -1, np.int32)
    score = np.zeros(P, np.int64)
    refused = np.zeros(P, np.uint32)
    # 2. one pod at a time
    for p in range(P):
        rc, rm, g = int(req_cpu[p]), int(req_mem[p]), int(group[p])
        feasible = (rc <= fc) & (rm <= fm) & ((sel[p][None, :] & ~labels) == 0).all(axis=1)
        cand = feasible.copy()
        if g >= 0:
            for k in range(K):
                if skew[g, k]:
                    cand &= (dom[k] >= 0) & (cnt[g][k] + 1 - m[g, k] <= skew[g, k])[dn[k]]
        refused[p] = int(feasible.sum() - cand.sum())
        if not cand.any():
            continue
        s = np.where(cand, scores_at(fc, fm, ac, am, rc, rm, np.zeros(N, np.int64), policy), INT64_MIN)
        n = int(s.argmax())  # first maximum: ties to the lower node index
        node[p], score[p] = n, s[n]
        fc[n] -= rc
        fm[n] -= rm
        if g >= 0:
            for k in range(K):
                if skew[g, k]:
                    cnt[g][k][dom[k][n]] += 1
                    if not forced[g, k]:
                        m[g, k] = int(cnt[g][k][in_e[g][k]].min())
    # 3. the counts: the final ones for the constrained keys, existing (or 0) for the others
    counts = [np.array([cnt[g][k] for g in range(G)], np.uint32).reshape(G, D[k]) for k in range(K)]
    return node, score, refused, counts


def skew_ok_at_each_turn(labels, sel, group, keys, max_skew, node, existing=None):
    """Replays the bindings of one call (no minDomains) and checks, at each placed pod's turn, its group's skew rule for
    every constrained key: the chosen domain's count before the pod is below m + max_skew, m over the group's eligible
    domains.  Returns the first failing pod, or None."""
    labels = np.asarray(labels, np.uint64).reshape(len(keys[0][0]), -1)
    sel = np.asarray(sel, np.uint64).reshape(len(group), -1)
    skew = np.asarray(max_skew, np.int64).reshape(-1, len(keys))
    G = skew.shape[0]
    cnt = {}
    elig = {}
    for g in range(G):
        members = np.nonzero(np.asarray(group) == g)[0]
        if not len(members):
            continue
        ok = ((sel[members[0]][None, :] & ~labels) == 0).all(axis=1)
        for k, (d, _) in enumerate(keys):
            if skew[g, k]:
                ok &= np.asarray(d) >= 0
        for k, (d, nd) in enumerate(keys):
            e = np.zeros(nd, bool)
            e[np.asarray(d)[ok]] = True
            elig[g, k] = e
            cnt[g, k] = np.zeros(nd, np.int64) if existing is None else np.asarray(existing[k], np.int64)[g].copy()
    for p, n in enumerate(node):
        g = int(group[p])
        if n < 0 or g < 0:
            continue
        for k, (d, _) in enumerate(keys):
            if not skew[g, k]:
                continue
            c, dk = cnt[g, k], int(np.asarray(d)[n])
            if dk < 0 or c[dk] + 1 - c[elig[g, k]].min() > skew[g, k]:
                return p
            c[dk] += 1
    return None
