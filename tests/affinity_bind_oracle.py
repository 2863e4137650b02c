"""CPU restatement of inter-pod affinity when binding (ks_affinity_bind, include/ksched.h; DESIGN.md 5n).

affinity_bind_packed binds the pods one at a time.  Rules 1-3 are restated per term, as upstream InterPodAffinity's
Filter states them: for each pod it walks the bound pods (the existing ones, then every earlier pod of the queue) and
their terms, never a compiled counter.  The spread half is spread_bind_oracle.spread_bind_packed itself, called on a
one-pod queue whose existing counts are the counts so far: once with every node and once with the nodes rules 1-3
refuse made unfit, so the first call gives the spread refusals and the second the binding.  It charges free_cpu /
free_mem in place and returns (node_idx [P], score [P], refused [P, 2], counts) as Snapshot.affinity_bind does.

terms: a list of (owner, kind, key, targets); existing_pods: None or (groups, nodes)."""
import numpy as np

from spread_bind_oracle import spread_bind_packed

AFFINITY, ANTI = 0, 1


def affinity_mask(g, bound, terms, dom):
    """The nodes that pass rules 1-3 for a pod of group g, with bound a list of (group, node) and dom the K
    node_domain arrays."""
    N = dom[0].shape[0]
    ok = np.ones(N, bool)
    if g < 0:
        return ok
    by_owner = {}
    for t in terms:
        by_owner.setdefault(t[0], []).append(t)
    # 1. incoming anti-affinity: a bound pod of a target group in the node's domain of the term's key
    for owner, kind, k, targets in by_owner.get(g, ()):
        if kind != ANTI:
            continue
        for h, m in bound:
            if h in targets and dom[k][m] >= 0:
                ok &= dom[k] != dom[k][m]
    # 2. existing pods' anti-affinity: a bound pod whose anti term targets g, in the node's domain of that key
    for h, m in bound:
        for owner, kind, k, targets in by_owner.get(h, ()):
            if kind == ANTI and g in targets and dom[k][m] >= 0:
                ok &= dom[k] != dom[k][m]
    # 3. affinity: every key present; some bound pod matching every term in the node's domain of each term's key, or
    # the first-pod rule
    aff = [(k, targets) for owner, kind, k, targets in by_owner.get(g, ()) if kind == AFFINITY]
    if not aff:
        return ok
    matching = [m for h, m in bound if all(h in targets for _, targets in aff)]
    has_keys = np.ones(N, bool)
    exist = np.ones(N, bool)
    counts_empty = True
    for k, _ in aff:
        has_keys &= dom[k] >= 0
        here = {int(dom[k][m]) for m in matching if dom[k][m] >= 0}
        counts_empty &= not here
        exist &= np.isin(dom[k], list(here)) & (dom[k] >= 0)
    self_match = all(g in targets for _, targets in aff)
    return ok & has_keys & (exist | (counts_empty and self_match))


def affinity_bind_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, group, n_groups,
                         keys, terms=(), existing_pods=None, max_skew=None, min_domains=None, existing=None, policy=0):
    fc, fm = free_cpu, free_mem
    N, P, K, G = fc.shape[0], len(req_cpu), len(keys), int(n_groups)
    W = np.asarray(labels, np.uint64).reshape(N, -1).shape[1] if N else 1
    sel = np.asarray(sel, np.uint64).reshape(P, W if not P else -1)
    group = np.asarray(group, np.int64).reshape(P)
    dom = [np.asarray(d, np.int64).reshape(N) for d, _ in keys]
    D = [int(n) for _, n in keys]
    skew = np.zeros((G, K), np.int64) if max_skew is None else np.asarray(max_skew, np.int64).reshape(G, K)
    terms = [(int(o), int(kd), int(k), {int(t) for t in np.asarray(tg).reshape(-1)}) for o, kd, k, tg in terms]
    bound = [] if existing_pods is None else [(int(h), int(m)) for h, m in zip(*existing_pods)]
    cnt = [np.zeros((G, d), np.int64) if existing is None else np.asarray(existing[k], np.int64).reshape(G, d).copy()
           for k, d in enumerate(D)]
    node = np.full(P, -1, np.int32)
    score = np.zeros(P, np.int64)
    refused = np.zeros((P, 2), np.uint32)
    for p in range(P):
        g = int(group[p])
        q = dict(req_cpu=np.asarray(req_cpu, np.int64)[p:p + 1], req_mem=np.asarray(req_mem, np.int64)[p:p + 1],
                 sel=sel[p:p + 1], group=[g], keys=keys, max_skew=skew, min_domains=min_domains, policy=policy)
        feasible = int(((q["req_cpu"][0] <= fc) & (q["req_mem"][0] <= fm) &
                        ((sel[p][None, :] & ~np.asarray(labels, np.uint64).reshape(N, W)) == 0).all(axis=1)).sum())
        # spread alone: its refusals and candidate count
        _, _, spread_ref, _ = spread_bind_packed(fc.copy(), fm.copy(), alloc_cpu, alloc_mem, labels, existing=cnt, **q)
        passing = affinity_mask(g, bound, terms, dom)
        # spread among the nodes rules 1-3 pass: the binding
        gfc, gfm = np.where(passing, fc, -1), np.where(passing, fm, -1)
        n, s, ref2, cnt2 = spread_bind_packed(gfc, gfm, alloc_cpu, alloc_mem, labels, existing=cnt, **q)
        fit_pass = int((passing & (q["req_cpu"][0] <= fc) & (q["req_mem"][0] <= fm) &
                        ((sel[p][None, :] & ~np.asarray(labels, np.uint64).reshape(N, W)) == 0).all(axis=1)).sum())
        refused[p] = (spread_ref[0], (feasible - int(spread_ref[0])) - (fit_pass - int(ref2[0])))
        if n[0] < 0:
            continue
        node[p], score[p] = n[0], s[0]
        fc[n[0]] -= q["req_cpu"][0]
        fm[n[0]] -= q["req_mem"][0]
        cnt = [c.astype(np.int64) for c in cnt2]
        if g >= 0:
            bound.append((g, int(n[0])))
    counts = [c.astype(np.uint32) for c in cnt]
    return node, score, refused, counts
