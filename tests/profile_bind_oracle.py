"""CPU restatement of soft constraints when binding (ks_profile_bind, include/ksched.h; DESIGN.md 5o).

profile_bind_packed binds the pods one at a time, as kube-scheduler's default profile runs one cycle per pod:
  - Filter: fit and selector, the hard spread rule against each constrained key's minimum over the group's eligible
    domains (recomputed from the counts at every turn), and rules 1-3 from affinity_bind_oracle.affinity_mask;
  - PodTopologySpread Score as upstream's scoring.go is structured: the ignored set and each key's domains as Python
    sets of label values over the filtered nodes (the missing label counts as a value of its own when the group's
    constraints are system-defaulted), math.log weights, a float sum per node and an explicit half-away-from-zero
    round, then NormalizeScore;
  - InterPodAffinity Score as processExistingPod walks it: every bound pod against the incoming pod's preferred terms
    and against the bound pod's own required-affinity and preferred terms, into a per-(key, value) map, then the
    min-max normalisation over the filtered nodes.
It never uses a compiled counter.  It charges free_cpu / free_mem in place and returns (node_idx [P], score [P],
parts [P, 3], refused [P, 2], counts, soft_counts) as Snapshot.profile_bind does; the counts are lists of K arrays
[G, D_k].  terms: (owner, kind 0-3, key, targets); term_weight: one weight per term (0 for required terms)."""
import math

import numpy as np

from affinity_bind_oracle import AFFINITY, ANTI, affinity_mask
from replicas_oracle import _specs
from spread_oracle import scores_at

PREFERRED, ANTI_PREFERRED = 2, 3


def go_round(x):
    """Go's math.Round: half away from zero."""
    a = abs(x)
    f = math.floor(a)
    r = f + 1 if a - f >= 0.5 else f
    return int(r if x >= 0 else -r)


def pts_scores(F, g, soft_skew, soft_all, dom, sc):
    """PodTopologySpread's score of every node of F (a list of node indices), a dict node -> pts."""
    K = len(dom)
    sigma = [k for k in range(K) if soft_skew[g][k] >= 1] if g >= 0 else []
    if not sigma:
        return {n: 0 for n in F}  # Skip
    require_all = bool(soft_all[g])
    ignored = set()
    values = {k: set() for k in sigma}
    for n in F:
        if require_all and any(dom[k][n] < 0 for k in sigma):
            ignored.add(n)
            continue
        for k in sigma:
            values[k].add(int(dom[k][n]))  # -1 stands for the empty label value
    weight = {k: math.log(float(len(values[k]) + 2)) for k in sigma}
    raw = {}
    for n in F:
        if n in ignored:
            continue
        score = 0.0
        for k in sigma:
            if dom[k][n] >= 0:
                score += float(sc[k][g][dom[k][n]]) * weight[k] + float(soft_skew[g][k] - 1)
        raw[n] = go_round(score)
    lo = min(raw.values()) if raw else None
    hi = 0
    for v in raw.values():
        hi = max(hi, v)
    out = {}
    for n in F:
        if n in ignored:
            out[n] = 0
        elif hi == 0:
            out[n] = 100
        else:
            out[n] = 100 * (hi + lo - raw[n]) // hi  # non-negative: floor is Go's truncation
    return out


def ipa_raw(g, bound, terms, weights, hard_weight, dom):
    """InterPodAffinity's raw score of every node (int64 array [N]) for an incoming pod of group g."""
    N = dom[0].shape[0]
    topo = {}  # (key, value) -> score

    def add(k, m, v):
        if dom[k][m] >= 0:
            topo[k, int(dom[k][m])] = topo.get((k, int(dom[k][m])), 0) + v

    if g >= 0:
        for h, m in bound:
            for t, (owner, kind, k, targets) in enumerate(terms):
                if owner == g and h in targets:  # the incoming pod's preferred terms
                    if kind == PREFERRED:
                        add(k, m, weights[t])
                    elif kind == ANTI_PREFERRED:
                        add(k, m, -weights[t])
                if owner == h and g in targets:  # the bound pod's terms
                    if kind == AFFINITY and hard_weight > 0:
                        add(k, m, hard_weight)
                    elif kind == PREFERRED:
                        add(k, m, weights[t])
                    elif kind == ANTI_PREFERRED:
                        add(k, m, -weights[t])
    raw = np.zeros(N, np.int64)
    for (k, v), s in topo.items():
        raw += np.where(dom[k] == v, s, 0)
    return raw


def profile_bind_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, group, n_groups,
                        keys, terms=(), existing_pods=None, max_skew=None, min_domains=None, existing=None, policy=4,
                        soft_skew=None, soft_all_keys=None, term_weight=None, hard_affinity_weight=1, weight_spread=2,
                        weight_affinity=2):
    fc, fm = free_cpu, free_mem
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    N, P, K, G = fc.shape[0], len(req_cpu), len(keys), int(n_groups)
    labels, sel = _specs(labels, sel, N, P)
    group = np.asarray(group, np.int64).reshape(P)
    dom = [np.asarray(d, np.int64).reshape(N) for d, _ in keys]
    D = [int(n) for _, n in keys]
    skew = np.zeros((G, K), np.int64) if max_skew is None else np.asarray(max_skew, np.int64).reshape(G, K)
    mind = np.zeros((G, K), np.int64) if min_domains is None else np.asarray(min_domains, np.int64).reshape(G, K)
    soft = np.zeros((G, K), np.int64) if soft_skew is None else np.asarray(soft_skew, np.int64).reshape(G, K)
    soft_all = np.ones(G, np.int64) if soft_all_keys is None else np.asarray(soft_all_keys, np.int64).reshape(G)
    terms = [(int(o), int(kd), int(k), {int(t) for t in np.asarray(tg).reshape(-1)}) for o, kd, k, tg in terms]
    weights = [0] * len(terms) if term_weight is None else [int(w) for w in term_weight]
    required = [t for t in terms if t[1] in (AFFINITY, ANTI)]
    bound = [] if existing_pods is None else [(int(h), int(m)) for h, m in zip(*existing_pods)]

    def start():
        return [np.zeros((G, d), np.int64) if existing is None else np.asarray(existing[k], np.int64).reshape(G, d).copy()
                for k, d in enumerate(D)]
    cnt, sc = start(), start()
    # each group's eligible domains per constrained key (selector and every constrained key present)
    elig = {}
    for g in range(G):
        members = np.nonzero(group == g)[0]
        gsel = sel[members[0]] if len(members) else np.zeros(labels.shape[1], np.uint64)
        ok = ((gsel[None, :] & ~labels) == 0).all(axis=1)
        for k in range(K):
            if skew[g, k]:
                ok &= dom[k] >= 0
        for k in range(K):
            if skew[g, k]:
                e = np.zeros(D[k], bool)
                e[dom[k][ok]] = True
                elig[g, k] = e
    node = np.full(P, -1, np.int32)
    score = np.zeros(P, np.int64)
    parts = np.zeros((P, 3), np.int64)
    refused = np.zeros((P, 2), np.uint32)
    for p in range(P):
        rc, rm, g = int(req_cpu[p]), int(req_mem[p]), int(group[p])
        feasible = (rc <= fc) & (rm <= fm) & ((sel[p][None, :] & ~labels) == 0).all(axis=1)
        spread_ok = np.ones(N, bool)
        if g >= 0:
            for k in range(K):
                if not skew[g, k]:
                    continue
                e = elig[g, k]
                m = 0 if not e.any() or e.sum() < mind[g, k] else int(cnt[k][g][e].min())
                d = dom[k]
                spread_ok &= (d >= 0) & (cnt[k][g][np.where(d >= 0, d, 0)] + 1 - m <= skew[g, k])
        passing = affinity_mask(g, bound, required, dom)
        refused[p] = ((feasible & ~spread_ok).sum(), (feasible & spread_ok & ~passing).sum())
        F = np.nonzero(feasible & spread_ok & passing)[0].tolist()
        if not F:
            continue
        policy_score = scores_at(fc, fm, ac, am, rc, rm, np.zeros(N, np.int64), policy)
        pts = pts_scores(F, g, soft, soft_all, dom, sc)
        iraw = ipa_raw(g, bound, terms, weights, hard_affinity_weight, dom)
        lo, hi = min(int(iraw[n]) for n in F), max(int(iraw[n]) for n in F)
        best = None
        for n in F:
            ipa = int(100.0 * (float(int(iraw[n]) - lo) / float(hi - lo))) if hi > lo else 0
            total = int(policy_score[n]) + weight_spread * pts[n] + weight_affinity * ipa
            if best is None or total > best[0]:  # ascending n: ties to the lower index
                best = (total, n, int(policy_score[n]), pts[n], ipa)
        total, n = best[0], best[1]
        node[p], score[p], parts[p] = n, total, best[2:]
        fc[n] -= rc
        fm[n] -= rm
        if g < 0:
            continue
        for k in range(K):
            if skew[g, k]:
                cnt[k][g][dom[k][n]] += 1
        sigma = [k for k in range(K) if soft[g, k] >= 1]
        if sigma and (not soft_all[g] or all(dom[k][n] >= 0 for k in sigma)):
            for k in sigma:
                if dom[k][n] >= 0:
                    sc[k][g][dom[k][n]] += 1
        bound.append((g, n))
    return (node, score, parts, refused, [c.astype(np.uint32) for c in cnt], [c.astype(np.uint32) for c in sc])
