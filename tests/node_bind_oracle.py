"""CPU restatement of taints and node affinity when binding (ks_node_bind, include/ksched.h; DESIGN.md 5p).

The two plugins are restated over strings, the way upstream structures them:
  - taints and tolerations as dicts, with upstream's ToleratesTaint; the filter looks for an untolerated NoSchedule or
    NoExecute taint, the score counts the PreferNoSchedule taints that the tolerations with an empty or
    PreferNoSchedule effect do not tolerate;
  - node-affinity requirements evaluated against each node's label map (In, NotIn, Exists, DoesNotExist, Gt, Lt), terms
    ORed for the required affinity, weights summed for the preferred one;
  - DefaultNormalizeScore(100, reverse) over each pod's filtered nodes.
node_bind_packed binds the pods one at a time as profile_bind_oracle.profile_bind_packed does, with these filters
ahead of the hard spread rule, spread eligibility honouring the required node affinity, and both scores in the total.
compile_rules turns the same strings into the numbered masks and domain sets Snapshot.node_bind takes; it never feeds
node_bind_packed, so the device is checked against an evaluation that does not go through it.
group_rules[g]: {"tolerations": [...], "required": [term, ...] or None, "preferred": [(weight, term), ...]}, a term a
list of {"key", "operator", "values"}."""
import numpy as np

from affinity_bind_oracle import AFFINITY, ANTI, affinity_mask
from profile_bind_oracle import ipa_raw, pts_scores
from replicas_oracle import _specs
from spread_oracle import scores_at

HARD_EFFECTS = ("NoSchedule", "NoExecute")
SOFT = "PreferNoSchedule"


def tolerates(tol, taint):
    """Upstream's Toleration.ToleratesTaint."""
    if tol.get("effect", "") and tol["effect"] != taint["effect"]:
        return False
    if tol.get("key", "") and tol["key"] != taint["key"]:
        return False
    op = tol.get("operator", "")
    if op in ("", "Equal"):
        return tol.get("value", "") == taint.get("value", "")
    return op == "Exists"


def untolerated_hard(taints, tols):
    return any(t["effect"] in HARD_EFFECTS and not any(tolerates(x, t) for x in tols) for t in taints)


def intolerable_soft(taints, tols):
    soft = [x for x in tols if x.get("effect", "") in ("", SOFT)]
    return sum(1 for t in taints if t["effect"] == SOFT and not any(tolerates(x, t) for x in soft))


def _int64(s):
    try:
        v = int(s, 10)
    except (TypeError, ValueError):
        return None
    return v if -(1 << 63) <= v < (1 << 63) and s.strip() == s and "_" not in s else None


def requirement_matches(req, labels):
    key, op, values = req["key"], req["operator"], list(req.get("values", ()))
    has = key in labels
    if op == "In":
        return has and labels[key] in values
    if op == "NotIn":
        return not has or labels[key] not in values
    if op == "Exists":
        return has
    if op == "DoesNotExist":
        return not has
    if op in ("Gt", "Lt"):
        if not has:
            return False
        a, b = _int64(labels[key]), _int64(values[0])
        if a is None or b is None:
            return False
        return a > b if op == "Gt" else a < b
    raise ValueError(op)


def term_matches(term, labels):
    return len(term) > 0 and all(requirement_matches(r, labels) for r in term)


def required_ok(rule, labels):
    req = rule.get("required") if rule else None
    return not req or any(term_matches(t, labels) for t in req)  # no term list: no required affinity


def preferred_raw(rule, labels):
    return sum(w for w, t in (rule.get("preferred", ()) if rule else ()) if term_matches(t, labels))


def normalize(raw, reverse):
    """Upstream DefaultNormalizeScore(100, reverse) over a dict node -> raw."""
    mx = max(list(raw.values()) + [0])
    if mx == 0:
        return {n: 100 if reverse else 0 for n in raw}
    return {n: 100 - 100 * v // mx if reverse else 100 * v // mx for n, v in raw.items()}


def node_bind_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, group, n_groups, keys,
                     node_labels, node_taints, group_rules, terms=(), existing_pods=None, max_skew=None,
                     min_domains=None, existing=None, policy=4, soft_skew=None, soft_all_keys=None, term_weight=None,
                     hard_affinity_weight=1, weight_spread=2, weight_affinity=2, weight_taint=3,
                     weight_node_affinity=2):
    """Returns (node_idx [P], score [P], parts [P, 5], refused [P, 4], counts, soft_counts) as Snapshot.node_bind."""
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
    rule = [group_rules[g] if g < len(group_rules) else {} for g in range(G)]

    def rule_of(g):
        return rule[g] if g >= 0 else {}
    taint_ok = {g: np.array([not untolerated_hard(node_taints[n], rule_of(g).get("tolerations", ()))
                             for n in range(N)], bool) for g in range(-1, G)}
    aff_ok = {g: np.array([required_ok(rule_of(g), node_labels[n]) for n in range(N)], bool) for g in range(-1, G)}

    def start():
        return [np.zeros((G, d), np.int64) if existing is None else np.asarray(existing[k], np.int64).reshape(G, d).copy()
                for k, d in enumerate(D)]
    cnt, sc = start(), start()
    # eligible domains: selector, required node affinity (Honor) and every constrained key; taints ignored
    elig = {}
    for g in range(G):
        members = np.nonzero(group == g)[0]
        gsel = sel[members[0]] if len(members) else np.zeros(labels.shape[1], np.uint64)
        ok = ((gsel[None, :] & ~labels) == 0).all(axis=1) & aff_ok[g]
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
    parts = np.zeros((P, 5), np.int64)
    refused = np.zeros((P, 4), np.uint32)
    for p in range(P):
        rc, rm, g = int(req_cpu[p]), int(req_mem[p]), int(group[p])
        feasible = (rc <= fc) & (rm <= fm) & ((sel[p][None, :] & ~labels) == 0).all(axis=1)
        tol = feasible & taint_ok[g]
        nodeaff = tol & aff_ok[g]
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
        refused[p] = ((feasible & ~taint_ok[g]).sum(), (tol & ~aff_ok[g]).sum(), (nodeaff & ~spread_ok).sum(),
                      (nodeaff & spread_ok & ~passing).sum())
        F = np.nonzero(nodeaff & spread_ok & passing)[0].tolist()
        if not F:
            continue
        policy_score = scores_at(fc, fm, ac, am, rc, rm, np.zeros(N, np.int64), policy)
        pts = pts_scores(F, g, soft, soft_all, dom, sc)
        iraw = ipa_raw(g, bound, terms, weights, hard_affinity_weight, dom)
        lo, hi = min(int(iraw[n]) for n in F), max(int(iraw[n]) for n in F)
        tols = rule_of(g).get("tolerations", ())
        tt = normalize({n: intolerable_soft(node_taints[n], tols) for n in F}, True)
        na = normalize({n: preferred_raw(rule_of(g), node_labels[n]) for n in F}, False)
        best = None
        for n in F:
            ipa = int(100.0 * (float(int(iraw[n]) - lo) / float(hi - lo))) if hi > lo else 0
            total = (int(policy_score[n]) + weight_spread * pts[n] + weight_affinity * ipa + weight_taint * tt[n] +
                     weight_node_affinity * na[n])
            if best is None or total > best[0]:  # ascending n: ties to the lower index
                best = (total, n, int(policy_score[n]), pts[n], ipa, tt[n], na[n])
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


def expr_set(req, values, D):
    """The domain set of one requirement over a key whose domains carry `values` (index = domain), bit D = absent."""
    op, vals = req["operator"], list(req.get("values", ()))
    members = [d for d, v in enumerate(values) if requirement_matches(req, {req["key"]: v})]
    if op in ("NotIn", "DoesNotExist"):
        members.append(D)
    words = np.zeros((D + 64) // 64, np.uint64)
    for i in members:
        words[i // 64] |= np.uint64(1 << (i % 64))
    return words


def compile_rules(node_labels, node_taints, group_rules, weight_taint=3, weight_node_affinity=2):
    """The Snapshot.node_bind rules dict of the same strings: taint triples numbered in order of first appearance,
    tolerations compiled with ToleratesTaint, the rule keys' domains numbered in sorted value order."""
    N, G = len(node_labels), len(group_rules)
    triples = []
    for ts in node_taints:
        for t in ts:
            k = (t["key"], t.get("value", ""), t["effect"])
            if k not in triples:
                triples.append(k)
    assert len(triples) <= 64
    bit = {t: np.uint64(1 << i) for i, t in enumerate(triples)}
    hard = np.zeros(N, np.uint64)
    softm = np.zeros(N, np.uint64)
    for n, ts in enumerate(node_taints):
        for t in ts:
            b = bit[t["key"], t.get("value", ""), t["effect"]]
            if t["effect"] == SOFT:
                softm[n] |= b
            else:
                hard[n] |= b
    tol_h = np.zeros(G, np.uint64)
    tol_s = np.zeros(G, np.uint64)
    for g, r in enumerate(group_rules):
        tols = r.get("tolerations", ())
        for (k, v, e), b in bit.items():
            taint = {"key": k, "value": v, "effect": e}
            if e != SOFT and any(tolerates(x, taint) for x in tols):
                tol_h[g] |= b
            if e == SOFT and any(tolerates(x, taint) for x in tols if x.get("effect", "") in ("", SOFT)):
                tol_s[g] |= b
    names = sorted({r["key"] for g in group_rules for t in (g.get("required") or []) + [t for _, t in
                    g.get("preferred", ())] for r in t})
    kid = {k: i for i, k in enumerate(names)}
    values = {k: sorted({lab[k] for lab in node_labels if k in lab}) for k in names}
    rule_keys = []
    for k in names:
        idx = {v: i for i, v in enumerate(values[k])}
        rule_keys.append((np.array([idx[lab[k]] if k in lab else -1 for lab in node_labels], np.int32),
                          len(values[k])))
    node_terms = []
    for g, r in enumerate(group_rules):
        for w, terms in ((0, r.get("required") or []), *[(w, [t]) for w, t in r.get("preferred", ())]):
            for t in terms:
                node_terms.append((g, w, [(kid[q["key"]], expr_set(q, values[q["key"]], len(values[q["key"]])))
                                          for q in t]))
    return dict(n_taints=len(triples), taint_hard=hard, taint_soft=softm, tolerate_hard=tol_h, tolerate_soft=tol_s,
                rule_keys=rule_keys, node_terms=node_terms, weight_taint=weight_taint,
                weight_node_affinity=weight_node_affinity)


ZONES, TYPES = ("z0", "z1", "z2"), ("m5", "c5", "r5", "g4", "p4")


def random_cluster(rng, N, G, n_taints=3):
    """Node label maps (zone, instance type, gen with some non-integers, a few nodes without each key), node taints
    (control-plane NoSchedule on 3 nodes, a 5% GPU pool NoSchedule, PreferNoSchedule spot nodes, and with n_taints > 3
    further distinct triples until n_taints exist) and per-group rules: tolerations, required terms of In / NotIn /
    Exists / DoesNotExist / Gt / Lt, an empty term now and then, and up to two preferred terms."""
    labels = []
    for n in range(N):
        lab = {}
        if rng.random() < 0.95:
            lab["zone"] = ZONES[int(rng.integers(0, 3))]
        if rng.random() < 0.9:
            lab["type"] = TYPES[int(rng.integers(0, 5))]
        if rng.random() < 0.8:
            lab["gen"] = str(int(rng.integers(1, 6))) if rng.random() < 0.9 else "x1"
        labels.append(lab)
    taints = [[] for _ in range(N)]
    if n_taints:
        for n in rng.choice(N, min(3, N), replace=False):
            taints[n].append({"key": "node-role.kubernetes.io/control-plane", "value": "", "effect": "NoSchedule"})
    if n_taints >= 2:
        for n in np.nonzero(rng.random(N) < 0.05)[0]:
            taints[n].append({"key": "gpu", "value": "true", "effect": "NoSchedule"})
    if n_taints >= 3:
        for n in np.nonzero(rng.random(N) < 0.2)[0]:
            taints[n].append({"key": "spot", "value": "", "effect": "PreferNoSchedule"})
    effects = ("NoSchedule", "NoExecute", "PreferNoSchedule")
    extra = [{"key": f"t{i % 20}", "value": f"v{i // 20}", "effect": effects[i % 3]} for i in range(max(0, n_taints - 3))]
    for t in extra:  # every extra triple on at least one node, and on about 3% of them
        for n in set([int(rng.integers(0, N))] + np.nonzero(rng.random(N) < 0.03)[0].tolist()):
            taints[n].append(t)
    tol_pool = [
        {"key": "node-role.kubernetes.io/control-plane", "operator": "Exists", "effect": "NoSchedule"},
        {"key": "gpu", "operator": "Equal", "value": "true", "effect": ""},
        {"key": "spot", "operator": "Exists", "effect": "PreferNoSchedule"},
        {"key": "spot", "operator": "Exists", "effect": "NoSchedule"},  # tolerates no PreferNoSchedule taint
        {"key": "", "operator": "Exists", "effect": ""},  # tolerates everything
        {"key": "t3", "operator": "Equal", "value": "v0", "effect": ""},
        {"key": "t4", "operator": "Exists", "effect": "NoExecute"},
    ]
    reqs = [
        {"key": "zone", "operator": "In", "values": ["z0", "z1"]},
        {"key": "zone", "operator": "NotIn", "values": ["z2"]},
        {"key": "type", "operator": "In", "values": ["m5", "c5", "r5"]},
        {"key": "type", "operator": "Exists"},
        {"key": "gen", "operator": "DoesNotExist"},
        {"key": "gen", "operator": "Gt", "values": ["2"]},
        {"key": "gen", "operator": "Lt", "values": ["4"]},
        {"key": "zone", "operator": "In", "values": ["z9"]},
    ]

    def term():
        return [reqs[int(i)] for i in rng.choice(len(reqs), int(rng.integers(1, 3)), replace=False)]
    rules = []
    for g in range(G):
        r = {"tolerations": [tol_pool[int(i)] for i in rng.choice(len(tol_pool), int(rng.integers(0, 3)), replace=False)]
             if rng.random() < 0.6 else []}
        u = rng.random()
        if u < 0.5:
            r["required"] = [term() for _ in range(int(rng.integers(1, 3)))] + ([[]] if rng.random() < 0.1 else [])
        if rng.random() < 0.6:
            r["preferred"] = [(int(rng.integers(1, 101)), term()) for _ in range(int(rng.integers(1, 3)))]
        rules.append(r)
    return labels, taints, rules
