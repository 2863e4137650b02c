"""CPU restatement of extended resources when binding (ks_fit_bind, include/ksched.h; DESIGN.md 5r).

Upstream's NodeResourcesFit fitsRequest is restated over resource-name maps: the pod count (`len(pods) + 1 > allowed`,
checked for every pod), then each scalar resource the pod requests with a non-zero quantity against allocatable minus
what the node's pods request, a name missing from the node's allocatable counting as 0.  The maps are the input: this
module never reads the arrays a caller compiles for the device (compile_resources makes those, for the device tests
and the host-layer tests to compare against).  Everything else - cpu, memory, selector, taints, node affinity, spread,
inter-pod affinity, scores and tie order - is node_bind_oracle's, whose helpers the walk below calls in the same order
as node_bind_packed.
alloc[n]: {name: int} of node n (cpu and memory are not read); bound: [(node, {name: int})] of the pods already on the
nodes; pod_res[p]: {name: int} of queued pod p."""
import numpy as np

from affinity_bind_oracle import AFFINITY, ANTI, affinity_mask
from node_bind_oracle import intolerable_soft, normalize, preferred_raw, required_ok, untolerated_hard
from profile_bind_oracle import ipa_raw, pts_scores
from replicas_oracle import _specs
from spread_oracle import scores_at

CPU_MEM = ("cpu", "memory")


def fits_request(req, alloc, requested, n_pods):
    """Upstream fitsRequest without cpu and memory: the names that are insufficient on the node ("pods" first)."""
    out = []
    if n_pods + 1 > alloc.get("pods", 0):
        out.append("pods")
    for name, q in req.items():
        if name in CPU_MEM or name == "pods" or q == 0:
            continue
        if q > alloc.get(name, 0) - requested.get(name, 0):
            out.append(name)
    return out


class NodeUsage:
    """What the pods on each node request, by name, and how many pods there are."""

    def __init__(self, N, bound):
        self.req = [dict() for _ in range(N)]
        self.pods = [0] * N
        for n, r in bound:
            self.add(n, r)

    def add(self, n, r):
        self.pods[n] += 1
        for name, q in r.items():
            if name not in CPU_MEM:
                self.req[n][name] = self.req[n].get(name, 0) + q


def fit_bind_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, group, n_groups, keys,
                    node_labels, node_taints, group_rules, alloc, bound, pod_res, terms=(), existing_pods=None,
                    max_skew=None, min_domains=None, existing=None, policy=4, soft_skew=None, soft_all_keys=None,
                    term_weight=None, hard_affinity_weight=1, weight_spread=2, weight_affinity=2, weight_taint=3,
                    weight_node_affinity=2):
    """Returns (node_idx [P], score [P], parts [P, 5], refused [P, 5], counts, soft_counts, usage) as Snapshot.fit_bind
    with a NodeUsage in place of free_r; free_cpu / free_mem are charged in place."""
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
    placed = [] if existing_pods is None else [(int(h), int(m)) for h, m in zip(*existing_pods)]
    rule = [group_rules[g] if g < len(group_rules) else {} for g in range(G)]
    usage = NodeUsage(N, bound)

    def rule_of(g):
        return rule[g] if g >= 0 else {}
    taint_ok = {g: np.array([not untolerated_hard(node_taints[n], rule_of(g).get("tolerations", ()))
                             for n in range(N)], bool) for g in range(-1, G)}
    aff_ok = {g: np.array([required_ok(rule_of(g), node_labels[n]) for n in range(N)], bool) for g in range(-1, G)}

    def start():
        return [np.zeros((G, d), np.int64) if existing is None else np.asarray(existing[k], np.int64).reshape(G, d).copy()
                for k, d in enumerate(D)]
    cnt, sc = start(), start()
    # eligible domains: selector, required node affinity and every constrained key; resources and taints play no part
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
    refused = np.zeros((P, 5), np.uint32)
    for p in range(P):
        rc, rm, g = int(req_cpu[p]), int(req_mem[p]), int(group[p])
        feasible = (rc <= fc) & (rm <= fm) & ((sel[p][None, :] & ~labels) == 0).all(axis=1)
        res_ok = np.array([not fits_request(pod_res[p], alloc[n], usage.req[n], usage.pods[n]) for n in range(N)], bool)
        fit = feasible & res_ok
        tol = fit & taint_ok[g]
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
        passing = affinity_mask(g, placed, required, dom)
        refused[p] = ((feasible & ~res_ok).sum(), (fit & ~taint_ok[g]).sum(), (tol & ~aff_ok[g]).sum(),
                      (nodeaff & ~spread_ok).sum(), (nodeaff & spread_ok & ~passing).sum())
        F = np.nonzero(nodeaff & spread_ok & passing)[0].tolist()
        if not F:
            continue
        policy_score = scores_at(fc, fm, ac, am, rc, rm, np.zeros(N, np.int64), policy)
        pts = pts_scores(F, g, soft, soft_all, dom, sc)
        iraw = ipa_raw(g, placed, terms, weights, hard_affinity_weight, dom)
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
        usage.add(n, pod_res[p])
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
        placed.append((g, n))
    return (node, score, parts, refused, [c.astype(np.uint32) for c in cnt], [c.astype(np.uint32) for c in sc], usage)


def batch_names(pod_res):
    """"pods", then every other name some pod requests with a non-zero quantity, in order of first request."""
    names = ["pods"]
    for r in pod_res:
        for name, q in r.items():
            if name not in CPU_MEM and name != "pods" and q != 0 and name not in names:
                names.append(name)
    return names


def compile_resources(alloc, bound, pod_res, names=None):
    """The arrays ks_fit_bind takes for these maps: (names, node_free int64 [R, N], pod_req int64 [P, R])."""
    names = batch_names(pod_res) if names is None else names
    usage = NodeUsage(len(alloc), bound)
    free = np.array([[alloc[n].get(r, 0) - (usage.pods[n] if r == "pods" else usage.req[n].get(r, 0))
                      for n in range(len(alloc))] for r in names], np.int64).reshape(len(names), len(alloc))
    req = np.array([[1 if r == "pods" else q.get(r, 0) for r in names] for q in pod_res],
                   np.int64).reshape(len(pod_res), len(names))
    return names, free, req


def final_free(alloc, usage, names):
    """free_r after a walk, from the NodeUsage fit_bind_packed returns."""
    return np.array([[alloc[n].get(r, 0) - (usage.pods[n] if r == "pods" else usage.req[n].get(r, 0))
                      for n in range(len(alloc))] for r in names], np.int64).reshape(len(names), len(alloc))
