"""Shared helpers of the bind-walk edge tests (test_bind_edges.py on the CPU, test_bind_edges_gpu.py on the H100): the
value families of test_commit_paths_gpu.py shaped into bind queues, the walk's node slices, the five calls' oracles
behind one signature, and reduced_reference, a vectorised restatement of the five calls where only resources matter.

Every result is the 7-tuple (node_idx, score, parts, refused, counts, soft_counts, free_r), None where a call has no
such output: spread and affinity have no parts, soft counts or free_r; profile and node no free_r."""
import numpy as np

from affinity_bind_oracle import AFFINITY, ANTI, affinity_bind_packed
from fit_bind_oracle import compile_resources, final_free, fit_bind_packed
from node_bind_oracle import node_bind_packed
from profile_bind_oracle import ANTI_PREFERRED, PREFERRED, profile_bind_packed
from spread_bind_oracle import spread_bind_packed
from spread_oracle import scores_at
from test_commit_paths_gpu import _family, _slice_edges
from test_fit_bind_gpu import EXTRA

CALLS = ("spread", "affinity", "profile", "node", "fit")
POLICIES = {"spread": (0, 1, 3, 4), "affinity": (0, 1, 3, 4), "profile": (1, 3, 4), "node": (1, 3, 4),
            "fit": (1, 3, 4)}
REFUSAL_WORDS = {"spread": 1, "affinity": 2, "profile": 2, "node": 4, "fit": 5}
PART_WORDS = {"profile": 3, "node": 5, "fit": 5}
NAMES = ["pods"] + EXTRA  # resource r of the arrays is NAMES[r]; "pods" requests 1 per pod, as compile_resources
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SETUP_WARPS = 8  # k_affinity_setup / k_profile_setup: one warp per existing pod, 8 per CTA, at most 4 CTAs per SM


def bind_slices(N, sms):
    """The walk's node slices, as the launcher sizes k_bind_seq: grid = min(SMs, ceil(N / 128)) CTAs of ceil(N / grid)
    nodes (the formula of k_stream_batch, test_commit_paths_gpu._slices); a slice longer than 256 gives one thread
    several nodes"""
    grid = max(1, min(sms, (N + 127) // 128))
    return grid, (N + grid - 1) // grid


def setup_passes(E, sms):
    """Turns of the grid-stride loop of k_affinity_setup / k_profile_setup over E existing pods"""
    grid = max(1, min((E + SETUP_WARPS - 1) // SETUP_WARPS, 4 * sms))
    return (E + grid * SETUP_WARPS - 1) // (grid * SETUP_WARPS)


def edge_keys(rng, N, sms):
    """Three topology keys whose domains cut across the walk's slice edges: zones one slice long shifted by half a
    slice (every slice edge lies inside a zone), with a quarter of the edge nodes lacking the key; hostnames with 5% of
    the nodes lacking it; three stripes n % 3 (every domain in every slice)."""
    _, chunk = bind_slices(N, sms)
    n = np.arange(N)
    zone = ((n + chunk // 2) // chunk).astype(np.int32)
    Dz = int(zone.max()) + 1 if N else 1
    e = _slice_edges(N, sms) if N else np.zeros(0, np.int64)
    zone[e[rng.random(len(e)) < 0.25]] = -1
    host = n.astype(np.int32)
    host[rng.random(N) < 0.05] = -1
    return [(zone, Dz), (host, max(N, 1)), ((n % 3).astype(np.int32), 3)]


def bind_family(name, rng, N, P, W, sms, G):
    """test_commit_paths_gpu._family as a bind queue: (ac, am, lab, fc, fm, rc, rm, sel, group, keys).  Pods fall in
    groups -1 .. G - 1 at random and every pod of group g carries g's selector (the bind calls require one selector per
    group); keys from edge_keys."""
    ac, am, lab, fc, fm, rc, rm, sel = _family(name, rng, N, P, W, sms)
    group = rng.integers(-1, G, P).astype(np.int32) if G else np.full(P, -1, np.int32)
    sel = sel.copy()
    if G and P:
        gsel = sel[rng.integers(0, P, G)]
        sel[group >= 0] = gsel[group[group >= 0]]
    return ac, am, lab, fc, fm, rc, rm, sel, group, edge_keys(rng, N, sms)


def constraints(rng, G, keys):
    """(max_skew, min_domains, existing) for G groups: group 0 constrains every key at max_skew 1, the others draw
    {0, 1, 2, 5} per key; the second half of the groups ask for one more domain than key 0 has; existing counts 0-2."""
    K = len(keys)
    skew = np.array([0, 1, 2, 5], np.uint32)[rng.integers(0, 4, (G, K))]
    skew[0] = 1
    mind = np.zeros((G, K), np.uint32)
    mind[G // 2:, 0] = keys[0][1] + 1
    ex = [rng.integers(0, 3, (G, D)).astype(np.uint32) for _, D in keys]
    return skew, mind, ex


def reduced_resources(rng, N, P, R, pods=(-1, 13), per_node=(-3, 9), gpu_share=0.5):
    """(node_free [R, N], pod_req [P, R]) for R resources NAMES[:R]: pod slots drawn from `pods`, the other amounts from
    `per_node` (negative free included); every pod requests one pod slot, and each other resource with probability
    gpu_share, 1-3 units"""
    free = rng.integers(per_node[0], per_node[1], (R, N)).astype(np.int64)
    if R:
        free[0] = rng.integers(pods[0], pods[1], N)
    req = np.where(rng.random((P, R)) < gpu_share, rng.integers(1, 4, (P, R)), 0).astype(np.int64)
    if R:
        req[:, 0] = 1
    return free, req


def resource_maps(node_free, pod_req):
    """The same resources as fit_bind_oracle's name maps: (alloc, bound, pod_res) with no bound pod"""
    R, N = node_free.shape
    alloc = [{NAMES[r]: int(node_free[r, n]) for r in range(R)} for n in range(N)]
    pod_res = [{NAMES[r]: int(q[r]) for r in range(1, R)} for q in pod_req]
    return alloc, [], pod_res


def no_rules(N, G):
    """Node label maps, taints and group rules that pass every node (TaintToleration 100 on every node)"""
    return [{}] * N, [[]] * N, [{}] * G


def oracle(call, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, policy, terms=(), ex_pods=None, skew=None,
           mind=None, ex=None, soft=None, term_weight=None, hard=1, cluster=None, res=None):
    """The call's oracle, free_cpu / free_mem charged in place; cluster = (node labels, taints, group rules) for node and
    fit, res = (alloc, bound, pod_res) name maps for fit.  Returns the 7-tuple."""
    if call == "spread":
        sk = np.zeros((G, len(keys)), np.uint32) if skew is None else skew
        node, score, ref, cnt = spread_bind_packed(fc, fm, ac, am, lab, rc, rm, sel, group, keys, sk, mind, ex, policy)
        return node, score, None, ref, cnt, None, None
    if call == "affinity":
        node, score, ref, cnt = affinity_bind_packed(fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms, ex_pods,
                                                     skew, mind, ex, policy)
        return node, score, None, ref, cnt, None, None
    kw = dict(soft_skew=soft, term_weight=term_weight, hard_affinity_weight=hard)
    if call == "profile":
        return profile_bind_packed(fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms, ex_pods, skew, mind, ex,
                                   policy, **kw) + (None,)
    nl, nt, gr = cluster if cluster is not None else no_rules(len(fc), G)
    if call == "node":
        return node_bind_packed(fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, nl, nt, gr, terms, ex_pods, skew,
                                mind, ex, policy, **kw) + (None,)
    alloc, bound, pod_res = res
    out = fit_bind_packed(fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, nl, nt, gr, alloc, bound, pod_res, terms,
                          ex_pods, skew, mind, ex, policy, **kw)
    return out[:6] + (final_free(alloc, out[6], fit_names(pod_res)),)


def fit_names(pod_res):
    """The resource rows a fit call is given for these pods: "pods", then EXTRA's names some pod requests"""
    return ["pods"] + [nm for nm in EXTRA if any(nm in r for r in pod_res)]


def fit_arrays(res):
    """(node_free, pod_req) of name maps, rows in fit_names order"""
    alloc, bound, pod_res = res
    _, free, req = compile_resources(alloc, bound, pod_res, fit_names(pod_res))
    return free, req


def reduced_reference(call, fc, fm, ac, am, lab, rc, rm, sel, policy, node_free=None, pod_req=None, weight_taint=3):
    """The five calls where only resources matter: every pod in group -1 or a group without constraints, no terms, no
    soft keys, node rules that pass every node, R scalar resources (node_free [R, N], pod_req [P, R], fit only).  Per
    pod: fit, selector and the resources the pod requests, the policy's score from spread_oracle.scores_at (j = 0) plus
    the constant parts (pts 0, ipa 0, TaintToleration 100 at weight_taint for node and fit, NodeAffinity 0), the
    lowest-index argmax, free_cpu / free_mem charged in place and free_r charged.  Returns the 7-tuple with counts and
    soft counts None (they stay the existing counts)."""
    N, P = len(fc), len(rc)
    ac, am = np.asarray(ac, np.int64), np.asarray(am, np.int64)
    lab = np.asarray(lab, np.uint64).reshape(N, -1)
    sel = np.asarray(sel, np.uint64).reshape(P, -1)
    free_r = None if node_free is None else np.array(node_free, np.int64).reshape(-1, N)
    req = None if pod_req is None else np.asarray(pod_req, np.int64).reshape(P, -1)
    const = 100 * weight_taint if call in ("node", "fit") else 0
    node = np.full(P, -1, np.int32)
    score = np.zeros(P, np.int64)
    refused = np.zeros((P, REFUSAL_WORDS[call]), np.uint32)
    parts = np.zeros((P, PART_WORDS[call]), np.int64) if call in PART_WORDS else None
    match = {}
    for p in range(P):
        ok = match.get(sel[p].tobytes())
        if ok is None:
            ok = match[sel[p].tobytes()] = ((sel[p][None, :] & ~lab) == 0).all(axis=1)
        q_c, q_m = int(rc[p]), int(rm[p])
        cand = ok & (fc >= q_c) & (fm >= q_m)
        if req is not None:
            on = np.flatnonzero(req[p])
            if len(on):
                res_ok = (free_r[on] >= req[p, on][:, None]).all(axis=0)
                refused[p, 0] = np.count_nonzero(cand & ~res_ok)
                cand &= res_ok
        idx = np.flatnonzero(cand)
        if not len(idx):
            continue
        s = scores_at(fc[idx], fm[idx], ac[idx], am[idx], q_c, q_m, np.zeros(len(idx), np.int64), policy)
        n = int(idx[int(s.argmax())])  # first maximum: the lowest index
        node[p], score[p] = n, int(s.max()) + const
        if parts is not None:
            parts[p, 0] = s.max()
            if PART_WORDS[call] == 5:
                parts[p, 3] = 100
        fc[n] -= q_c
        fm[n] -= q_m
        if req is not None:
            free_r[:, n] -= req[p]
    return node, score, parts, refused[:, 0] if call == "spread" else refused, None, None, free_r


def existing_pods(rng, keys, G, E, lacking=0.05):
    """E existing pods (groups, nodes) over G groups: a share `lacking` of them on nodes that lack key 0 or key 1, the
    rest on nodes that carry both"""
    lack = np.flatnonzero((keys[0][0] < 0) | (keys[1][0] < 0))
    full = np.flatnonzero((keys[0][0] >= 0) & (keys[1][0] >= 0))
    nodes = full[rng.integers(0, len(full), E)].astype(np.int32)
    on_lack = rng.random(E) < lacking
    nodes[on_lack] = lack[rng.integers(0, len(lack), int(on_lack.sum()))]
    return rng.integers(0, G, E).astype(np.int32), nodes


def pod_terms(rng, G, K, preferred):
    """Required affinity and anti-affinity terms on a third of the groups each (anti on key 1, affinity on key 0 towards
    two other groups), and with preferred one or two weighted preferred terms (kinds 2 and 3) per group.  Returns
    (terms, term_weight)."""
    terms, weights = [], []
    for g in range(G):
        u = rng.random()
        if u < 1 / 3:
            terms.append((g, ANTI, 1, [g, int(rng.integers(0, G))]))
            weights.append(0)
        elif u < 2 / 3:
            terms.append((g, AFFINITY, 0, sorted({int(x) for x in rng.integers(0, G, 2)})))
            weights.append(0)
        if preferred:
            for _ in range(int(rng.integers(1, 3))):
                terms.append((g, PREFERRED if rng.random() < 0.6 else ANTI_PREFERRED, int(rng.integers(0, K)),
                              [int(rng.integers(0, G))]))
                weights.append(int(rng.integers(1, 101)))
    return terms, weights


# The shapes of test_bind_edges_gpu.py, checked on the CPU by test_bind_edges.py
FAMILY_N = (1, 129, 16_897, 33_793)  # one node, one slice and a bit, 132 SMs' last slice empty, slices of 257 nodes
LARGE_N = 150_000                    # slices of 1,137 nodes on 132 SMs (1,316 on 114)
TIE_N = 33_793                       # the smallest N with slices longer than 256 on 132 SMs
EXISTING_E, EXISTING_N = 20_000, 3_000
RULE_CLASSES, RULE_N = 64, 16_897    # 1.08 M rule words
FULL_P, FULL_N = 65_536, 2_000


def full_queue(rng, N, P, W=1, G=4):
    """A full-size queue that fills most nodes before it ends: (fc, fm, ac, am, lab, rc, rm, sel, group, keys,
    node_free, pod_req).  About 24 pods' cpu and memory per node; 10-39 pod slots per node and 0, 4 or 8 GPUs, 15% of
    the pods asking for 1 or 2.  G groups without constraints and group -1, each group with a one-bit selector or none;
    keys: 7 zones (8% of the nodes without one) and hostnames."""
    ac = rng.choice([4000, 8000, 16000], N).astype(np.int64)
    am = rng.choice([16, 32, 64], N).astype(np.int64) << 30
    fc, fm = ac - rng.integers(0, 1000, N), am - rng.integers(0, 2 << 30, N)
    lab = rng.integers(0, 1 << 63, (N, W), dtype=np.uint64) | rng.integers(0, 1 << 63, (N, W), dtype=np.uint64)
    rc, rm = rng.integers(0, 800, P).astype(np.int64), rng.integers(0, 3 << 30, P).astype(np.int64)
    group = rng.integers(-1, G, P).astype(np.int32)
    gsel = np.zeros((G + 1, W), np.uint64)
    for g in range(1, G + 1):
        if g % 2:
            gsel[g, int(rng.integers(0, W))] = np.uint64(1) << np.uint64(rng.integers(0, 64))
    sel = gsel[group + 1]
    zone = rng.integers(0, 7, N).astype(np.int32)
    zone[rng.random(N) < 0.08] = -1
    keys = [(zone, 7), (np.arange(N, dtype=np.int32), N)]
    node_free = np.stack([rng.integers(10, 40, N), rng.choice([0, 4, 8], N)]).astype(np.int64)
    pod_req = np.stack([np.ones(P), np.where(rng.random(P) < 0.15, rng.integers(1, 3, P), 0)], 1).astype(np.int64)
    return fc, fm, ac, am, lab, rc, rm, sel, group, keys, node_free, pod_req
