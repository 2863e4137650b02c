"""Bind walks at their edges (-m gpu): ks_spread_bind, ks_affinity_bind, ks_profile_bind, ks_node_bind and ks_fit_bind bit
for bit against their oracles (tests/*_bind_oracle.py) or, where only resources matter, against
bind_edges.reduced_reference: node, score, parts, every refusal word, hard and soft counts, the final free[] and free_r.

The inputs reach what the benign tests of each call do not: the value families of the claim-committing paths (adversarial
values, one key everywhere, rising scores, negative free, allocatable <= 0 or tiny, values at the request limits, ties at
slice edges); node counts whose slices give one thread several nodes (N > 256 * SMs); existing-pod sets that take the
setup kernels' grid-stride loop round again (E > 8 * 4 * SMs); node-rule words beyond one pass of k_node_rules_setup;
queues of KS_SPREAD_BIND_MAX_PODS pods; free_r at the ends of int64; and requests at exactly the limits and one unit
above.  After every call free[] lies within +-2^36 millicores / +-2^55 bytes."""
import numpy as np
import pytest

from bind_edges import (AFFINITY, ANTI, CALLS, EXISTING_E, EXISTING_N, FAMILY_N, FULL_N, FULL_P, LARGE_N,
                        POLICIES, PREFERRED, RULE_CLASSES, RULE_N, TIE_N, bind_family, bind_slices, constraints,
                        edge_keys, existing_pods, fit_arrays, full_queue, no_rules, oracle, pod_terms,
                        reduced_reference, resource_maps, setup_passes)
from node_bind_oracle import compile_rules, random_cluster
from test_commit_paths_gpu import FAMILIES, INT64_MAX, INT64_MIN, KS_ERR_RANGE, LIM_C, LIM_M, _free_in_range, _load
from test_fit_bind_gpu import resources
from test_replicas_gpu import _nodes, load
from test_spread_bind_gpu import key_set, mixed_queue
from test_spread_gpu import zone_labels

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sms(ks):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def device(call, snap, rc, rm, sel, group, G, keys, policy, terms=(), ex_pods=None, skew=None, mind=None, ex=None,
           soft=None, term_weight=None, hard=1, rules=None, node_free=None, pod_req=None):
    """The call on the snapshot, as the 7-tuple of bind_edges.oracle"""
    if call == "spread":
        sk = np.zeros((G, len(keys)), np.uint32) if skew is None else skew
        idx, score, ref, cnt = snap.spread_bind(rc, rm, sel, group, keys, sk, mind, ex, policy)
        return idx, score, None, ref, cnt, None, None
    if call == "affinity":
        idx, score, ref, cnt = snap.affinity_bind(rc, rm, sel, group, G, keys, terms, ex_pods, skew, mind, ex, policy)
        return idx, score, None, ref, cnt, None, None
    args = (rc, rm, sel, group, G, keys, terms, ex_pods, skew, mind, ex, policy)
    kw = dict(soft_skew=soft, term_weight=term_weight, hard_affinity_weight=hard)
    if call == "profile":
        return snap.profile_bind(*args, **kw) + (None,)
    if call == "node":
        return snap.node_bind(*args, rules=rules, **kw) + (None,)
    return snap.fit_bind(*args, rules=rules, node_free=node_free, pod_req=pod_req, **kw)


FIELDS = ("node_idx", "score", "parts", "refused", "counts", "soft_counts", "free_r")


def same(got, want, tag):
    for name, g, w in zip(FIELDS, got, want):
        if w is None:
            continue
        if name in ("counts", "soft_counts"):
            assert g is not None and len(g) == len(w), f"{name} {tag}"
            assert all(np.array_equal(a, b) for a, b in zip(g, w)), f"{name} {tag}"
            continue
        bad = np.nonzero((np.asarray(g) != np.asarray(w)).reshape(len(g), -1).any(1))[0] if g.shape == w.shape else []
        assert g.shape == w.shape and not len(bad), f"{name} {tag}: first rows {bad[:8]}"


def run(call, snap, nodes, queue, policy, tag, **kw):
    """Load nodes = (ac, am, lab, fc, fm), run the call and its oracle on queue = (rc, rm, sel, group, G, keys) and compare
    everything; cluster / res (name maps) feed the oracle and become rules / node_free, pod_req for the device."""
    ac, am, lab, fc, fm = nodes
    rc, rm, sel, group, G, keys = queue
    cluster, res = kw.pop("cluster", None), kw.pop("res", None)
    if call in ("node", "fit"):
        cluster = cluster if cluster is not None else no_rules(len(fc), G)
        kw["rules"] = compile_rules(*cluster)
    if call == "fit":
        kw["node_free"], kw["pod_req"] = fit_arrays(res)
    _load(snap, ac, am, lab, fc, fm)
    got = device(call, snap, rc, rm, sel, group, G, keys, policy, **kw)
    ofc, ofm = fc.copy(), fm.copy()
    for k in ("rules", "node_free", "pod_req"):
        kw.pop(k, None)
    want = oracle(call, ofc, ofm, ac, am, lab, rc, rm, sel, group, G, keys, policy, cluster=cluster, res=res, **kw)
    same(got, want, tag)
    gfc, gfm = _free_in_range(snap)
    assert np.array_equal(gfc, ofc) and np.array_equal(gfm, ofm), f"free {tag}"
    return got


def scoring(call, rng, G, K):
    """Terms, soft skews and weights for a family run: anti-affinity on hostnames within group 0, required affinity of
    group 1 to itself (the first-pod rule) and, for the scored calls, a preferred term of group 2 and soft skews"""
    terms = [(0, ANTI, 1, [0]), (1, AFFINITY, 0, [1])]
    if call == "spread":
        return {}
    if call == "affinity":
        return dict(terms=terms)
    return dict(terms=terms + [(2, PREFERRED, 2, [0, 3])], term_weight=[0, 0, 60], hard=3,
                soft=np.array([0, 1, 3], np.uint32)[rng.integers(0, 3, (G, K))])


# ------------------------------------------------------------------------------------- 1. families x calls x policies
FAMILY_CASES = [(call, fam) for call in CALLS for fam in FAMILIES]


@pytest.mark.parametrize("call,fam", FAMILY_CASES, ids=[f"{c}-{f.replace(' ', '_')}" for c, f in FAMILY_CASES])
def test_families(ks, sms, call, fam):
    """Every (call, value family) pair, and by the policy rotation every (call, policy) pair; N cycles through 1, 129,
    16,897 (132 SMs: the last slice empty) and 33,793 (slices of 257: a thread scans two nodes), W through 1, 2, 4, 8.
    Requests within [0, 2^36] / [0, 2^55]; negative free and allocatable <= 0 as set_nodes takes them; LEAST_ALLOCATED
    near 1.8e18 under tiny allocatable with the weighted parts on top."""
    i = CALLS.index(call) * len(FAMILIES) + FAMILIES.index(fam)
    N, W = FAMILY_N[i % 4], (1, 2, 4, 8)[(i // 4) % 4]
    policy = POLICIES[call][FAMILIES.index(fam) % len(POLICIES[call])]
    P = 160 if N < 1000 else 64 if call in ("spread", "affinity") else 20
    G = 4
    rng = np.random.default_rng([i, N, W, policy])
    ac, am, lab, fc, fm, rc, rm, sel, group, keys = bind_family(fam, rng, N, P, W, sms, G)
    skew, mind, ex = constraints(rng, G, keys)
    kw = dict(skew=skew, mind=mind if i % 2 else None, ex=ex if i % 3 else None, **scoring(call, rng, G, len(keys)))
    if call in ("node", "fit"):
        kw["cluster"] = random_cluster(rng, N, G, 3 + 61 * (i % 2))
    if call == "fit":
        kw["res"] = resources(rng, N, P, 2 + i % 7)
    with ks.Snapshot(0) as snap:
        got = run(call, snap, (ac, am, lab, fc, fm), (rc, rm, sel, group, G, keys), policy,
                  f"{call} {fam} N={N} W={W} policy={policy}", **kw)
    assert rc.max() <= LIM_C and rm.max() <= LIM_M
    if fam == "rising" and N > 1 and call == "spread":
        assert (got[0] >= 0).any()


# -------------------------------------------------------------------------------------------------------- 2. large N
@pytest.mark.parametrize("call", ["spread", "node", "fit"])
def test_large_n_mixed_queue(ks, sms, call):
    """N = 150,000: slices of ceil(N / SMs) nodes (1,137 on 132 SMs), so every thread scans five or more nodes and the
    per-thread strict '>' and the CTA-order merge settle every tie; a mixed queue of workloads and unconstrained pods"""
    N, W, G = LARGE_N, 2, 4
    P = 200 if call == "spread" else 12
    assert bind_slices(N, sms)[1] > 4 * 256
    rng = np.random.default_rng([N, CALLS.index(call)])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3, "host"))
    lab = zone_labels(lab, *keys[0])
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 3000), mem=(0, 12 << 30))
    kw = dict(skew=skew, mind=mind, ex=ex)
    if call != "spread":
        kw.update(terms=[(0, ANTI, 1, [0]), (1, PREFERRED, 0, [2])], term_weight=[0, 40],
                  soft=np.array([0, 1, 3], np.uint32)[rng.integers(0, 3, (G, 2))], cluster=random_cluster(rng, N, G, 3))
    if call == "fit":
        kw["res"] = resources(rng, N, P, 3)
    with ks.Snapshot(0) as snap:
        got = run(call, snap, (ac, am, lab, fc, fm), (rc, rm, sel, group, G, keys), 4 if call != "spread" else 0,
                  f"{call} N={N}", **kw)
    assert (got[0] >= 0).sum() > P // 2


@pytest.mark.parametrize("call", CALLS)
def test_homogeneous_ties_across_strides_and_ctas(ks, sms, call):
    """One key everywhere at N = 33,793 (slices of 257 on 132 SMs, 297 on 114): every choice is a tie, decided by the
    strict '>' inside a thread's stride and by the merge in CTA order"""
    N, W, G, P = TIE_N, 1, 4, 24
    assert bind_slices(N, sms)[1] > 256
    rng = np.random.default_rng([N, CALLS.index(call), 1])
    ac, am, lab, fc, fm, rc, rm, sel, group, keys = bind_family("homogeneous", rng, N, P, W, sms, G)
    skew, _, _ = constraints(rng, G, keys)
    kw = dict(skew=skew, **scoring(call, rng, G, len(keys)))
    if call == "fit":
        kw["res"] = resources(rng, N, P, 3)
    with ks.Snapshot(0) as snap:
        run(call, snap, (ac, am, lab, fc, fm), (rc, rm, sel, group, G, keys), POLICIES[call][-1], f"{call} N={N}", **kw)


# ------------------------------------------------------------------------------------------------ 3. existing pods
@pytest.mark.parametrize("call", ["affinity", "profile", "node", "fit"])
def test_many_existing_pods(ks, sms, call):
    """E = 20,000 existing pods over 16 groups (8 * 4 * SMs = 4,224 warps on 132 SMs: the setup kernels' grid-stride loop
    turns five times), about 5% on nodes that lack a key, with required affinity and anti-affinity, preferred terms of
    both kinds and a hard-affinity weight of 5 (k_profile_setup's 64-bit atomics of negative and positive
    coefficients).  The counters show through the bindings, refusals and parts."""
    N, W, G, P, E = EXISTING_N, 1, 16, 30, EXISTING_E
    assert setup_passes(E, sms) >= 2
    rng = np.random.default_rng([E, CALLS.index(call)])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = edge_keys(rng, N, sms)
    ex_pods = existing_pods(rng, keys, G, E)
    terms, weights = pod_terms(rng, G, len(keys), preferred=call != "affinity")
    group = rng.integers(-1, G, P).astype(np.int32)
    rc, rm = rng.integers(0, 3000, P).astype(np.int64), rng.integers(0, 12 << 30, P).astype(np.int64)
    sel = np.zeros((P, W), np.uint64)
    skew = np.zeros((G, len(keys)), np.uint32)
    skew[:4, 0] = 2
    kw = dict(terms=terms, ex_pods=ex_pods, skew=skew)
    if call != "affinity":
        kw.update(term_weight=weights, hard=5, soft=np.array([0, 1, 2], np.uint32)[rng.integers(0, 3, (G, len(keys)))])
    if call in ("node", "fit"):
        kw["cluster"] = random_cluster(rng, N, G, 3)
    if call == "fit":
        kw["res"] = resources(rng, N, P, 2)
    with ks.Snapshot(0) as snap:
        got = run(call, snap, (ac, am, lab, fc, fm), (rc, rm, sel, group, G, keys), 4 if call != "affinity" else 1,
                  f"{call} E={E}", **kw)
    assert (got[0] >= 0).any() and got[3][:, -1].any()  # some pods bound, some nodes refused by rules 1-3


# ---------------------------------------------------------------------------------------------- 4. node-rule classes
@pytest.mark.parametrize("call", ["node", "fit"])
def test_rule_classes_beyond_one_pass(ks, sms, call):
    """63 groups with distinct rules (and group -1): 64 classes x 16,897 nodes = 1.08 M rule words, eight passes of
    k_node_rules_setup's grid of 4 * SMs CTAs x 256 threads on 132 SMs"""
    N, W, G, P = RULE_N, 1, RULE_CLASSES - 1, 40
    assert RULE_CLASSES * N > 4 * sms * 256
    rng = np.random.default_rng([N, G, CALLS.index(call)])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3,))
    nl, nt, gr = random_cluster(rng, N, G, 8)
    for g, r in enumerate(gr):  # a preferred term of weight g + 1 makes every group's class its own
        r["preferred"] = list(r.get("preferred", [])) + [(g + 1, [{"key": "zone", "operator": "Exists"}])]
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 3000), mem=(0, 12 << 30))
    kw = dict(skew=skew, ex=ex, cluster=(nl, nt, gr))
    if call == "fit":
        kw["res"] = resources(rng, N, P, 2)
    with ks.Snapshot(0) as snap:
        got = run(call, snap, (ac, am, lab, fc, fm), (rc, rm, sel, group, G, keys), 1, f"{call} classes", **kw)
    assert (got[0] >= 0).any() and got[2][:, 4].any()  # some NodeAffinity parts above 0


# ------------------------------------------------------------------------------------------------- 5. full-size queues
@pytest.mark.parametrize("policy", [1, 3, 4])
@pytest.mark.parametrize("call", CALLS)
def test_full_size_queue(ks, sms, call, policy):
    """P = KS_SPREAD_BIND_MAX_PODS = 65,536 pods over 2,000 nodes that fill before the queue ends (pod slots and GPUs
    under fit, cpu and memory otherwise): long runs of the walk's pod loop, and for profile, node and fit of pass 1's
    clearing of the other parity's domain bitmap (the zone key), against reduced_reference, with free[] and free_r"""
    rng = np.random.default_rng([FULL_P, CALLS.index(call), policy])
    fc, fm, ac, am, lab, rc, rm, sel, group, keys, node_free, pod_req = full_queue(rng, FULL_N, FULL_P)
    G = int(group.max()) + 1
    assert FULL_P == ks.capi.KS_SPREAD_BIND_MAX_PODS
    kw = {}
    if call in ("node", "fit"):
        kw["rules"] = compile_rules(*no_rules(FULL_N, G))
    if call == "fit":
        kw.update(node_free=node_free, pod_req=pod_req)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got = device(call, snap, rc, rm, sel, group, G, keys, policy, **kw)
        ofc, ofm = fc.copy(), fm.copy()
        want = reduced_reference(call, ofc, ofm, ac, am, lab, rc, rm, sel, policy, *((node_free, pod_req)
                                                                                     if call == "fit" else ()))
        same(got, want, f"{call} P={FULL_P} policy={policy}")
        assert all(not c.any() for c in got[4]) and (got[5] is None or all(not c.any() for c in got[5]))
        gfc, gfm = _free_in_range(snap)
        assert np.array_equal(gfc, ofc) and np.array_equal(gfm, ofm)
    assert (got[0][-2000:] < 0).mean() > 0.5 and (got[0] >= 0).sum() > FULL_P // 3  # the nodes filled on the way


@pytest.mark.parametrize("call", CALLS)
def test_one_pod_over_the_queue_limit(ks, call):
    """P = 65,537: KS_ERR_RANGE before any device work, free[] unchanged"""
    rng = np.random.default_rng(3)
    N, P = 300, ks.capi.KS_SPREAD_BIND_MAX_PODS + 1
    fc, fm, ac, am, lab = _nodes(rng, N, 1)
    keys = [(np.arange(N, dtype=np.int32), N)]
    kw = {}
    if call in ("node", "fit"):
        kw["rules"] = compile_rules(*no_rules(N, 1))
    if call == "fit":
        kw.update(node_free=np.ones((1, N), np.int64), pod_req=np.ones((P, 1), np.int64))
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        with pytest.raises(ks.KsError) as e:
            device(call, snap, np.zeros(P, np.int64), np.zeros(P, np.int64), np.zeros((P, 1), np.uint64),
                   np.full(P, -1, np.int32), 1, keys, 1, **kw)
        assert e.value.code == KS_ERR_RANGE
        gfc, gfm = snap.free()
        assert np.array_equal(gfc, fc) and np.array_equal(gfm, fm)


def test_full_size_hostname_group_is_the_replica_plan(ks):
    """65,536 identical pods in one hostname-spread group (max_skew 1 over 2,000 hosts): the minimum rises 32 times, each
    time through spread_bind_commit's rescan of the domains at m, and the bindings, scores, counts and free[] equal
    ks_place_replicas_spread's copy list committed by ks_snapshot_commit_claims (test_one_group_is_the_replica_plan)"""
    rng = np.random.default_rng(0xB5)
    N, W, R = FULL_N, 1, FULL_P
    ac, am = np.full(N, 64000, np.int64), np.full(N, 256 << 30, np.int64)
    fc, fm = ac - rng.integers(0, 2000, N), am - rng.integers(0, 8 << 30, N)
    lab = np.zeros((N, W), np.uint64)
    rc, rm, sel = np.array([500], np.int64), np.array([1 << 30], np.int64), np.zeros((1, W), np.uint64)
    dom = np.arange(N, dtype=np.int32)
    skew = np.ones((1, 1), np.uint32)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        plan = snap.place_replicas_spread(rc, rm, sel, [R], dom, N, skew[:, 0], None, None, 4)
        acc = snap.commit_claims(plan[1], np.repeat(rc, R), np.repeat(rm, R))
        assert acc[plan[1] >= 0].all()
        want_free = snap.free()
        load(ks, snap, fc, fm, ac, am, lab)
        got = snap.spread_bind(np.repeat(rc, R), np.repeat(rm, R), np.repeat(sel, R, axis=0), np.zeros(R), [(dom, N)],
                               skew, None, None, 4)
        assert np.array_equal(got[0], plan[1]) and np.array_equal(got[1], plan[2])
        assert np.array_equal(got[3][0], plan[4].reshape(1, N))
        gfc, gfm = snap.free()
        assert np.array_equal(gfc, want_free[0]) and np.array_equal(gfm, want_free[1])
    assert (got[0] >= 0).all() and got[3][0].min() == R // N and got[3][0].max() == R // N + 1


# ------------------------------------------------------------------------------------------- 6. resource extremes
def test_fit_resource_extremes(ks, sms):
    """ks_fit_bind with R = 8: node_free across [INT64_MIN + 1, INT64_MAX], resources 1-6 never requested (zero requests
    against negative free), resource 7 requested up to INT64_MAX, among them requests exactly equal to a node's free;
    cpu and memory zero against negative free.  free_r exact at the ends of int64."""
    N, P, W, G = 129, 400, 1, 2
    rng = np.random.default_rng(0xE7)
    pool = np.array([INT64_MIN + 1, -(1 << 62), -1, 0, 1, 2, 1 << 40, INT64_MAX - 1, INT64_MAX], np.int64)
    node_free = pool[rng.integers(0, len(pool), (8, N))]
    node_free[0] = rng.integers(-1, 6, N)  # pod slots
    node_free[0, :4], node_free[7, :4] = 5, INT64_MAX
    req = np.zeros((P, 8), np.int64)
    req[:, 0] = 1
    req[:, 7] = np.array([0, 1, 2, 1 << 40, INT64_MAX - 1, INT64_MAX], np.int64)[rng.integers(0, 6, P)]
    ac, am = rng.choice([0, 1000], N).astype(np.int64), rng.choice([0, 1 << 30], N).astype(np.int64)
    fc, fm = rng.choice([-1000, -1, 0, 500, 1000], N).astype(np.int64), rng.choice([-1, 0, 1 << 30], N).astype(np.int64)
    fc[:4], fm[:4] = 1000, 1 << 30  # the nodes of INT64_MAX free take what fits them
    lab = np.zeros((N, W), np.uint64)
    rc, rm = rng.choice([0, 0, 0, 1], P).astype(np.int64), rng.choice([0, 0, 1], P).astype(np.int64)
    group = rng.integers(-1, G, P).astype(np.int32)
    keys = [(np.arange(N, dtype=np.int32), N)]
    res = resource_maps(node_free, req)
    with ks.Snapshot(0) as snap:
        got = run("fit", snap, (ac, am, lab, fc, fm), (rc, rm, np.zeros((P, W), np.uint64), group, G, keys), 3,
                  "resource extremes", skew=np.zeros((G, 1), np.uint32), res=res)
        want = reduced_reference("fit", fc.copy(), fm.copy(), ac, am, lab, rc, rm, np.zeros((P, W), np.uint64), 3,
                                 node_free, req)
        same(got, want, "resource extremes, reduced")
    bound = got[0] >= 0
    assert (bound & (req[:, 7] == INT64_MAX)).any() and (got[6][7] == 0).any()  # a request equal to free took it
    assert (~bound & (req[:, 7] > 0)).any() and got[3][:, 0].any()
    assert np.array_equal(got[6][1:7], node_free[1:7])  # never requested: never charged


# ------------------------------------------------------------------------------------------------ 7. request limits
@pytest.mark.parametrize("call", CALLS)
def test_requests_at_the_limits(ks, orc, call):
    """Requests of exactly 2^36 millicores and 2^55 bytes are taken and bound where free allows (nodes with free at the
    limits); one unit more in either gives KS_ERR_RANGE with free[] unchanged and the select index still the oracle's"""
    N, W, G = 257, 1, 2
    rng = np.random.default_rng([LIM_C, CALLS.index(call)])
    ac, am = np.full(N, LIM_C, np.int64), np.full(N, LIM_M, np.int64)
    fc, fm = ac.copy(), am.copy()
    fc[::2], fm[::3] = LIM_C - 1, LIM_M - 1
    lab = np.zeros((N, W), np.uint64)
    P = 12
    rc = np.array([LIM_C, 0, LIM_C, 1] * 3, np.int64)
    rm = np.array([LIM_M, LIM_M, 0, 1] * 3, np.int64)
    sel = np.zeros((P, W), np.uint64)
    group = (np.arange(P) % 3 - 1).astype(np.int32)
    keys = [(np.arange(N, dtype=np.int32), N)]
    res = resource_maps(np.full((2, N), 3, np.int64), np.ones((P, 2), np.int64)) if call == "fit" else None
    skew = np.zeros((G, 1), np.uint32)
    with ks.Snapshot(0) as snap:
        got = run(call, snap, (ac, am, lab, fc, fm), (rc, rm, sel, group, G, keys), POLICIES[call][-1],
                  f"{call} at the limits", skew=skew, res=res)
        assert (got[0][(rc == LIM_C) & (rm == LIM_M)] >= 0).all()  # bound where free allows
        before = snap.free()
        kw = {}
        if call in ("node", "fit"):
            kw["rules"] = compile_rules(*no_rules(N, G))
        if call == "fit":
            kw["node_free"], kw["pod_req"] = fit_arrays(res)
        for c, m in ((LIM_C + 1, 0), (0, LIM_M + 1)):
            qc, qm = rc.copy(), rm.copy()
            qc[5], qm[5] = c, m
            with pytest.raises(ks.KsError) as e:
                device(call, snap, qc, qm, sel, group, G, keys, POLICIES[call][-1], skew=skew, **kw)
            assert e.value.code == KS_ERR_RANGE, (call, c, m)
            after = _free_in_range(snap)
            assert np.array_equal(after[0], before[0]) and np.array_equal(after[1], before[1])
        oidx, oscore = orc.run_packed(*before, ac, am, lab, rc, rm, sel, policy=1, want_mask=False)[:2]
        for flags in (ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR):
            r = snap.select(rc, rm, sel, policy=1, flags=flags)
            assert np.array_equal(r.node_idx, oidx) and np.array_equal(r.score, oscore), (call, r.path)
