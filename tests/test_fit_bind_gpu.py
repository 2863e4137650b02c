"""Extended resources when binding (ks_fit_bind) on the H100: node, total, five parts, five refusals, hard and soft
counts, the final free[] and free_r bit for bit against tests/fit_bind_oracle.py (which evaluates resource-name maps)
across R = 1-8, label widths 1-8, policies 1, 3 and 4, rules NULL and given, with and without existing pods, node counts
at the CTA-slice edges, one node and the empty snapshot; L1 and L4 against ks_node_bind on the device, with the same
launches (one more with rules NULL); host errors leaving free[] unchanged; ks_select on both paths after the call; and ksh_reconcile_fit end to
end with status 8 and a second call that sees the first call's GPU and pod usage."""
import ctypes as C

import numpy as np
import pytest

from affinity_bind_oracle import ANTI
from fit_bind_oracle import compile_resources, final_free, fit_bind_packed
from node_bind_oracle import compile_rules, random_cluster
from profile_bind_oracle import PREFERRED
from test_replicas_gpu import _nodes, load
from test_spread_bind_gpu import key_set, mixed_queue
from test_spread_gpu import zone_labels

pytestmark = pytest.mark.gpu

POLICIES = (1, 3, 4)
GPU = "nvidia.com/gpu"
EXTRA = [GPU, "example.com/fpga", "ephemeral-storage", "hugepages-2Mi", "example.com/a", "example.com/b",
         "example.com/c"]


def resources(rng, N, P, R):
    """Name maps for R resources ("pods" and R - 1 others): node allocatable (some names missing, a few nodes without
    "pods"), bound pods (some nodes over-committed), and pod requests (about half zero)."""
    names = EXTRA[:R - 1]
    alloc = []
    for n in range(N):
        a = {} if rng.random() < 0.03 else {"pods": int(rng.integers(0, 12))}
        for nm in names:
            if rng.random() < 0.7:
                a[nm] = int(rng.integers(0, 9))
        alloc.append(a)
    bound = [(int(rng.integers(0, N)), {nm: int(rng.integers(0, 3)) for nm in names if rng.random() < 0.5})
             for _ in range(N // 2)] if N else []
    pod_res = [{nm: int(rng.integers(1, 4)) if rng.random() < 0.5 else 0 for nm in names} for _ in range(P)]
    return alloc, bound, pod_res


def check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, cluster, res, terms=(), ex_pods=None, skew=None,
          mind=None, ex=None, policy=4, with_rules=True, **scoring):
    nl, nt, gr = cluster
    alloc, bound, pod_res = res
    names, free0, req = compile_resources(alloc, bound, pod_res, ["pods"] + [nm for nm in EXTRA if any(
        nm in r for r in pod_res)])
    wt, wn = (3, 2) if with_rules else (0, 0)
    rules = compile_rules(nl, nt, gr, wt, wn) if with_rules else None
    got = snap.fit_bind(rc, rm, sel, group, G, keys, terms, ex_pods, skew, mind, ex, policy, rules=rules,
                        node_free=free0, pod_req=req, **scoring)
    ofc, ofm = fc.copy(), fm.copy()
    want = fit_bind_packed(ofc, ofm, ac, am, lab, rc, rm, sel, group, G, keys, nl if with_rules else [{}] * len(fc),
                           nt if with_rules else [[]] * len(fc), gr if with_rules else [{}] * G, alloc, bound, pod_res,
                           terms, ex_pods, skew, mind, ex, policy, weight_taint=wt, weight_node_affinity=wn, **scoring)
    if not with_rules:  # parts 3 and 4 are 0 without rules, as ks_node_bind's K1
        want[2][:, 3:] = 0
    for i in range(4):
        assert np.array_equal(got[i], want[i]), (i, np.nonzero((got[i] != want[i]).reshape(len(rc), -1))[0][:8])
    for i in (4, 5):
        if got[i] is not None:
            assert all(np.array_equal(a, b) for a, b in zip(got[i], want[i])), i
    assert np.array_equal(got[6], final_free(alloc, want[6], names))
    gfc, gfm = snap.free()
    assert np.array_equal(gfc, ofc) and np.array_equal(gfm, ofm)
    return got


CASES = [  # (W, N, key modes, groups, pods, taints, R)
    (1, 1, (1,), 3, 20, 3, 1),
    (2, 127, (3, "host"), 4, 80, 1, 2),
    (4, 128, (3,), 5, 80, 64, 8),
    (8, 129, ("host",), 3, 60, 0, 3),
    (1, 2100, (3, "host"), 6, 80, 64, 5),
    (2, 3000, (3, 7), 6, 80, 3, 8),
    (4, 16896, (3, "host"), 6, 40, 3, 4),
    (8, 16897, (3,), 6, 40, 64, 6),
]


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("case", CASES, ids=[f"W{c[0]}-N{c[1]}-R{c[6]}" for c in CASES])
def test_against_the_oracle(ks, case, policy):
    W, N, modes, G, P, T, R = case
    rng = np.random.default_rng([W, N, R, policy, 0xF1B])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, modes)
    lab = zone_labels(lab, *keys[0])
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 3000), mem=(0, 12 << 30))
    cluster = random_cluster(rng, N, G, T)
    res = resources(rng, N, P, R)
    terms = [(0, ANTI, len(keys) - 1, [0]), (1, PREFERRED, 0, [2])]
    ex_pods = (np.array([0, 2], np.int32), np.array([0, N - 1], np.int32)) if N > 1 and R % 2 else None
    soft = np.array([0, 1, 3], np.uint32)[rng.integers(0, 3, (G, len(keys)))]
    with ks.Snapshot(0) as snap:
        for with_rules in (True, False):
            load(ks, snap, fc, fm, ac, am, lab)
            got = check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, cluster, res, terms, ex_pods, skew,
                        mind, ex, policy, with_rules, soft_skew=soft, term_weight=[0, 40])
            if N > 1000:
                assert (got[0] >= 0).any() and got[3][:, 0].any()


@pytest.mark.parametrize("policy", POLICIES)
def test_l1_l4_against_node_bind(ks, policy):
    """L1: res NULL is ks_node_bind bit for bit with word 0 = 0.  L4: ample resources (every node_free at least the
    queue's total request) likewise, free_r charged by the requests.  Same launches per call as ks_node_bind with rules,
    one more (k_node_rules_setup) with rules NULL."""
    rng = np.random.default_rng(0xF1B2 + policy)
    N, W, G, P = 3000, 2, 5, 100
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (4, "host"))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 3000), mem=(0, 12 << 30))
    nl, nt, gr = random_cluster(rng, N, G, 3)
    rules = compile_rules(nl, nt, gr)
    terms = [(0, ANTI, 1, [0]), (1, PREFERRED, 0, [1, 2])]
    kw = dict(soft_skew=np.array([0, 1, 3], np.uint32)[rng.integers(0, 3, (G, 2))], term_weight=[0, 50])
    req = rng.integers(0, 4, (P, 3)).astype(np.int64)
    ample = np.tile(req.sum(0)[:, None] + rng.integers(0, 5, (3, N)), 1).astype(np.int64)
    for r in (rules, None):
        with ks.Snapshot(0) as snap:
            load(ks, snap, fc, fm, ac, am, lab)
            n0 = ks.launch_count()
            want = snap.node_bind(rc, rm, sel, group, G, keys, terms, None, skew, mind, ex, policy, rules=r, **kw)
            launches = ks.launch_count() - n0
            want_free = snap.free()
            for node_free, pod_req in ((None, None), (ample, req)):
                load(ks, snap, fc, fm, ac, am, lab)
                n0 = ks.launch_count()
                got = snap.fit_bind(rc, rm, sel, group, G, keys, terms, None, skew, mind, ex, policy, rules=r,
                                    node_free=node_free, pod_req=pod_req, **kw)
                # with rules NULL, ks_node_bind runs ks_profile_bind's walk (K1), which has no k_node_rules_setup
                assert ks.launch_count() - n0 == launches + (r is None)
                assert snap.last_path() == "fit_bind"
                assert all(np.array_equal(a, b) for a, b in zip(snap.free(), want_free))
                assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
                assert np.array_equal(got[2], want[2]) and np.array_equal(got[3][:, 1:], want[3])
                assert not got[3][:, 0].any()
                for i in (4, 5):
                    assert all(np.array_equal(a, b) for a, b in zip(got[i], want[i]))
                if node_free is None:
                    assert got[6].shape == (0, N)
                else:
                    charged = node_free.copy()
                    for p, n in enumerate(got[0]):
                        if n >= 0:
                            charged[:, n] -= pod_req[p]
                    assert np.array_equal(got[6], charged)  # L3


def test_one_node_and_empty_snapshot(ks):
    rng = np.random.default_rng(0xF1B3)
    N, W, G, P = 200, 1, 3, 12
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3,))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P)
    nl, nt, gr = random_cluster(rng, N, G, 3)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac[:0], am[:0], lab[:0])
        got = snap.fit_bind(rc, rm, sel, group, G, [(d[:0], n) for d, n in keys], (), None, skew, None, ex, 4,
                            rules=compile_rules([], [], gr), node_free=np.zeros((2, 0), np.int64),
                            pod_req=np.ones((P, 2), np.int64))
        assert (got[0] == -1).all() and not got[1].any() and not got[2].any() and not got[3].any()
        assert got[6].shape == (2, 0)
        load(ks, snap, fc[:1], fm[:1], ac[:1], am[:1], lab[:1])
        check(snap, fc[:1], fm[:1], ac[:1], am[:1], lab[:1], rc, rm, sel, group, G, [(d[:1], n) for d, n in keys],
              (nl[:1], nt[:1], gr), resources(rng, 1, P, 3), skew=skew, ex=ex, policy=3)
        # no pod: out_free is node_free
        load(ks, snap, fc, fm, ac, am, lab)
        nf = rng.integers(-5, 5, (3, N)).astype(np.int64)
        got = snap.fit_bind(rc[:0], rm[:0], sel[:0], group[:0], G, keys, node_free=nf, pod_req=np.zeros((0, 3), np.int64))
        assert np.array_equal(got[6], nf)


def test_errors_leave_free_unchanged(ks):
    rng = np.random.default_rng(0xF1B4)
    N, W, G, P = 200, 1, 3, 10
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3,))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P)
    neg = np.ones((P, 2), np.int64)
    neg[3, 1] = -1
    bad = [
        (np.zeros((9, N), np.int64), np.zeros((P, 9), np.int64), ks.capi.KS_ERR_RANGE),  # R = 9
        (np.zeros((2, N), np.int64), neg, ks.capi.KS_ERR_RANGE),  # a negative request
    ]
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        for nf, pr, code in bad:
            with pytest.raises(ks.KsError) as e:
                snap.fit_bind(rc, rm, sel, group, G, keys, (), None, skew, node_free=nf, pod_req=pr)
            assert e.value.code == code
            assert all(np.array_equal(a, b) for a, b in zip(snap.free(), (fc, fm)))
        with pytest.raises(ks.KsError) as e:  # every check of ks_node_bind still runs
            snap.fit_bind(rc, rm, sel, group, G, keys, (), None, skew, policy=0, node_free=np.zeros((1, N), np.int64),
                          pod_req=np.ones((P, 1), np.int64))
        assert e.value.code == ks.capi.KS_ERR_INVALID
        # NULL node_free or pod_req with R > 0
        pods, keep = snap._pods(rc, rm, sel)
        d0 = np.zeros(N, np.int32)
        topo = ks.capi.ks_spread_multi(1, (C.c_uint32 * 4)(1), (C.c_void_p * 4)(d0.ctypes.data), None, None, None)
        aff = ks.capi.ks_pod_affinity()
        sc = ks.capi.ks_bind_scoring(None, None, None, 1, 2, 2)
        idx = np.empty(P, np.int32)
        pr, nf = np.ones(P, np.int64), np.zeros(N, np.int64)
        for res in (ks.capi.ks_bind_resources(1, None, pr.ctypes.data), ks.capi.ks_bind_resources(1, nf.ctypes.data,
                                                                                                   None)):
            got = ks.lib.ks_fit_bind(snap._h, C.byref(pods), group.ctypes.data, G, C.byref(topo), C.byref(aff),
                                     C.byref(sc), None, C.byref(res), 4, idx.ctypes.data, None, None, None, None, None,
                                     None)
            assert got == ks.capi.KS_ERR_INVALID
            assert all(np.array_equal(a, b) for a, b in zip(snap.free(), (fc, fm)))


def test_select_after_the_call(ks):
    """ks_select on both paths sees the free[] the call charged (the derived index is rebuilt)."""
    rng = np.random.default_rng(0xF1B5)
    N, W, G, P = 5000, 1, 4, 120
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3,))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(500, 6000), mem=(1 << 30, 16 << 30))
    alloc, bound, pod_res = resources(rng, N, P, 3)
    names, nf, pr = compile_resources(alloc, bound, pod_res, ["pods"] + EXTRA[:2])
    with ks.Snapshot(0) as snap, ks.Snapshot(0) as ref:
        load(ks, snap, fc, fm, ac, am, lab)
        snap.select(rc, rm, sel, policy=ks.KS_SCORE_LEAST_ALLOCATED, flags=ks.KS_SELECT_FORCE_BITPAR)  # builds the index
        got = snap.fit_bind(rc, rm, sel, group, G, keys, (), None, skew, node_free=nf, pod_req=pr)
        assert (got[0] >= 0).sum() > 10
        cfc, cfm = snap.free()
        load(ks, ref, cfc, cfm, ac, am, lab)
        for flags in (ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR):
            a = snap.select(rc, rm, sel, policy=ks.KS_SCORE_LEAST_ALLOCATED, flags=flags)
            b = ref.select(rc, rm, sel, policy=ks.KS_SCORE_LEAST_ALLOCATED, flags=flags)
            assert np.array_equal(a.node_idx, b.node_idx) and np.array_equal(a.score, b.score), flags


def test_reconcile_fit(ks):
    """ksh_reconcile_fit: a GPU pool of two 8-GPU nodes behind a taint, small pods against a pod limit of 3.  The first
    call binds two 4-GPU pods per GPU node and gives the fifth status 8; the pods of the pod-limited group fill their
    nodes.  A second call sees the first call's GPUs and pods."""
    import json
    arena = ks.objects.ObjectArena()
    N = 6
    nodes = [{"name": f"n{i}", "labels": {"kubernetes.io/hostname": f"n{i}"},
              "allocatable": {"cpu": "32", "memory": "68719476736", "pods": "3", **({GPU: "8"} if i >= 4 else {})}}
             for i in range(N)]
    gpu_taint = {"key": "gpu", "value": "true", "effect": "NoSchedule"}
    rules = [{}, {"tolerations": [{"key": "gpu", "operator": "Exists"}]}]
    gpu_pods = [{"name": f"g{i}", "containers": [{"cpu": "1", "memory": "1073741824", GPU: "4"}]} for i in range(5)]
    small = [{"name": f"s{i}", "containers": [{"cpu": "100m", "memory": "1048576"}]} for i in range(4 * 3)]
    pods = gpu_pods + small
    group = np.array([1] * 5 + [0] * 12, np.int32)
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(nodes), N)
        ctx.set_node_taints({"n4": [gpu_taint], "n5": [gpu_taint]})
        names = [ctx.node_name(i) for i in range(N)]
        status, node, bodies = ctx.reconcile_fit(arena.pods(pods), len(pods), group, 2, ["kubernetes.io/hostname"],
                                                 group_rules=rules)
        gpu_nodes = sorted(names[n] for n in node[:5] if n >= 0)
        assert gpu_nodes == ["n4", "n4", "n5", "n5"]
        assert (status[:5] == ks.host.KSH_RECONCILE_OK).sum() == 4
        assert (status[:5] == ks.host.KSH_RECONCILE_INSUFFICIENT_RESOURCES).sum() == 1
        # 4 plain nodes x 3 pods = 12 small pods, none on the tainted GPU nodes
        assert (status[5:] == ks.host.KSH_RECONCILE_OK).all()
        assert all(names[n] in ("n0", "n1", "n2", "n3") for n in node[5:])
        for i in np.nonzero(node >= 0)[0]:
            assert json.loads(bodies[i])["target"]["name"] == names[node[i]]
        more = [{"name": f"h{i}", "containers": [{"cpu": "1", GPU: "1"}]} for i in range(2)] + \
               [{"name": "t0", "containers": [{"cpu": "100m"}]}]
        status2, node2, _ = ctx.reconcile_fit(arena.pods(more), 3, np.array([1, 1, 0], np.int32), 2,
                                              ["kubernetes.io/hostname"], group_rules=rules)
        # every GPU is taken (4 + 4 on each GPU node): status 8 for both GPU pods.  Every plain node holds 3 pods (word 0
        # = 4) and the GPU nodes, with one pod slot left each, refuse t0 by their taint: status 7
        assert (node2 == -1).all()
        assert status2.tolist() == [ks.host.KSH_RECONCILE_INSUFFICIENT_RESOURCES] * 2 + \
            [ks.host.KSH_RECONCILE_NODE_RULES_UNSATISFIED]
        names_r, free_r, _ = ctx.compile_resources(arena.pods(more), 3)
        assert names_r == ["pods", GPU]
        assert sorted(free_r[0].tolist()) == [0, 0, 0, 0, 1, 1] and sorted(free_r[1].tolist()) == [0] * 6
