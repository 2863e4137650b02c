"""Taints and node affinity when binding (ks_node_bind) on the H100: node, total, five parts, four refusals, hard and
soft counts and the final free[] bit for bit against tests/node_bind_oracle.py (which evaluates the rules over strings)
across label widths 1-8, policies 1, 3 and 4, 0, 1, 3 and 64 taints, node counts at the CTA-slice edges, one node and
the empty snapshot; multi-word domain sets on a hostname key; spread eligibility honouring node affinity; classes at
the rule-word cap and one over it; K1 and K2 against ks_profile_bind on the device; host errors leaving free[]
unchanged; and ksh_reconcile_nodes end to end with status 7."""
import numpy as np
import pytest

from affinity_bind_oracle import ANTI
from node_bind_oracle import compile_rules, node_bind_packed, random_cluster
from profile_bind_oracle import ANTI_PREFERRED, PREFERRED
from test_replicas_gpu import _nodes, _specs, load
from test_spread_bind_gpu import key_set, mixed_queue
from test_spread_gpu import zone_labels

pytestmark = pytest.mark.gpu

POLICIES = (1, 3, 4)


def check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, cluster, terms=(), ex_pods=None, skew=None,
          mind=None, ex=None, policy=4, wt=3, wn=2, **scoring):
    nl, nt, gr = cluster
    rules = compile_rules(nl, nt, gr, wt, wn)
    got = snap.node_bind(rc, rm, sel, group, G, keys, terms, ex_pods, skew, mind, ex, policy, rules=rules, **scoring)
    ofc, ofm = fc.copy(), fm.copy()
    want = node_bind_packed(ofc, ofm, ac, am, lab, rc, rm, sel, group, G, keys, nl, nt, gr, terms, ex_pods, skew, mind,
                            ex, policy, weight_taint=wt, weight_node_affinity=wn, **scoring)
    for i in range(4):
        assert np.array_equal(got[i], want[i]), (i, np.nonzero((got[i] != want[i]).reshape(len(rc), -1))[0][:8])
    for i in (4, 5):
        if got[i] is not None:
            assert all(np.array_equal(a, b) for a, b in zip(got[i], want[i])), i
    gfc, gfm = snap.free()
    assert np.array_equal(gfc, ofc) and np.array_equal(gfm, ofm)
    return got


CASES = [  # (W, N, key modes, groups, pods, taints)
    (1, 1, (1,), 3, 20, 3),
    (2, 127, (3, "host"), 4, 80, 1),
    (4, 128, (3,), 5, 80, 64),
    (8, 129, ("host",), 3, 60, 0),
    (1, 2100, (3, "host"), 6, 80, 64),
    (2, 3000, (3, 7), 6, 80, 3),
    (4, 16896, (3, "host"), 6, 40, 3),
    (8, 16897, (3,), 6, 40, 64),
]


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("case", CASES, ids=[f"W{c[0]}-N{c[1]}-T{c[5]}" for c in CASES])
def test_against_the_oracle(ks, case, policy):
    W, N, modes, G, P, T = case
    rng = np.random.default_rng([W, N, T, policy, 0x90D])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, modes)
    lab = zone_labels(lab, *keys[0])
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 3000), mem=(0, 12 << 30))
    cluster = random_cluster(rng, N, G, T)
    terms = [(0, ANTI, len(keys) - 1, [0]), (1, PREFERRED, 0, [2]), (2, ANTI_PREFERRED, 0, [1])]
    soft = np.array([0, 1, 3], np.uint32)[rng.integers(0, 3, (G, len(keys)))]
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got = check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, cluster, terms, None, skew, mind, ex,
                    policy, soft_skew=soft, soft_all_keys=(rng.random(G) < 0.5).astype(np.uint8),
                    term_weight=[0, 40, 70])
    if N > 1000:
        assert (got[0] >= 0).any() and got[3][:, 1].any()
        if T:
            assert got[3][:, 0].any()


def test_honor_spread_eligibility(ks):
    """A zone whose nodes all fail the group's required node affinity is not an eligible domain: with it counted the
    minimum would stay 0 there and block every other zone after one pod each."""
    N, W = 9, 1
    fc = np.full(N, 64000, np.int64)
    fm = np.full(N, 256 << 30, np.int64)
    ac, am = fc.copy(), fm.copy()
    lab = np.zeros((N, W), np.uint64)
    zone = np.arange(N, dtype=np.int32) // 3
    keys = [(zone, 3)]
    nl = [{"zone": f"z{z}", "pool": "drain" if z == 2 else "live"} for z in zone]
    nt = [[] for _ in range(N)]
    gr = [{"required": [[{"key": "pool", "operator": "NotIn", "values": ["drain"]}]]}]
    P = 6
    group = np.zeros(P, np.int32)
    rc, rm = np.full(P, 100, np.int64), np.full(P, 1 << 20, np.int64)
    sel = np.zeros((P, W), np.uint64)
    skew = np.ones((1, 1), np.uint32)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got = check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, 1, keys, (nl, nt, gr), skew=skew)
    assert (got[0] >= 0).all() and (zone[got[0]] < 2).all()


def test_rule_word_cap(ks):
    """4 096 classes x 16 384 nodes is exactly 2^26 rule words; one group more is KS_ERR_RANGE before free[] changes.
    The pods use groups 0-3 only, so the oracle runs on those four groups."""
    rng = np.random.default_rng(0x90D1)
    N, W, P = 16384, 1, 40
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3,))
    nl, nt, _ = random_cluster(rng, N, 4, 3)
    for i in range(12):  # 12 further NoSchedule taints: 4 095 distinct toleration masks
        nt[int(rng.integers(0, N))].append({"key": f"k{i}", "value": "", "effect": "NoSchedule"})
    names = [f"k{i}" for i in range(12)]

    def groups(G):
        return [{"tolerations": [{"key": names[i], "operator": "Exists"} for i in range(12) if (g + 1) >> i & 1],
                 "preferred": [(g % 100 + 1, [{"key": "zone", "operator": "In", "values": ["z0"]}])]}
                for g in range(G)]
    group = rng.integers(-1, 4, P).astype(np.int32)
    rc, rm, sel = _specs(rng, P, W, cpu=(0, 3000), mem=(0, 8 << 30))
    sel[:] = 0
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        gr = groups(4095)
        rules = compile_rules(nl, nt, gr)
        got = snap.node_bind(rc, rm, sel, group, 4095, keys, rules=rules, want_counts=False)
        ofc, ofm = fc.copy(), fm.copy()
        want = node_bind_packed(ofc, ofm, ac, am, lab, rc, rm, sel, group, 4, keys, nl, nt, gr[:4])
        assert all(np.array_equal(a, b) for a, b in zip(got[:4], want[:4]))
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), (ofc, ofm)))
        load(ks, snap, fc, fm, ac, am, lab)
        with pytest.raises(ks.KsError) as e:
            snap.node_bind(rc, rm, sel, group, 4096, keys, rules=compile_rules(nl, nt, groups(4096)),
                           want_counts=False)
        assert e.value.code == ks.capi.KS_ERR_RANGE
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), (fc, fm)))


@pytest.mark.parametrize("policy", POLICIES)
def test_k1_k2_against_profile_bind(ks, policy):
    """K1: rules None is ks_profile_bind with zero refusal words 0-1 and parts 3-4.  K2: no taint and no node-affinity
    term binds the same nodes, every score 100 * weight_taint higher, tt = 100 and na = 0 on every bound pod."""
    rng = np.random.default_rng(0x90D2 + policy)
    N, W, G, P = 3000, 2, 5, 100
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (4, "host"))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 3000), mem=(0, 12 << 30))
    terms = [(0, ANTI, 1, [0]), (1, PREFERRED, 0, [1, 2])]
    soft = np.array([0, 1, 3], np.uint32)[rng.integers(0, 3, (G, 2))]
    kw = dict(soft_skew=soft, term_weight=[0, 50])
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        want = snap.profile_bind(rc, rm, sel, group, G, keys, terms, None, skew, mind, ex, policy, **kw)
        want_free = snap.free()
        load(ks, snap, fc, fm, ac, am, lab)
        k1 = snap.node_bind(rc, rm, sel, group, G, keys, terms, None, skew, mind, ex, policy, **kw)
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), want_free))
        load(ks, snap, fc, fm, ac, am, lab)
        k2 = snap.node_bind(rc, rm, sel, group, G, keys, terms, None, skew, mind, ex, policy,
                            rules=dict(tolerate_hard=np.zeros(G, np.uint64), weight_taint=3), **kw)
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), want_free))
    for got in (k1, k2):
        assert np.array_equal(got[0], want[0])
        assert np.array_equal(got[2][:, :3], want[2])
        assert np.array_equal(got[3][:, 2:], want[3]) and not got[3][:, :2].any()
        for i in (4, 5):
            assert all(np.array_equal(a, b) for a, b in zip(got[i], want[i]))
    assert np.array_equal(k1[1], want[1]) and not k1[2][:, 3:].any()
    bound = want[0] >= 0
    assert np.array_equal(k2[1], want[1] + 300 * bound)
    assert (k2[2][bound, 3] == 100).all() and not k2[2][:, 4].any()


def test_one_node_and_empty_snapshot(ks):
    rng = np.random.default_rng(0x90D3)
    N, W, G, P = 200, 1, 3, 12
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3,))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P)
    nl, nt, gr = random_cluster(rng, N, G, 3)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac[:0], am[:0], lab[:0])
        got = snap.node_bind(rc, rm, sel, group, G, [(d[:0], n) for d, n in keys], (), None, skew, None, ex, 4,
                             rules=compile_rules([], [], gr))
        assert (got[0] == -1).all() and not got[1].any() and not got[2].any() and not got[3].any()
        assert all(np.array_equal(a, np.asarray(b, np.uint32)) for a, b in zip(got[4], ex))
        load(ks, snap, fc[:1], fm[:1], ac[:1], am[:1], lab[:1])
        check(snap, fc[:1], fm[:1], ac[:1], am[:1], lab[:1], rc, rm, sel, group, G, [(d[:1], n) for d, n in keys],
              (nl[:1], nt[:1], gr), skew=skew, ex=ex, policy=3)


def test_errors_leave_free_unchanged(ks):
    rng = np.random.default_rng(0x90D4)
    N, W, G, P = 200, 1, 3, 10
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3,))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P)
    dom = (np.arange(N) % 4).astype(np.int32)
    ok_set = np.array([0b1], np.uint64)
    bad = [
        (dict(weight_taint=101), ks.capi.KS_ERR_INVALID),
        (dict(weight_node_affinity=101), ks.capi.KS_ERR_INVALID),
        (dict(n_taints=65), ks.capi.KS_ERR_RANGE),
        (dict(n_taints=2, taint_hard=np.full(N, 4, np.uint64)), ks.capi.KS_ERR_INVALID),
        (dict(n_taints=2, tolerate_soft=np.full(G, 8, np.uint64)), ks.capi.KS_ERR_INVALID),
        (dict(rule_keys=[(dom, 4)] * 17), None),  # refused by the Python layer
        (dict(rule_keys=[(dom, 3)]), ks.capi.KS_ERR_INVALID),  # a domain outside [-1, D)
        (dict(rule_keys=[(dom, 4)], node_terms=[(0, 0, [(1, ok_set)])]), ks.capi.KS_ERR_INVALID),  # key 1 of 1
        (dict(rule_keys=[(dom, 4)], node_terms=[(0, 0, [(0, np.array([1 << 5], np.uint64))])]),
         ks.capi.KS_ERR_INVALID),  # a bit above D
        (dict(rule_keys=[(dom, 4)], node_terms=[(0, 0, [(0, np.array([1, 0], np.uint64))])]),
         ks.capi.KS_ERR_INVALID),  # two words for five bits
        (dict(rule_keys=[(dom, 4)], node_terms=[(3, 0, [(0, ok_set)])]), ks.capi.KS_ERR_INVALID),  # owner
        (dict(rule_keys=[(dom, 4)], node_terms=[(0, 101, [(0, ok_set)])]), ks.capi.KS_ERR_INVALID),  # weight
        (dict(rule_keys=[(dom, 4)], node_terms=[(0, 1, [(0, ok_set)])] * 4097), ks.capi.KS_ERR_RANGE),
    ]
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        for rules, code in bad:
            if code is None:
                with pytest.raises(ValueError):
                    snap.node_bind(rc, rm, sel, group, G, keys, (), None, skew, rules=rules)
                continue
            with pytest.raises(ks.KsError) as e:
                snap.node_bind(rc, rm, sel, group, G, keys, (), None, skew, rules=rules)
            assert e.value.code == code, rules
            got = snap.free()
            assert np.array_equal(got[0], fc) and np.array_equal(got[1], fm), rules
        with pytest.raises(ks.KsError) as e:  # every check of ks_profile_bind still runs
            snap.node_bind(rc, rm, sel, group, G, keys, (), None, skew, policy=0, rules={})
        assert e.value.code == ks.capi.KS_ERR_INVALID


def test_hostname_sets(ks):
    """Expression sets of several words: In / NotIn / DoesNotExist over a hostname key of 299 domains (five words), the
    absent bit in the last word, the preferred raw from a set bit above 64."""
    rng = np.random.default_rng(0x90D5)
    N, W, G, P = 300, 1, 4, 60
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3,))
    nl = [{"host": f"h{n}"} if n != 250 else {} for n in range(N)]
    nt = [[] for _ in range(N)]
    gr = [{"required": [[{"key": "host", "operator": "In", "values": [f"h{n}" for n in range(60, 300, 7)]}]]},
          {"required": [[{"key": "host", "operator": "NotIn", "values": [f"h{n}" for n in range(0, 290)]}]]},
          {"required": [[{"key": "host", "operator": "DoesNotExist"}], [{"key": "host", "operator": "In",
                                                                         "values": ["h199", "h64", "h128"]}]]},
          {"preferred": [(90, [{"key": "host", "operator": "In", "values": ["h201", "h130"]}]),
                         (10, [{"key": "host", "operator": "NotIn", "values": ["h201"]}])]}]
    group = rng.integers(0, G, P).astype(np.int32)
    rc, rm, _ = _specs(rng, P, W, cpu=(0, 1000), mem=(0, 2 << 30))
    sel = np.zeros((P, W), np.uint64)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got = check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, (nl, nt, gr), policy=1)
    assert set(got[0][group == 1].tolist()) <= {250, -1} | set(range(290, 300))
    assert set(got[0][group == 2].tolist()) <= {250, 199, 64, 128, -1} and (got[0] >= 0).sum() > P // 2


def test_null_and_cap_errors(ks):
    """The host checks of the packed rules that Snapshot.node_bind cannot express: NULL arrays, decreasing term offsets
    and set words beyond 2^26, each KS_ERR_INVALID / KS_ERR_RANGE before free[] changes."""
    import ctypes as C
    from importlib import import_module
    smod = import_module(ks.Snapshot.__module__)
    rng = np.random.default_rng(0x90D6)
    N, W, G, P = 100, 1, 2, 4
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    dom = (np.arange(N) % 4).astype(np.int32)
    base = dict(rule_keys=[(dom, 4)], node_terms=[(0, 0, [(0, smod.node_set(4, [1]))]), (1, 5, [])])

    def mutate(nr, field, value):
        setattr(nr, field, value)

    cases = [
        (lambda nr: nr.node_domain.__setitem__(0, None), ks.capi.KS_ERR_INVALID),
        (lambda nr: mutate(nr, "expr_key", None), ks.capi.KS_ERR_INVALID),
        (lambda nr: mutate(nr, "expr_set", None), ks.capi.KS_ERR_INVALID),
        (lambda nr: mutate(nr, "term_owner", None), ks.capi.KS_ERR_INVALID),
        (lambda nr: mutate(nr, "term_expr_offset", C.addressof(dec)), ks.capi.KS_ERR_INVALID),
        (lambda nr: mutate(nr, "expr_set_offset", C.addressof(far)), ks.capi.KS_ERR_RANGE),
    ]
    dec = (C.c_uint32 * 3)(1, 0, 1)  # term 0: offsets decrease
    far = (C.c_uint64 * 2)(1 << 26, (1 << 26) + 1)  # one word, past 2^26
    rc, rm = np.full(P, 100, np.int64), np.full(P, 1 << 20, np.int64)
    sel = np.zeros((P, W), np.uint64)
    group = np.array([0, 1, -1, 0], np.int32)
    keys = [(np.zeros(N, np.int32), 1)]
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        snap.node_bind(rc, rm, sel, group, G, keys, rules=base)  # the base rules are valid
        load(ks, snap, fc, fm, ac, am, lab)
        for change, code in cases:
            nr, hold = smod.node_rules(base)
            change(nr)
            pods, keep = snap._pods(rc, rm, sel)
            d0 = np.zeros(N, np.int32)
            topo = ks.capi.ks_spread_multi(1, (C.c_uint32 * 4)(1), (C.c_void_p * 4)(d0.ctypes.data), None, None, None)
            aff = ks.capi.ks_pod_affinity()
            sc = ks.capi.ks_bind_scoring(None, None, None, 1, 2, 2)
            idx = np.empty(P, np.int32)
            got = ks.lib.ks_node_bind(snap._h, C.byref(pods), group.ctypes.data, G, C.byref(topo), C.byref(aff),
                                      C.byref(sc), C.byref(nr), 4, idx.ctypes.data, None, None, None, None, None)
            assert got == code, (ks.lib.ks_last_error().decode(), code)
            f = snap.free()
            assert np.array_equal(f[0], fc) and np.array_equal(f[1], fm)


def test_reconcile_nodes(ks):
    """ksh_reconcile_nodes equals ks_node_bind on the packed arrays with the same rules, statuses included: a group
    whose required affinity no node passes gets status 7, and the ordinary pods avoid the tainted nodes."""
    import json
    arena = ks.objects.ObjectArena()
    N = 12
    nodes = [{"name": f"n{i}", "labels": {"zone": f"z{i % 3}", "kubernetes.io/hostname": f"n{i}",
                                          "type": ["m5", "c5", "g4"][i // 4]},
              "allocatable": {"cpu": "4", "memory": "8589934592"}} for i in range(N)]
    taints = {"n0": [CP_TAINT], "n8": [GPU], "n9": [GPU], "n5": [SPOT]}
    rules = [{},  # ordinary pods
             {"tolerations": [{"key": "gpu", "operator": "Exists"}],
              "required": [[{"key": "type", "operator": "In", "values": ["g4"]}]]},
             {"required": [[{"key": "zone", "operator": "In", "values": ["z9"]}]]},  # nowhere: status 7
             {"preferred": [(80, [{"key": "zone", "operator": "NotIn", "values": ["z0"]}])],
              "tolerations": [{"operator": "Exists", "effect": "PreferNoSchedule"}]}]
    P = 16
    group = np.array([i % 4 for i in range(P)], np.int32)
    pods = [{"name": f"p{i}", "containers": [{"cpu": "500m", "memory": "536870912"}]} for i in range(P)]
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(nodes), N)
        ctx.set_node_taints(taints)
        names = [ctx.node_name(i) for i in range(N)]
        hdom, hval = ctx.topology_domains("kubernetes.io/hostname")
        ac, am, lab, bn, bc, bm = ctx.export_packed()
        rc, rm, sel = ctx.pack_pods(arena.pods(pods), P)
        nl = [nodes[int(names[i][1:])]["labels"] for i in range(N)]
        nt = [taints.get(names[i], []) for i in range(N)]
        soft = np.tile([0], (4, 1)).astype(np.uint32)
        with ks.Snapshot(0) as s:
            s.set_nodes(ac, am, lab)
            s.set_bound(bn, bc, bm)
            want = s.node_bind(rc, rm, sel, group, 4, [(hdom, len(hval))], max_skew=None, soft_skew=soft,
                               rules=compile_rules(nl, nt, rules))
        status, node, bodies = ctx.reconcile_nodes(arena.pods(pods), P, group, 4, ["kubernetes.io/hostname"],
                                                   soft_skew=soft, group_rules=rules)
    assert np.array_equal(node, want[0])
    for i in range(P):
        if want[0][i] >= 0:
            assert status[i] == ks.host.KSH_RECONCILE_OK and json.loads(bodies[i])["target"]["name"] == names[node[i]]
        elif want[3][i, :2].any() and not want[3][i, 2:].any():
            assert status[i] == ks.host.KSH_RECONCILE_NODE_RULES_UNSATISFIED
    assert (status[group == 2] == ks.host.KSH_RECONCILE_NODE_RULES_UNSATISFIED).all()
    bound0 = [names[n] for n in node[group == 0]]
    assert "n0" not in bound0 and "n8" not in bound0 and "n9" not in bound0
    assert set(names[n] for n in node[group == 1]) <= {"n8", "n9", "n10", "n11"}


CP_TAINT = {"key": "node-role.kubernetes.io/control-plane", "value": "", "effect": "NoSchedule"}
GPU = {"key": "gpu", "value": "true", "effect": "NoSchedule"}
SPOT = {"key": "spot", "value": "", "effect": "PreferNoSchedule"}
