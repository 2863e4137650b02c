"""Inter-pod affinity when binding (ks_affinity_bind) on the H100: nodes, scores, both refusals, counts and the final
free[] bit for bit against tests/affinity_bind_oracle.py across label widths, policies, 1 to 4 keys, node counts at the
CTA-slice edges, one node and the empty snapshot, existing pods, duplicate terms, both term kinds on one key, 4 096
groups and 150 000 nodes; identities I1-I4 of include/ksched.h against the existing device calls; every error code
leaving free[] unchanged; a following ks_select on both kernel paths; and the host layer (ksh_reconcile_affinity)."""
import ctypes as C
import json

import numpy as np
import pytest

from affinity_bind_oracle import AFFINITY, ANTI, affinity_bind_packed
from test_replicas_gpu import _nodes, _specs, load
from test_spread_bind_gpu import key_set, mixed_queue
from test_spread_gpu import D_SEED, _gv1_zoned, zone_labels

pytestmark = pytest.mark.gpu

ZONE, HOST = "topology.kubernetes.io/zone", "kubernetes.io/hostname"
POLICIES = (0, 1, 3, 4)


def check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms, ex_pods=None, skew=None, mind=None, ex=None,
          policy=0):
    got = snap.affinity_bind(rc, rm, sel, group, G, keys, terms, ex_pods, skew, mind, ex, policy)
    ofc, ofm = fc.copy(), fm.copy()
    want = affinity_bind_packed(ofc, ofm, ac, am, lab, rc, rm, sel, group, G, keys, terms, ex_pods, skew, mind, ex,
                                policy)
    for i in range(3):
        assert np.array_equal(got[i], want[i]), (i, np.nonzero((got[i] != want[i]).reshape(len(rc), -1))[0][:8])
    if got[3] is not None:
        for a, b in zip(got[3], want[3]):
            assert np.array_equal(a, b)
    gfc, gfm = snap.free()
    assert np.array_equal(gfc, ofc) and np.array_equal(gfm, ofm)
    return got, (ofc, ofm)


def random_terms(rng, G, K, T, hot=4):
    """T terms over G groups, most of them among the first `hot` groups (so they meet in the queue); both kinds, self
    and cross targets, and one exact duplicate and one both-kinds-on-one-key pair."""
    terms = []
    for _ in range(T):
        owner = int(rng.integers(0, min(G, hot))) if rng.random() < 0.8 else int(rng.integers(0, G))
        kind = ANTI if rng.random() < 0.6 else AFFINITY
        tg = sorted(set(rng.integers(0, min(G, hot), int(rng.integers(1, 3))).tolist()))
        if kind == AFFINITY and rng.random() < 0.5:
            tg = sorted(set(tg) | {owner})  # self-affine: the first-pod rule
        terms.append((owner, kind, int(rng.integers(0, K)), tg))
    if terms:
        terms.append(terms[0])  # duplicate term
        o, _, k, tg = terms[0]
        terms.append((o, AFFINITY if terms[0][1] == ANTI else ANTI, k, tg))  # both kinds on one key
    return terms


CASES = [  # (W, N, key modes, groups, pods, terms)
    (1, 1, (1,), 3, 20, 3),
    (2, 127, (3, "host"), 4, 120, 5),
    (4, 128, (3,), 5, 120, 6),
    (8, 129, ("host",), 3, 100, 4),
    (1, 1000, (3, "host"), 8, 200, 8),
    (2, 2100, ("edge", "host"), 6, 150, 6),
    (4, 3000, (3, 7, "host"), 6, 150, 8),
    (8, 16896, (7, 3, 5, "host"), 6, 80, 8),
    (1, 16897, (3,), 6, 80, 5),
]


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("case", CASES, ids=[f"W{c[0]}-N{c[1]}-" + "+".join(map(str, c[2])) for c in CASES])
def test_against_the_oracle(ks, case, policy):
    W, N, modes, G, P, T = case
    rng = np.random.default_rng([W, N, len(modes), policy, 0xAF] + [D_SEED.get(str(m), 5) for m in modes])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, modes)
    lab = zone_labels(lab, *keys[0])
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 3000), mem=(0, 12 << 30))
    terms = random_terms(rng, G, len(keys), T)
    E = int(rng.integers(0, 2 * G + 1))
    ex_pods = (rng.integers(0, G, E), rng.integers(0, N, E))
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got, _ = check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms, ex_pods, skew, mind, ex, policy)
        load(ks, snap, fc, fm, ac, am, lab)  # no spread, no existing pods
        check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms, None, None, None, None, policy)
    if N > 1:
        assert (got[0] >= 0).any() and got[2][:, 1].any(), "some pods placed, some nodes refused by affinity"


def test_many_groups(ks):
    """4 096 groups, terms among far-apart groups, existing pods of many groups: the update lists and counter bases of
    groups at the top of the range."""
    rng = np.random.default_rng(0xAF10)
    N, W, G, P = 400, 2, 4096, 150
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (5, "host"))
    hot = rng.choice(G, 12, replace=False)
    group = hot[rng.integers(0, 12, P)].astype(np.int32)
    group[rng.random(P) < 0.1] = -1
    rc, rm, _ = _specs(rng, P, W, cpu=(0, 3000), mem=(0, 8 << 30))
    sel = np.zeros((P, W), np.uint64)
    terms = [(int(hot[i]), ANTI if i % 3 else AFFINITY, i % 2, [int(hot[(i + 1) % 12]), int(hot[i])]) for i in range(12)]
    terms += [(int(g), ANTI, 1, [int(g)]) for g in rng.choice(G, 50)]
    ex_pods = (rng.integers(0, G, 300), rng.integers(0, N, 300))
    for policy in (0, 4):
        with ks.Snapshot(0) as snap:
            load(ks, snap, fc, fm, ac, am, lab)
            got, _ = check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms, ex_pods, policy=policy)
            assert (got[0] >= 0).any() and got[2][:, 1].any()


def test_150k_nodes(ks):
    rng = np.random.default_rng(0xAF11)
    N, W, G, P = 150_000, 1, 6, 40
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3, "host"))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P)
    terms = [(0, ANTI, 1, [0]), (1, AFFINITY, 0, [0]), (2, ANTI, 0, [3]), (4, AFFINITY, 0, [4])]
    ex_pods = (np.array([0, 3, 0]), np.array([5, 149_999, 77_777]))
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms, ex_pods, skew, None, ex, 1)


@pytest.mark.parametrize("policy", POLICIES)
def test_identities(ks, policy):
    """I1: no terms = ks_spread_bind (spread refusals, counts, free[]), no affinity refusal.  I2: no terms and no
    spread = ks_gang_bind with singletons.  I4: g anti h = h anti g."""
    rng = np.random.default_rng(0xAF12 + policy)
    N, W, G, P = 3000, 2, 5, 500
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3, "host"))
    lab = zone_labels(lab, *keys[0])
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        want = snap.spread_bind(rc, rm, sel, group, keys, skew, mind, ex, policy)
        wfree = snap.free()
        load(ks, snap, fc, fm, ac, am, lab)
        got = snap.affinity_bind(rc, rm, sel, group, G, keys, [], None, skew, mind, ex, policy)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert np.array_equal(got[2][:, 0], want[2]) and not got[2][:, 1].any()
        assert all(np.array_equal(a, b) for a, b in zip(got[3], want[3]))
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), wfree))
        load(ks, snap, fc, fm, ac, am, lab)
        want = snap.gang_bind(rc, rm, sel, np.arange(P + 1), np.zeros(P), policy) + snap.free()
        load(ks, snap, fc, fm, ac, am, lab)
        got = snap.affinity_bind(rc, rm, sel, group, G, keys, policy=policy)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and not got[2].any()
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), want[4:]))
        ex_pods = (np.array([0, 1, 2]), np.array([10, 20, 30]))
        runs = []
        for term in ((0, ANTI, 0, [1]), (1, ANTI, 0, [0])):
            load(ks, snap, fc, fm, ac, am, lab)
            runs.append(snap.affinity_bind(rc, rm, sel, group, G, keys, [term, (2, ANTI, 1, [2])], ex_pods, skew, mind,
                                           ex, policy) + snap.free())
        for a, b in zip(runs[0], runs[1]):
            assert all(np.array_equal(x, y) for x, y in zip(a, b)) if isinstance(a, list) else np.array_equal(a, b)
        assert runs[0][2][:, 1].any()


@pytest.mark.parametrize("policy", POLICIES)
def test_self_anti_affinity_is_the_replica_prefix(ks, policy):
    """I3: one group of R identical pods, anti-affine to itself on a key every node carries: the prefix of
    ks_place_replicas_spread's copy list (max_skew 1) up to the first copy whose domain holds one, the rest unbound."""
    rng = np.random.default_rng(0xAF13 + policy)
    N, W, R = 2500, 1, 900
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    for dom, D in ((np.arange(N, dtype=np.int32), N), (rng.integers(0, 40, N).astype(np.int32), 40)):
        rc, rm, sel = _specs(rng, 1, W, cpu=(500, 3000), mem=(1 << 30, 8 << 30), sel_p=0.5)
        with ks.Snapshot(0) as snap:
            load(ks, snap, fc, fm, ac, am, lab)
            plan = snap.place_replicas_spread(rc, rm, sel, [R], dom, D, [1], [0], None, policy)
            node, score = plan[1], plan[2]
            seen, cut = set(), len(node)
            for i, n in enumerate(node):
                if n < 0 or dom[n] in seen:
                    cut = i
                    break
                seen.add(dom[n])
            load(ks, snap, fc, fm, ac, am, lab)
            got = snap.affinity_bind(np.repeat(rc, R), np.repeat(rm, R), np.repeat(sel, R, axis=0), np.zeros(R), 1,
                                     [(dom, D)], [(0, ANTI, 0, [0])], policy=policy)
            assert np.array_equal(got[0][:cut], node[:cut]) and np.array_equal(got[1][:cut], score[:cut])
            assert (got[0][cut:] == -1).all() and cut > 0


def test_following_select_sees_the_charges(ks, orc):
    rng = np.random.default_rng(0xAF14)
    N, W = 4000, 1
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3, "host"))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, 6, 500, cpu=(1000, 9000), mem=(4 << 30, 40 << 30))
    terms = random_terms(rng, 6, 2, 6)
    qc, qm, qs = _specs(rng, 300, W)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        snap.select(qc, qm, qs, policy=0, flags=ks.KS_SELECT_FORCE_BITPAR)  # builds the index before the call
        _, (ofc, ofm) = check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, 6, keys, terms, None, skew, mind, ex, 0)
        for policy in (0, 1):
            widx, wscore = orc.run_packed(ofc, ofm, ac, am, lab, qc, qm, qs, policy=policy, want_mask=False)[:2]
            for flags in (ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR):
                r = snap.select(qc, qm, qs, policy=policy, flags=flags)
                assert np.array_equal(r.node_idx, widx) and np.array_equal(r.score, wscore), (policy, r.path)


def test_errors_leave_free_unchanged(ks):
    rng = np.random.default_rng(0xAF15)
    N, W, G = 300, 1, 3
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3, "host"))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, 50)
    terms = [(0, ANTI, 1, [0]), (1, AFFINITY, 0, [0, 1])]
    ex_pods = (np.array([0, 1]), np.array([3, 4]))
    E_INV, E_RANGE = ks.capi.KS_ERR_INVALID, ks.capi.KS_ERR_RANGE

    def call(snap, terms=terms, ex_pods=ex_pods, G=G, skew=skew, rc=rc, policy=0, keys=keys):
        with pytest.raises(ks.KsError) as e:
            snap.affinity_bind(rc, rm, sel, group, G, keys, terms, ex_pods, skew, None, None, policy)
        return e.value.code

    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        before = snap.free()
        assert call(snap, terms=[(3, ANTI, 0, [0])]) == E_INV        # owner out of range
        assert call(snap, terms=[(-1, ANTI, 0, [0])]) == E_INV
        assert call(snap, terms=[(0, ANTI, 0, [3])]) == E_INV        # target out of range
        assert call(snap, terms=[(0, 2, 0, [0])]) == E_INV           # kind
        assert call(snap, terms=[(0, ANTI, 2, [0])]) == E_INV        # key >= K
        assert call(snap, ex_pods=([3], [0])) == E_INV               # existing group
        assert call(snap, ex_pods=([0], [N])) == E_INV               # existing node
        assert call(snap, ex_pods=([0], [-1])) == E_INV
        assert call(snap, policy=2) == E_INV
        big = rc.copy()
        big[7] = (1 << 36) + 1
        assert call(snap, rc=big) == E_RANGE
        T = ks.capi.KS_AFFINITY_MAX_TERMS + 1
        assert call(snap, terms=[(0, ANTI, 0, [0])] * T) == E_RANGE
        assert call(snap, terms=[(0, ANTI, 0, np.zeros(1 << 22, np.int32)), (0, ANTI, 0, [0])]) == E_RANGE
        # counters: 60 groups with a B and an A array on a key of 2^20 domains, 120 * 2^20 words > 2^26
        wide = [(np.arange(N, dtype=np.int32) % 1000, 1 << 20)]
        assert call(snap, keys=wide, terms=[(g, kd, 0, [g]) for g in range(60) for kd in (ANTI, AFFINITY)],
                    ex_pods=None, G=60, skew=None) == E_RANGE
        # raw struct: decreasing offsets, NULL arrays, too many existing pods
        pods = ks.capi.ks_pods(len(rc), rc.ctypes.data, rm.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
        idx = np.empty(len(rc), np.int32)
        topo = ks.capi.ks_spread_multi(1, (C.c_uint32 * 4)(keys[0][1]), (C.c_void_p * 4)(keys[0][0].ctypes.data), None,
                                       None, None)
        g32 = np.ascontiguousarray(group, np.int32)
        own, kind, key = np.zeros(2, np.int32), np.ones(2, np.uint8), np.zeros(2, np.uint32)
        off, tgt = np.array([0, 2, 1], np.uint64), np.zeros(2, np.int32)

        def raw(aff):
            return ks.lib.ks_affinity_bind(snap._h, C.byref(pods), g32.ctypes.data, G, C.byref(topo), C.byref(aff), 0,
                                           idx.ctypes.data, None, None, None)

        assert raw(ks.capi.ks_pod_affinity(2, own.ctypes.data, kind.ctypes.data, key.ctypes.data, off.ctypes.data,
                                           tgt.ctypes.data, 0, None, None)) == E_INV
        assert raw(ks.capi.ks_pod_affinity(1, own.ctypes.data, None, key.ctypes.data, off.ctypes.data,
                                           tgt.ctypes.data, 0, None, None)) == E_INV
        assert raw(ks.capi.ks_pod_affinity(0, None, None, None, None, None, 1, None, None)) == E_INV
        assert raw(ks.capi.ks_pod_affinity(0, None, None, None, None, None, (1 << 24) + 1, own.ctypes.data,
                                           own.ctypes.data)) == E_RANGE
        after = snap.free()
        assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])


def test_one_node_and_empty_snapshot(ks):
    with ks.Snapshot(0) as snap:
        snap.set_nodes(np.zeros(0), np.zeros(0), np.zeros((0, 1)))
        got = snap.affinity_bind([1, 0, 5], [1, 0, 5], np.zeros((3, 1)), [0, -1, 1], 2, [(np.zeros(0, np.int32), 3)],
                                 [(0, ANTI, 0, [0, 1])], None, [[1], [0]])
        assert (got[0] == -1).all() and (got[1] == 0).all() and not got[2].any()
    rng = np.random.default_rng(0xAF16)
    fc, fm, ac, am, lab = _nodes(rng, 1, 1)
    rc, rm, sel = _specs(rng, 6, 1, cpu=(0, 0), mem=(0, 0), sel_p=0)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got, _ = check(snap, fc, fm, ac, am, lab, rc, rm, sel, [0, 0, 1, 1, 2, -1], 3, [(np.zeros(1, np.int32), 1)],
                       [(0, ANTI, 0, [0]), (2, AFFINITY, 0, [1])])
        assert got[0].tolist()[:2] == [0, -1]


def _objects(g, nodes):
    nodes = [dict(nd, labels=dict(nd["labels"], **{HOST: nd["name"]})) for nd in nodes]
    pods = []
    for i in range(12):
        base = g["pods"][1] if i % 3 else g["pods"][2]  # 500m / 1 GiB, and 1500m / 3 GiB
        pods.append(dict(base, name=f"w{i % 3}-{i}", ns="apps"))
    pods[4] = dict(pods[4], node_name="n0")  # already bound: skipped
    pods[7] = dict(pods[7], ns=None)           # no namespace: no Binding
    return nodes, pods


def test_host_layer(ks):
    """ksh_reconcile_affinity equals ks_affinity_bind on the packed arrays over the pods that go to the device;
    statuses (SPREAD_UNSATISFIED before AFFINITY_UNSATISFIED before NO_NODE_FOUND), Binding bodies, the bound list and
    the charged snapshot; an existing pod on a node not in the store is skipped."""
    g, nodes = _gv1_zoned()
    nodes, objs = _objects(g, nodes)
    group = np.array([i % 3 for i in range(12)], np.int32)
    skew = np.array([[1, 0], [0, 0], [0, 0]], np.uint32)  # workload 0: zone spread
    terms = [(0, ANTI, 1, [0]), (1, ANTI, 1, [1]), (2, AFFINITY, 0, [0])]  # workload 1: held off n0-n3 below
    arena = ks.objects.ObjectArena()
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(nodes), len(nodes))
        names = [ctx.node_name(i) for i in range(ctx.n_nodes)]
        existing_pods = [(1, names[n]) for n in range(4)] + [(0, "no-such-node")]
        zdom, zval = ctx.topology_domains(ZONE)
        hdom, hval = ctx.topology_domains(HOST)
        keys = [(zdom, len(zval)), (hdom, len(hval))]
        ac, am, lab, bn, bc, bm = ctx.export_packed()
        todo = [i for i in range(12) if i not in (4, 7)]
        rc, rm, sel = ctx.pack_pods(arena.pods([objs[i] for i in todo]), len(todo))
        with ks.Snapshot(0) as s:
            s.set_nodes(ac, am, lab)
            s.set_bound(bn, bc, bm)
            want = s.affinity_bind(rc, rm, sel, group[todo], 3, keys, terms, ([1] * 4, list(range(4))), skew)
            want_free = s.free()
        bound0 = ctx.num_bound
        status, node, bodies = ctx.reconcile_affinity(arena.pods(objs), 12, group, 3, [ZONE, HOST], terms,
                                                      existing_pods, skew)
        assert status[4] == ks.host.KSH_RECONCILE_OK and node[4] == -1 and bodies[4] is None
        assert status[7] == ks.host.KSH_RECONCILE_BINDING_OBJECT_FAILED and node[7] == -1
        assert np.array_equal(node[todo], want[0])
        for k, i in enumerate(todo):
            if want[0][k] >= 0:
                assert status[i] == ks.host.KSH_RECONCILE_OK
                body = json.loads(bodies[i])
                assert body["kind"] == "Binding" and body["target"]["name"] == names[want[0][k]]
                assert body["metadata"]["name"] == objs[i]["name"]
            elif want[2][k, 0] > 0:
                assert status[i] == ks.host.KSH_RECONCILE_SPREAD_UNSATISFIED and bodies[i] is None
            elif want[2][k, 1] > 0:
                assert status[i] == ks.host.KSH_RECONCILE_AFFINITY_UNSATISFIED and bodies[i] is None
            else:
                assert status[i] == ks.host.KSH_RECONCILE_NO_NODE_FOUND and bodies[i] is None
        placed = int((want[0] >= 0).sum())
        assert ctx.num_bound == bound0 + placed and placed > 0
        assert (status == ks.host.KSH_RECONCILE_AFFINITY_UNSATISFIED).any()
        exp = ctx.export_packed()
        with ks.Snapshot(0) as s:
            s.set_nodes(*exp[:3])
            s.set_bound(*exp[3:])
            f = s.free()
        assert np.array_equal(f[0], want_free[0]) and np.array_equal(f[1], want_free[1])
