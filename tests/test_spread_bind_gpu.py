"""Topology spread when binding (ks_spread_bind) on the H100: nodes, scores, refusals, counts and the final free[] bit for
bit against tests/spread_bind_oracle.py across label widths, node counts at the CTA-slice edges, key sets (zone,
hostname, both, keyless nodes), skews, minDomains, existing counts, unconstrained pods mixed in and every policy; both
identities of include/ksched.h on the device (ks_gang_bind with singleton groups, ks_place_replicas_spread(_multi) with
commit); a following ks_select on both kernel paths; every error code leaving free[] unchanged; the empty snapshot; and
the host layer (ksh_reconcile_spread)."""
import ctypes as C
import json

import numpy as np
import pytest

from spread_bind_oracle import spread_bind_packed
from test_replicas_gpu import _nodes, _specs, load
from test_spread_gpu import D_SEED, _gv1_zoned, domains, zone_labels

pytestmark = pytest.mark.gpu

ZONE, HOST = "topology.kubernetes.io/zone", "kubernetes.io/hostname"
POLICIES = (0, 1, 3, 4)


def check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, keys, skew, mind=None, ex=None, policy=0):
    got = snap.spread_bind(rc, rm, sel, group, keys, skew, mind, ex, policy)
    ofc, ofm = fc.copy(), fm.copy()
    want = spread_bind_packed(ofc, ofm, ac, am, lab, rc, rm, sel, group, keys, skew, mind, ex, policy)
    assert np.array_equal(got[0], want[0]), np.nonzero(got[0] != want[0])[0][:8]
    assert np.array_equal(got[1], want[1]), np.nonzero(got[1] != want[1])[0][:8]
    assert np.array_equal(got[2], want[2]), np.nonzero(got[2] != want[2])[0][:8]
    for a, b in zip(got[3], want[3]):
        assert np.array_equal(a, b)
    gfc, gfm = snap.free()
    assert np.array_equal(gfc, ofc) and np.array_equal(gfm, ofm)
    return got, (ofc, ofm)


def key_set(rng, N, modes):
    """One (node_domain, D) per mode; a 'host' key after another key also drops about 5% of nodes."""
    keys = []
    for mode in modes:
        dom, D = domains(rng, N, mode)
        if mode == "host" and keys:
            dom = dom.copy()
            dom[rng.random(N) < 0.05] = -1
        keys.append((dom, D))
    return keys


def mixed_queue(rng, N, W, keys, G, P, cpu=(0, 6000), mem=(0, 24 << 30)):
    """G workloads and unconstrained pods interleaved at random.  Workload 0 constrains every key at max_skew 1, workload
    1 the first key only; the others draw max_skew from {0, 1, 2, 5} per key.  Workload g's pods carry its own selector
    (workload 0 one that excludes every odd domain of key 0) and requests that vary within the workload."""
    K = len(keys)
    _, _, gsel = _specs(rng, G, W, sel_p=0.3)
    gsel[0, 0] |= np.uint64(1)
    skew = np.array([0, 1, 2, 5], np.uint32)[rng.integers(0, 4, (G, K))]
    skew[0] = 1
    if G > 1:
        skew[1] = 0
        skew[1, 0] = 2
    group = rng.integers(-1, G, P).astype(np.int32)
    rc, rm, sel = _specs(rng, P, W, cpu=cpu, mem=mem, sel_p=0.2)
    sel[group >= 0] = gsel[group[group >= 0]]
    rc[rng.random(P) < 0.05] = 0
    mind = np.zeros((G, K), np.uint32)
    ne = [len(np.unique(d[d >= 0])) for d, _ in keys]
    mind[G // 2:, 0] = ne[0] + (np.arange(G - G // 2) % 2)  # |E| and |E| + 1 on key 0
    ex = [rng.integers(0, 3, (G, D)).astype(np.uint32) for _, D in keys]
    return rc, rm, sel, group, skew, mind, ex


CASES = [  # (W, N, key modes, groups, pods)
    (1, 1, (1,), 3, 40),
    (2, 127, (3, "host"), 4, 300),
    (4, 128, (3,), 5, 300),
    (8, 129, ("host",), 3, 200),
    (1, 1000, (3, "host"), 8, 500),
    (2, 2100, ("edge", "host"), 6, 400),
    (4, 3000, (3, 7, "host"), 6, 400),
    (8, 16896, (7, "host"), 6, 150),
    (1, 16897, (3,), 6, 150),
]


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("case", CASES, ids=[f"W{c[0]}-N{c[1]}-" + "+".join(map(str, c[2])) for c in CASES])
def test_against_the_oracle(ks, case, policy):
    W, N, modes, G, P = case
    rng = np.random.default_rng([W, N, len(modes), policy] + [D_SEED.get(str(m), 5) for m in modes])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, modes)
    lab = zone_labels(lab, *keys[0])
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got, _ = check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, keys, skew, mind, ex, policy)
        # and without minDomains or existing counts
        load(ks, snap, fc, fm, ac, am, lab)
        check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, keys, skew, None, None, policy)
    if N > 1:
        assert (got[0] >= 0).any() and got[2].any(), "some pods placed, some nodes refused"


@pytest.mark.parametrize("policy", POLICIES)
def test_unconstrained_is_gang_bind_with_singletons(ks, policy):
    """Identity 1 on the device: group -1 everywhere, then every max_skew 0: the nodes, scores and final free[] of
    ks_gang_bind with singleton groups and min_member 0."""
    rng = np.random.default_rng(0xB1 + policy)
    N, P, W = 3000, 600, 2
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3, "host"))
    rc, rm, sel = _specs(rng, P, W, cpu=(0, 8000), mem=(0, 32 << 30))
    for group, G in ((np.full(P, -1, np.int32), 0), (rng.integers(0, 4, P).astype(np.int32), 4)):
        sel_g = sel.copy()
        if G:
            sel_g[:] = sel[group]  # one selector per group
        with ks.Snapshot(0) as snap:
            load(ks, snap, fc, fm, ac, am, lab)
            want = snap.gang_bind(rc, rm, sel_g, np.arange(P + 1), np.zeros(P), policy) + snap.free()
            load(ks, snap, fc, fm, ac, am, lab)
            got = snap.spread_bind(rc, rm, sel_g, group, keys, np.zeros((G, 2)), policy=policy)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
            assert not got[2].any()
            gfc, gfm = snap.free()
            assert np.array_equal(gfc, want[4]) and np.array_equal(gfm, want[5])
            assert (got[0] >= 0).sum() > P // 2


@pytest.mark.parametrize("policy", POLICIES)
def test_one_group_is_the_replica_plan(ks, policy):
    """Identity 2 on the device: one group of R identical pods constraining every key binds the copy list of
    ks_place_replicas_spread_multi (ks_place_replicas_spread for K = 1), with its counts, and free[] ends as after
    ks_snapshot_commit_claims of that list."""
    rng = np.random.default_rng(0xB2 + policy)
    N, W = 2500, 1
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    for modes in ((3,), ("host",), (3, "host"), (7, 3, "host")):
        keys = key_set(rng, N, modes)
        K = len(keys)
        rc, rm, sel = _specs(rng, 1, W, cpu=(500, 3000), mem=(1 << 30, 8 << 30), sel_p=0.5)
        R = 700
        skew = rng.integers(1, 3, (1, K)).astype(np.uint32)
        mind = np.zeros((1, K), np.uint32)
        ex = [rng.integers(0, 4, (1, D)).astype(np.uint32) for _, D in keys]
        with ks.Snapshot(0) as snap:
            load(ks, snap, fc, fm, ac, am, lab)
            if K == 1:
                plan = snap.place_replicas_spread(rc, rm, sel, [R], keys[0][0], keys[0][1], skew[:, 0], mind[:, 0],
                                                  ex[0], policy)
                plan_counts = [plan[4]]
            else:
                plan = snap.place_replicas_spread_multi(rc, rm, sel, [R], keys, skew, mind, ex, policy)
                plan_counts = plan[4]
            acc = snap.commit_claims(plan[1], np.repeat(rc, R), np.repeat(rm, R))
            assert acc[plan[1] >= 0].all()
            want_free = snap.free()
            load(ks, snap, fc, fm, ac, am, lab)
            got = snap.spread_bind(np.repeat(rc, R), np.repeat(rm, R), np.repeat(sel, R, axis=0), np.zeros(R), keys,
                                   skew, mind, ex, policy)
            assert np.array_equal(got[0], plan[1]) and np.array_equal(got[1], plan[2]), modes
            assert all(np.array_equal(a, b) for a, b in zip(got[3], plan_counts)), modes
            gfc, gfm = snap.free()
            assert np.array_equal(gfc, want_free[0]) and np.array_equal(gfm, want_free[1]), modes
            assert (got[0] >= 0).any()


def test_following_select_sees_the_charges(ks, orc):
    """After a call, ks_select on both kernel paths scores the charged free[] (the stale index is rebuilt)."""
    rng = np.random.default_rng(0xB3)
    N, W = 4000, 1
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3, "host"))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, 6, 800, cpu=(1000, 9000), mem=(4 << 30, 40 << 30))
    qc, qm, qs = _specs(rng, 300, W)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        snap.select(qc, qm, qs, policy=0, flags=ks.KS_SELECT_FORCE_BITPAR)  # builds the index before the call
        _, (ofc, ofm) = check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, keys, skew, mind, ex, 0)
        for policy in (0, 1):
            widx, wscore = orc.run_packed(ofc, ofm, ac, am, lab, qc, qm, qs, policy=policy, want_mask=False)[:2]
            for flags in (ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR):
                r = snap.select(qc, qm, qs, policy=policy, flags=flags)
                assert np.array_equal(r.node_idx, widx) and np.array_equal(r.score, wscore), (policy, r.path)


def test_errors_leave_free_unchanged(ks):
    rng = np.random.default_rng(0xB4)
    N, W = 300, 1
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3, "host"))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, 3, 50)
    E_INV, E_RANGE = ks.capi.KS_ERR_INVALID, ks.capi.KS_ERR_RANGE

    def call(snap, rc=rc, rm=rm, sel=sel, group=group, keys=keys, skew=skew, mind=mind, ex=ex, policy=0):
        with pytest.raises(ks.KsError) as e:
            snap.spread_bind(rc, rm, sel, group, keys, skew, mind, ex, policy)
        return e.value.code

    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        before = snap.free()
        big = rc.copy()
        big[7] = (1 << 36) + 1  # KS_MAX_CPU_MILLI + 1
        assert call(snap, rc=big) == E_RANGE
        neg = rm.copy()
        neg[3] = -1
        assert call(snap, rm=neg) == E_RANGE
        bad = group.copy()
        bad[5] = 3
        assert call(snap, group=bad) == E_INV
        bad[5] = -2
        assert call(snap, group=bad) == E_INV
        other = sel.copy()
        g0 = np.nonzero(group == 0)[0]
        other[g0[-1], 0] ^= np.uint64(1 << 40)
        assert call(snap, sel=other) == E_INV
        assert call(snap, policy=2) == E_INV
        wrong = [(keys[0][0].copy(), keys[0][1]), keys[1]]
        wrong[0][0][4] = keys[0][1]
        assert call(snap, keys=wrong) == E_INV
        assert call(snap, keys=[(keys[0][0], 0), keys[1]], ex=None) == E_RANGE
        too_many = [e.copy() for e in ex]
        too_many[1][2, 3] = ks.capi.KS_SPREAD_MAX_EXISTING + 1
        assert call(snap, ex=too_many) == E_RANGE
        P = ks.capi.KS_SPREAD_BIND_MAX_PODS + 1
        assert call(snap, rc=np.zeros(P), rm=np.zeros(P), sel=np.zeros((P, W)), group=np.full(P, -1)) == E_RANGE
        G = ks.capi.KS_SPREAD_BIND_MAX_GROUPS + 1
        assert call(snap, skew=np.ones((G, 2)), mind=None, ex=None) == E_RANGE
        wide = [(np.arange(N, dtype=np.int32) % 1000, 1 << 20)]
        assert call(snap, keys=wide, skew=np.ones((65, 1)), mind=None, ex=None) == E_RANGE  # 65 * 2^20 > 2^26
        # device-space pods
        pods = ks.capi.ks_pods(len(rc), rc.ctypes.data, rm.ctypes.data, sel.ctypes.data, ks.KS_MEM_DEVICE)
        idx = np.empty(len(rc), np.int32)
        sp = ks.capi.ks_spread_multi(1, (C.c_uint32 * 4)(keys[0][1]), (C.c_void_p * 4)(keys[0][0].ctypes.data),
                                     skew.ctypes.data, None, None)
        g32 = np.ascontiguousarray(group, np.int32)
        assert ks.lib.ks_spread_bind(snap._h, C.byref(pods), g32.ctypes.data, 3, C.byref(sp), 0, idx.ctypes.data, None,
                                     None, None) == E_INV
        after = snap.free()
        assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
        # P = 0 does nothing
        got = snap.spread_bind(rc[:0], rm[:0], sel[:0], group[:0], keys, skew, mind, ex)
        assert got[0].shape == (0,) and np.array_equal(snap.free()[0], before[0])


def test_empty_snapshot(ks):
    keys = [(np.zeros(0, np.int32), 3)]
    ex = [np.array([[1, 2, 3], [4, 5, 6]], np.uint32)]
    with ks.Snapshot(0) as snap:
        snap.set_nodes(np.zeros(0), np.zeros(0), np.zeros((0, 1)))
        got = snap.spread_bind([1, 0, 5], [1, 0, 5], np.zeros((3, 1)), [0, -1, 1], keys, [[1], [2]], None, ex)
        assert (got[0] == -1).all() and (got[1] == 0).all() and (got[2] == 0).all()
        assert np.array_equal(got[3][0], ex[0])


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
    """ksh_reconcile_spread equals ks_spread_bind on the packed arrays over the pods that go to the device; statuses,
    Binding bodies, the bound list, the charged snapshot, and KSH_RECONCILE_SPREAD_UNSATISFIED for pods that some node
    would take but the spread rule refused."""
    g, nodes = _gv1_zoned()
    nodes, objs = _objects(g, nodes)
    group = np.array([i % 3 if i % 3 < 2 else -1 for i in range(12)], np.int32)  # workloads 0, 1; every third none
    skew = np.array([[1, 1], [1, 0]], np.uint32)  # workload 0: zone + hostname, workload 1: zone only
    arena = ks.objects.ObjectArena()
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(nodes), len(nodes))
        names = [ctx.node_name(i) for i in range(ctx.n_nodes)]
        existing = [[[names[0], "no-such-node"], []], [[names[2]], [names[1]]]]
        zdom, zval = ctx.topology_domains(ZONE)
        hdom, hval = ctx.topology_domains(HOST)
        keys = [(zdom, len(zval)), (hdom, len(hval))]
        ex = [np.zeros((2, D), np.uint32) for _, D in keys]
        for gi in range(2):
            for k in range(2):
                for name in existing[gi][k]:
                    if name not in names:
                        continue
                    n = names.index(name)
                    if keys[k][0][n] >= 0 and all(skew[gi, k2] == 0 or keys[k2][0][n] >= 0 for k2 in range(2)):
                        ex[k][gi, keys[k][0][n]] += 1
        ac, am, lab, bn, bc, bm = ctx.export_packed()
        todo = [i for i in range(12) if i not in (4, 7)]
        rc, rm, sel = ctx.pack_pods(arena.pods([objs[i] for i in todo]), len(todo))
        with ks.Snapshot(0) as s:
            s.set_nodes(ac, am, lab)
            s.set_bound(bn, bc, bm)
            want = s.spread_bind(rc, rm, sel, group[todo], keys, skew, None, ex)
            want_free = s.free()
        bound0 = ctx.num_bound
        pods = arena.pods(objs)
        status, node, bodies = ctx.reconcile_spread(pods, 12, group, 2, [ZONE, HOST], skew, None, existing)
        assert status[4] == ks.host.KSH_RECONCILE_OK and node[4] == -1 and bodies[4] is None
        assert status[7] == ks.host.KSH_RECONCILE_BINDING_OBJECT_FAILED and node[7] == -1
        assert np.array_equal(node[todo], want[0])
        for k, i in enumerate(todo):
            if want[0][k] >= 0:
                assert status[i] == ks.host.KSH_RECONCILE_OK
                body = json.loads(bodies[i])
                assert body["kind"] == "Binding" and body["target"]["name"] == names[want[0][k]]
                assert body["metadata"]["name"] == objs[i]["name"]
            elif want[2][k] > 0:
                assert status[i] == ks.host.KSH_RECONCILE_SPREAD_UNSATISFIED and bodies[i] is None
            else:
                assert status[i] == ks.host.KSH_RECONCILE_NO_NODE_FOUND and bodies[i] is None
        placed = int((want[0] >= 0).sum())
        assert ctx.num_bound == bound0 + placed and placed > 0
        assert (status == ks.host.KSH_RECONCILE_SPREAD_UNSATISFIED).any()
        exp = ctx.export_packed()
        with ks.Snapshot(0) as s:  # the bound list now carries the binds: it rebuilds the charged free[]
            s.set_nodes(*exp[:3])
            s.set_bound(*exp[3:])
            f = s.free()
        assert np.array_equal(f[0], want_free[0]) and np.array_equal(f[1], want_free[1])
