"""Topology spread over several keys (ks_place_replicas_spread_multi) on the H100: rows, copy nodes, copy scores and
per-key counts bit for bit against tests/spread_multi_oracle.py across label widths, node counts around the 1024-node
block edge, key sets (zones + hostname, 7 + 64 domains, two partitions with equal D, three keys), skews, minDomains,
skewed existing counts, keyless nodes per key, selectors that exclude whole domains and every policy; K = 1 against
ks_place_replicas_spread; key-order invariance; commit with nothing charged; staging shared with other calls; the
errors; and the host layer."""
import ctypes as C

import numpy as np
import pytest

from spread_multi_oracle import spread_multi_packed
from test_replicas_gpu import _nodes, _specs, load
from test_spread_gpu import CASES, D_SEED, FIELDS, UNBOUNDED, ZONE, _gv1_zoned, domains, zone_labels

pytestmark = pytest.mark.gpu

HOST = "kubernetes.io/hostname"


def check(snap, fc, fm, ac, am, lab, rc, rm, sel, R, keys, skew, mind=None, ex=None, policy=0):
    got = snap.place_replicas_spread_multi(rc, rm, sel, R, keys, skew, mind, ex, policy)
    want = spread_multi_packed(fc, fm, ac, am, lab, rc, rm, sel, R, keys, skew, mind, ex, policy)
    for f in FIELDS:
        assert np.array_equal(got[0][f], want[0][f]), (f, got[0][f][:4], want[0][f][:4])
    assert np.array_equal(got[1], want[1]), np.nonzero(got[1] != want[1])[0][:8]
    assert np.array_equal(got[2], want[2]), np.nonzero(got[2] != want[2])[0][:8]
    assert np.array_equal(got[3], want[3])
    for a, b in zip(got[4], want[4]):
        assert np.array_equal(a, b)
    return got


def key_set(rng, N, modes):
    """One (node_domain, D) per mode; a second 'host' key also drops about 5% of nodes (keyless for that key only)."""
    keys = []
    for mode in modes:
        dom, D = domains(rng, N, mode)
        if mode == "host" and keys:
            dom = dom.copy()
            dom[rng.random(N) < 0.05] = -1
        keys.append((dom, D))
    return keys


MCASES = [  # (W, N, key modes, specs, replicas)
    (1, 1, (1, "host"), 3, 5),
    (2, 1023, (3, "host"), 6, 300),
    (4, 1024, (7, 64), 6, 400),
    (8, 1025, (5, 5), 6, 200),
    (1, 2100, ("edge", "host"), 4, 500),
    (2, 3000, (3, 7, "host"), 6, 400),
    (4, 2500, (64, 3), 6, 300),
]


@pytest.mark.parametrize("policy", [0, 1, 3, 4])
@pytest.mark.parametrize("case", MCASES, ids=[f"W{c[0]}-N{c[1]}-" + "+".join(map(str, c[2])) for c in MCASES])
def test_against_the_oracle(ks, case, policy):
    W, N, modes, T, Rmax = case
    rng = np.random.default_rng([W, N, len(modes), policy] + [D_SEED.get(str(m), 5) for m in modes])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, modes)
    lab = zone_labels(lab, *keys[0])
    K = len(keys)
    rc, rm, sel = _specs(rng, T, W, cpu=(0, 1500), mem=(0, 4 << 30), sel_p=0.2)
    sel[0, 0] |= np.uint64(1)  # spec 0 excludes every odd domain of key 0
    if T > 2:
        rc[2], rm[2] = 0, 0  # zero requests: unbounded copies per node
    R = rng.integers(0, Rmax + 1, T).astype(np.uint32)
    R[0] = Rmax
    skew = np.array([1, 2, 5, UNBOUNDED], np.uint32)[rng.integers(0, 4, (T, K))]
    skew[0] = 1
    ne = [len(np.unique(d[d >= 0])) for d, _ in keys]
    mind = np.zeros((T, K), np.int64)
    mind[T // 2:, 0] = ne[0] + (np.arange(T - T // 2) % 2)  # minDomains on key 0 only: |E| and |E| + 1
    ex = []
    for _, D in keys:
        e = rng.integers(0, 3, (T, D)).astype(np.uint32)
        e[:, : max(1, D // 4)] += rng.integers(0, 12, (T, max(1, D // 4))).astype(np.uint32)
        ex.append(e)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got = check(snap, fc, fm, ac, am, lab, rc, rm, sel, R, keys, skew, mind, ex, policy)
        check(snap, fc, fm, ac, am, lab, rc, rm, sel, R, keys, skew, None, None, policy)
    if N > 1:
        assert (got[0]["placed"] > 0).any()


@pytest.mark.parametrize("policy", [0, 1, 3, 4])
@pytest.mark.parametrize("case", CASES, ids=[f"W{c[0]}-N{c[1]}-D{c[2]}" for c in CASES])
def test_one_key_is_the_single_key_call(ks, case, policy):
    W, N, mode, T, Rmax = case
    rng = np.random.default_rng([W, N, D_SEED[str(mode)], policy, 1])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    dom, D = domains(rng, N, mode)
    lab = zone_labels(lab, dom, D)
    rc, rm, sel = _specs(rng, T, W, cpu=(0, 1500), mem=(0, 4 << 30), sel_p=0.2)
    R = rng.integers(0, Rmax + 1, T).astype(np.uint32)
    skew = np.array([1, 2, 5, UNBOUNDED] * T, np.uint32)[:T]
    mind = np.array([0, 1, 0, 4] * T, np.uint32)[:T]
    ex = rng.integers(0, 4, (T, D)).astype(np.uint32)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        one = snap.place_replicas_spread(rc, rm, sel, R, dom, D, skew, mind, ex, policy)
        multi = snap.place_replicas_spread_multi(rc, rm, sel, R, [(dom, D)], skew, mind, [ex], policy)
    assert np.array_equal(one[0], multi[0][:, 0])
    for a, b in zip(one[1:4], multi[1:4]):
        assert np.array_equal(a, b)
    assert np.array_equal(one[4], multi[4][0])


@pytest.mark.parametrize("policy", [0, 3])
def test_key_order_invariance(ks, policy):
    """Permuting the keys permutes each spec's rows and count blocks and leaves the copies unchanged; two keys with equal
    D make the primary change with the order."""
    rng = np.random.default_rng(0x0D + policy)
    N, T, W = 2000, 6, 1
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (6, 6, "host"))
    rc, rm, sel = _specs(rng, T, W)
    R = rng.integers(100, 800, T).astype(np.uint32)
    skew = rng.integers(1, 4, (T, 3)).astype(np.uint32)
    mind = rng.integers(0, 8, (T, 3)).astype(np.uint32)
    ex = [rng.integers(0, 5, (T, D)).astype(np.uint32) for _, D in keys]
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        base = check(snap, fc, fm, ac, am, lab, rc, rm, sel, R, keys, skew, mind, ex, policy)
        for perm in ((1, 0, 2), (2, 1, 0), (1, 2, 0)):
            p = list(perm)
            got = snap.place_replicas_spread_multi(rc, rm, sel, R, [keys[i] for i in p], skew[:, p], mind[:, p],
                                                   [ex[i] for i in p], policy)
            assert np.array_equal(got[0], base[0][:, p]), perm
            assert np.array_equal(got[1], base[1]) and np.array_equal(got[2], base[2]), perm
            for i, c in zip(p, got[4]):
                assert np.array_equal(c, base[4][i]), perm


def test_zone_and_hostname_bind_together(ks):
    """Zones with maxSkew 1 and hostname with maxSkew 1: no node takes a second copy before every eligible node with
    room holds one, and the zone counts stay within 1 of each other while every zone has room."""
    rng = np.random.default_rng(0x2F)
    N, W = 1500, 1
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    zone = (np.arange(N) % 3).astype(np.int32)
    keys = [(zone, 3), (np.arange(N, dtype=np.int32), N)]
    z = np.zeros(1, np.int64)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        rows, node, _, _, cnt = check(snap, fc, fm, ac, am, lab, z, z, np.zeros((1, W), np.uint64), [2 * N], keys,
                                      np.ones((1, 2), np.uint32))
    assert rows["placed"][0, 0] == 2 * N and len(set(node[:N].tolist())) == N
    assert cnt[0][0].tolist() == [2 * N // 3] * 3 and (cnt[1][0] == 2).all()


def test_commit_accepts_every_claim(ks):
    rng = np.random.default_rng(0xC0)
    N, T, W = 3000, 8, 2
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3, "host"))
    rc, rm, sel = _specs(rng, T, W)
    R = rng.integers(100, 2000, T).astype(np.uint32)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        rows, node, _, off, _ = snap.place_replicas_spread_multi(rc, rm, sel, R, keys, np.ones((T, 2)))
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), (fc, fm)))  # nothing charged
        for t in range(T):
            a, p = int(off[t]), int(rows["placed"][t, 0])
            load(ks, snap, fc, fm, ac, am, lab)
            acc = snap.commit_claims(node[a:a + p], np.repeat(rc[t], p), np.repeat(rm[t], p))
            assert acc.all(), t
    assert rows["placed"][:, 0].sum() > 1000


def test_staging_shared_with_other_calls(ks):
    """Interleaved with ks_place_replicas, ks_drain_check and the single-key call on one snapshot, each result equals the
    same call on a fresh snapshot."""
    rng = np.random.default_rng(0x5B)
    N, T, W = 3000, 32, 2
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    rc, rm, sel = _specs(rng, T, W)
    keys = key_set(rng, N, (5, "host"))
    R = rng.integers(0, 2000, T).astype(np.uint32)
    ex = [rng.integers(0, 5, (T, D)).astype(np.uint32) for _, D in keys]
    multi = lambda s: s.place_replicas_spread_multi(rc, rm, sel, R, keys, np.full((T, 2), 2), None, ex, 1)
    single = lambda s: s.place_replicas_spread(rc, rm, sel, R, keys[0][0], keys[0][1], np.full(T, 2), None, ex[0], 1)
    rep = lambda s: s.place_replicas(rc, rm, sel, R * 4, 0)
    drain = lambda s: s.drain_check(rc[:16], rm[:16], sel[:16], np.arange(8, dtype=np.int32),
                                    np.arange(0, 17, 2, dtype=np.uint64), 0)

    def fresh(fn):
        with ks.Snapshot(0) as s:
            load(ks, s, fc, fm, ac, am, lab)
            return fn(s)

    def same(a, b):
        if isinstance(a, list):
            return all(same(x, y) for x, y in zip(a, b))
        return np.array_equal(np.asarray(a), np.asarray(b))

    calls = (("multi", multi), ("rep", rep), ("multi", multi), ("drain", drain), ("single", single), ("multi", multi))
    want = {k: fresh(f) for k, f in calls}
    with ks.Snapshot(0) as s:
        load(ks, s, fc, fm, ac, am, lab)
        for step in range(2):
            for name, fn in calls:
                assert all(same(a, b) for a, b in zip(fn(s), want[name])), (step, name)


def test_empty_snapshot_and_errors(ks):
    T, W = 3, 1
    rc, rm, sel = np.ones(T, np.int64), np.ones(T, np.int64), np.zeros((T, W), np.uint64)
    R = np.array([2, 0, 3], np.uint32)
    ex = [np.arange(T * 2, dtype=np.uint32).reshape(T, 2), np.arange(T * 3, dtype=np.uint32).reshape(T, 3)]
    with ks.Snapshot(0) as snap:
        snap.set_nodes(np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, W), np.uint64))
        e0 = np.zeros(0, np.int32)
        rows, node, score, _, cnt = snap.place_replicas_spread_multi(rc, rm, sel, R, [(e0, 2), (e0, 3)],
                                                                     np.ones((T, 2)), existing=ex)
        assert rows.shape == (T, 2) and (rows["blocked_domain"] == -1).all() and (rows["placed"] == 0).all()
        assert (node == -1).all() and (score == 0).all() and all(np.array_equal(a, b) for a, b in zip(cnt, ex))
        N = 4
        fc = np.full(N, 1000, np.int64)
        load(ks, snap, fc, fc << 20, fc, fc << 20, np.zeros((N, W), np.uint64))
        dom0, dom1 = np.array([0, 1, -1, 0], np.int32), np.array([0, 1, 2, 2], np.int32)

        def code(keys=None, skew=None, mind=None, exist=None, policy=0):
            keys = keys or [(dom0, 2), (dom1, 3)]
            skew = np.ones((T, len(keys))) if skew is None else skew
            with pytest.raises(ks.KsError) as e:
                snap.place_replicas_spread_multi(rc, rm, sel, R, keys, skew, mind, exist, policy)
            return e.value.code

        assert code(keys=[(dom0, 2), (dom1, 0)]) == ks.capi.KS_ERR_RANGE
        assert code(keys=[(dom0, 2), (np.zeros(N, np.int32), (1 << 20) + 1)]) == ks.capi.KS_ERR_RANGE
        assert code(skew=np.array([[1, 1], [1, 0], [1, 1]])) == ks.capi.KS_ERR_RANGE
        assert code(exist=[ex[0], np.full((T, 3), (1 << 24) + 1)]) == ks.capi.KS_ERR_RANGE
        assert code(keys=[(dom0, 2), (np.array([0, 3, 0, 0], np.int32), 3)]) == ks.capi.KS_ERR_INVALID
        assert code(keys=[(dom0, 2), (np.array([0, -2, 0, 0], np.int32), 3)]) == ks.capi.KS_ERR_INVALID
        assert code(policy=2) == ks.capi.KS_ERR_INVALID
        out = (ks.capi.ks_spread_plan * (T * 5))()
        pods = ks.capi.ks_pods(T, rc.ctypes.data, rm.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
        skew = np.ones(T * 5, np.uint32)
        doms = (C.c_void_p * 4)(dom0.ctypes.data, dom1.ctypes.data, None, None)

        def raw(k, nd, d=doms, pods=pods, counts=None):
            sp = ks.capi.ks_spread_multi(k, (C.c_uint32 * 4)(*nd), d, skew.ctypes.data, None, None)
            return ks.lib.ks_place_replicas_spread_multi(snap._h, C.byref(pods), R.ctypes.data, C.byref(sp), 0, out,
                                                         None, None, counts)

        assert raw(0, [2, 3, 0, 0]) == ks.capi.KS_ERR_RANGE
        assert raw(5, [2, 3, 1, 1]) == ks.capi.KS_ERR_RANGE
        assert raw(3, [2, 3, 1, 0]) == ks.capi.KS_ERR_INVALID  # node_domain[2] NULL
        dev = ks.capi.ks_pods(T, rc.ctypes.data, rm.ctypes.data, sel.ctypes.data, ks.KS_MEM_DEVICE)
        assert raw(2, [2, 3, 0, 0], pods=dev) == ks.capi.KS_ERR_INVALID
        assert ks.lib.ks_place_replicas_spread_multi(snap._h, C.byref(pods), R.ctypes.data, None, 0, out, None, None,
                                                     None) == ks.capi.KS_ERR_INVALID
        big_t = 33  # 33 specs x (2 + 2^21 - 2) domains of counts > 2^26
        b_rc, b_sel, b_rep = np.zeros(big_t, np.int64), np.zeros((big_t, W), np.uint64), np.ones(big_t, np.uint32)
        b_pods = ks.capi.ks_pods(big_t, b_rc.ctypes.data, b_rc.ctypes.data, b_sel.ctypes.data, ks.KS_MEM_HOST)
        b_out, counts, b_skew = (ks.capi.ks_spread_plan * (big_t * 2))(), np.zeros(4, np.uint32), np.ones(big_t * 2,
                                                                                                           np.uint32)
        zeros = np.zeros(N, np.int32)
        sp = ks.capi.ks_spread_multi(2, (C.c_uint32 * 4)(1 << 20, 1 << 20, 0, 0),
                                     (C.c_void_p * 4)(zeros.ctypes.data, zeros.ctypes.data, None, None),
                                     b_skew.ctypes.data, None, None)
        assert ks.lib.ks_place_replicas_spread_multi(snap._h, C.byref(b_pods), b_rep.ctypes.data, C.byref(sp), 0,
                                                     b_out, None, None, counts.ctypes.data) == ks.capi.KS_ERR_RANGE
        assert (counts == 0).all()
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), (fc, fc << 20)))


def test_host_layer(ks):
    """Plans over objects equal the packed call on the exported arrays with ksh_context_topology_domains' domains;
    existing names count under a key only when the node carries every key; K = 1 equals ksh_place_replicas_spread; a key
    that no node carries empties every row and writes no counts."""
    g, nodes = _gv1_zoned()
    arena = ks.objects.ObjectArena()
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(nodes), len(nodes))
        pods = arena.pods(g["pods"])
        n = len(g["pods"])
        R = np.arange(n, dtype=np.uint32) % 7 + 1
        skew = (np.arange(n * 2, dtype=np.uint32) % 2 + 1).reshape(n, 2)
        names = [ctx.node_name(i) for i in range(ctx.n_nodes)]
        existing = [[[names[t % len(names)], "no-such-node", names[-1]], [names[(t + 1) % len(names)]]]
                    for t in range(n)]
        for policy in (0, 1):
            got = ctx.place_replicas_spread_multi(pods, n, R, [ZONE, HOST], skew, None, existing, policy)
            zdom, zval = ctx.topology_domains(ZONE)
            hdom, hval = ctx.topology_domains(HOST)
            keys = [(zdom, len(zval)), (hdom, max(len(hval), 1))]
            if not hval:  # GV-1 nodes carry no hostname label: every row is empty
                assert (got[0]["placed"] == 0).all() and (got[0]["blocked_domain"] == -1).all() and got[4] is None
            both = (zdom >= 0) & (hdom >= 0)
            ex = [np.zeros((n, D), np.uint32) for _, D in keys]
            for t in range(n):
                for k in range(2):
                    for name in existing[t][k]:
                        if name in names and both[names.index(name)]:
                            ex[k][t, keys[k][0][names.index(name)]] += 1
            ac, am, lab, bn, bc, bm = ctx.export_packed()
            rc, rm, sel = ctx.pack_pods(pods, n)
            with ks.Snapshot(0) as s:
                s.set_nodes(ac, am, lab)
                s.set_bound(bn, bc, bm)
                want = s.place_replicas_spread_multi(rc, rm, sel, R, keys, skew, None, ex, policy)
            for a, b in zip(got[:4], want[:4]):
                assert np.array_equal(a, b), policy
            if got[4] is not None:
                assert all(np.array_equal(a, b) for a, b in zip(got[4], want[4]))
            one = ctx.place_replicas_spread_multi(pods, n, R, [ZONE], skew[:, :1], None,
                                                  [[e[0]] for e in existing], policy)
            single = ctx.place_replicas_spread(pods, n, R, ZONE, skew[:, 0], None, [e[0] for e in existing], policy)
            assert np.array_equal(one[0][:, 0], single[0])
            for a, b in zip(one[1:4], single[1:4]):
                assert np.array_equal(a, b)
            assert np.array_equal(one[4][0], single[4])


def test_host_layer_with_hostnames(ks):
    """Zone + hostname labels on the nodes: the object-level plan equals the packed one, and a node without the zone
    label neither takes a copy nor counts its existing pods."""
    g, nodes = _gv1_zoned()
    nodes = [dict(nd, labels=dict(nd["labels"], **{HOST: nd["name"]})) for nd in nodes]
    arena = ks.objects.ObjectArena()
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(nodes), len(nodes))
        pods = arena.pods(g["pods"])
        n = len(g["pods"])
        R = np.full(n, 6, np.uint32)
        skew = np.ones((n, 2), np.uint32)
        names = [ctx.node_name(i) for i in range(ctx.n_nodes)]
        existing = [[[names[-1], names[0]], [names[-1]]] for _ in range(n)]
        got = ctx.place_replicas_spread_multi(pods, n, R, [ZONE, HOST], skew, None, existing, 0)
        zdom, zval = ctx.topology_domains(ZONE)
        hdom, hval = ctx.topology_domains(HOST)
        keys = [(zdom, len(zval)), (hdom, len(hval))]
        both = (zdom >= 0) & (hdom >= 0)
        ex = [np.zeros((n, D), np.uint32) for _, D in keys]
        for t in range(n):
            for k in range(2):
                for name in existing[t][k]:
                    i = names.index(name)
                    if both[i]:
                        ex[k][t, keys[k][0][i]] += 1
        ac, am, lab, bn, bc, bm = ctx.export_packed()
        rc, rm, sel = ctx.pack_pods(pods, n)
        with ks.Snapshot(0) as s:
            s.set_nodes(ac, am, lab)
            s.set_bound(bn, bc, bm)
            want = s.place_replicas_spread_multi(rc, rm, sel, R, keys, skew, None, ex, 0)
        for a, b in zip(got[:4], want[:4]):
            assert np.array_equal(a, b)
        assert all(np.array_equal(a, b) for a, b in zip(got[4], want[4]))
        keyless = [i for i in range(len(names)) if zdom[i] < 0]
        assert keyless and not np.isin(got[1], keyless).any()
