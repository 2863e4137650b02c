"""Topology spread for replica placement (ks_place_replicas_spread) on the H100: rows, copy nodes, copy scores and domain
counts bit for bit against the restatement of tests/spread_oracle.py across label widths, node counts around the block
and group edges, domain counts from 1 to N, skews, minDomains, skewed existing counts, keyless nodes and selectors that
exclude whole domains; the two identities (ks_place_replicas where the rule cannot bind, ks_select_topk for hostname
spreading); the tie rule across domains; commit with nothing charged; the limits and errors; staging shared with other
calls; and the host layer."""
import ctypes as C

import numpy as np
import pytest

from helpers import load_golden
from spread_oracle import spread_packed
from test_replicas_gpu import _nodes, _specs, load

pytestmark = pytest.mark.gpu

FIELDS = ("placed", "nodes", "max_per_node", "eligible_domains", "min_count", "blocked_domain", "last_score")
UNBOUNDED = 0xFFFFFFFF


def check(snap, fc, fm, ac, am, lab, rc, rm, sel, R, dom, D, skew, mind=None, ex=None, policy=0):
    got = snap.place_replicas_spread(rc, rm, sel, R, dom, D, skew, mind, ex, policy)
    want = spread_packed(fc, fm, ac, am, lab, rc, rm, sel, R, dom, D, skew, mind, ex, policy)
    for f in FIELDS:
        assert np.array_equal(got[0][f], want[0][f]), (f, got[0][f][:8], want[0][f][:8])
    assert np.array_equal(got[1], want[1]), np.nonzero(got[1] != want[1])[0][:8]
    assert np.array_equal(got[2], want[2]), np.nonzero(got[2] != want[2])[0][:8]
    assert np.array_equal(got[3], want[3])
    assert np.array_equal(got[4], want[4])
    return got


def domains(rng, N, mode):
    """node_domain for a mode: a domain count, 'host' (node n = domain n), or 'edge' (1025 nodes in domain 0 around a
    block edge, the rest in domain 1); about 8% of nodes without the key except for 'host'."""
    if mode == "host":
        return np.arange(N, dtype=np.int32), N
    if mode == "edge":
        dom = np.where(np.arange(N) < 1025, 0, 1).astype(np.int32)
        return dom, 2
    dom = rng.integers(0, mode, N).astype(np.int32)
    dom[rng.random(N) < 0.08] = -1
    return dom, mode


def zone_labels(lab, dom, D):
    """Bit 0 of word 0 set on the nodes of even domains only: a selector on it excludes every odd domain."""
    lab = lab.copy()
    lab[:, 0] &= ~np.uint64(1)
    lab[:, 0] |= ((dom >= 0) & (dom % 2 == 0)).astype(np.uint64)
    return lab


D_SEED = {"1": 1, "3": 3, "7": 7, "64": 64, "edge": 100, "host": 101}
CASES = [  # (W, N, domain mode, specs, replicas)
    (1, 1, 1, 4, 6),
    (2, 1023, 1, 6, 60),
    (4, 1024, 1, 6, 60),
    (8, 1025, 1, 6, 60),
    (1, 2100, "edge", 6, 80),
    (2, 3000, 3, 8, 120),
    (4, 2500, 7, 8, 120),
    (8, 4000, 64, 8, 200),
    (1, 1025, "host", 6, 1100),
    (2, 1500, "host", 4, 300),
    (1, 20000, 3, 3, 60),
]


@pytest.mark.parametrize("policy", [0, 1, 3, 4])
@pytest.mark.parametrize("case", CASES, ids=[f"W{c[0]}-N{c[1]}-D{c[2]}" for c in CASES])
def test_against_the_restatement(ks, case, policy):
    W, N, mode, T, Rmax = case
    rng = np.random.default_rng([W, N, D_SEED[str(mode)], policy])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    dom, D = domains(rng, N, mode)
    lab = zone_labels(lab, dom, D)
    rc, rm, sel = _specs(rng, T, W, cpu=(0, 1500), mem=(0, 4 << 30), sel_p=0.2)
    sel[0, 0] |= np.uint64(1)  # spec 0 excludes every odd domain
    if T > 1:
        sel[1, W - 1] |= np.uint64(1) << np.uint64(63)  # the never-set bit: no eligible domain
    if T > 2:
        rc[2], rm[2] = 0, 0  # zero requests: unbounded copies per node
    if T > 3 and N > 20:  # the cpu and memory limits on some nodes, negative free on others
        k = N // 10
        ac[:k], am[:k] = 1 << 36, 1 << 55
        fc[:k], fm[:k] = ac[:k] - rng.integers(0, 1000, k), am[:k] - rng.integers(0, 1 << 30, k)
        fc[k:2 * k] = -5
    R = rng.integers(0, Rmax + 1, T).astype(np.uint32)
    R[0] = Rmax
    skew = np.array([1, 2, 5, UNBOUNDED] * T, np.uint32)[:T]
    ne = np.array([len(np.unique(dom[dom >= 0]))] * T)
    mind = np.array([0, 1, 0, 1] * T, np.int64)[:T]
    mind[T // 2:] = ne[T // 2:] + (np.arange(T - T // 2) % 2)  # |E| and |E| + 1 (upper bounds on each spec's E)
    ex = rng.integers(0, 3, (T, D)).astype(np.uint32)
    ex[:, : max(1, D // 4)] += rng.integers(0, 12, (T, max(1, D // 4))).astype(np.uint32)  # some start above m + skew
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got = check(snap, fc, fm, ac, am, lab, rc, rm, sel, R, dom, D, skew, mind, ex, policy)
        check(snap, fc, fm, ac, am, lab, rc, rm, sel, R, dom, D, skew, None, None, policy)
    if N > 1:
        assert (got[0]["placed"] > 0).any()


@pytest.mark.parametrize("policy", [0, 1, 3, 4])
def test_unbinding_rule_equals_place_replicas(ks, policy):
    """One domain for every node, and a skew above every count: the plan is ks_place_replicas' plan."""
    rng = np.random.default_rng(0x1D + policy)
    N, T, W = 3000, 24, 2
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    rc, rm, sel = _specs(rng, T, W)
    R = rng.integers(0, 2000, T).astype(np.uint32)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        want = snap.place_replicas(rc, rm, sel, R, policy)
        D = 7
        dom = rng.integers(0, D, N).astype(np.int32)
        ex = rng.integers(0, 50, (T, D)).astype(np.uint32)
        for got in (snap.place_replicas_spread(rc, rm, sel, R, np.zeros(N, np.int32), 1, np.ones(T), policy=policy),
                    snap.place_replicas_spread(rc, rm, sel, R, dom, D, R + ex.max(1), existing=ex, policy=policy)):
            for f in ("placed", "nodes", "max_per_node", "last_score"):
                assert np.array_equal(got[0][f], want[0][f]), f
            assert np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
    assert (want[0]["placed"] > 0).any()


@pytest.mark.parametrize("policy", [0, 1, 3, 4])
def test_hostname_equals_topk(ks, policy):
    """node_domain[n] = n, max_skew 1, no existing pods, R <= 32: the copies are ks_select_topk's entries."""
    rng = np.random.default_rng(0x40 + policy)
    N, T, W = 2000, 32, 1
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    rc, rm, sel = _specs(rng, T, W)
    R = rng.integers(1, 33, T).astype(np.uint32)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        rows, node, score, off, _ = snap.place_replicas_spread(rc, rm, sel, R, np.arange(N, dtype=np.int32), N,
                                                               np.ones(T), policy=policy)
        idx, sc, cnt = snap.select_topk(rc, rm, sel, 32, policy)
    for t in range(T):
        a, r = int(off[t]), int(R[t])
        k = min(r, int(cnt[t]))
        assert rows["placed"][t] >= k  # a second round starts once every eligible node holds a copy
        assert node[a:a + k].tolist() == idx[t, :k].tolist() and score[a:a + k].tolist() == sc[t, :k].tolist(), t


def test_tie_rule_across_domains(ks):
    """Equal scores in two domains where the higher-index domain holds the lower nodes: every level compares (score,
    node) explicitly, so the lowest node wins, not the lowest domain or block."""
    N = 3000
    fc, fm = np.full(N, 4000, np.int64), np.full(N, 16 << 30, np.int64)
    lab = np.zeros((N, 1), np.uint64)
    dom = np.where(np.arange(N) < 1500, 2, np.where(np.arange(N) < 2600, 0, 1)).astype(np.int32)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, fc, fm, lab)
        for policy in (0, 1, 3, 4):
            for skew in (1, 3, UNBOUNDED):
                got = check(snap, fc, fm, fc, fm, lab, [1000], [1 << 30], np.zeros((1, 1), np.uint64), [12], dom, 3,
                            [skew], policy=policy)
                assert got[1][0] == 0
        hd = np.arange(N)[::-1].astype(np.int32)  # hostname domains in reverse: domain N-1 holds node 0
        got = check(snap, fc, fm, fc, fm, lab, [1000], [1 << 30], np.zeros((1, 1), np.uint64), [40], hd, N, [1])
        assert got[1][:40].tolist() == list(range(40))


def test_commit_accepts_every_claim_and_nothing_is_charged(ks):
    rng = np.random.default_rng(0xC0)
    N, T, W = 2000, 16, 1
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    rc, rm, sel = _specs(rng, T, W, sel_p=0)
    R = rng.integers(50, 400, T).astype(np.uint32)
    dom, D = domains(rng, N, 3)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        before = snap.select(rc, rm, sel)
        rows, node, score, off, _ = snap.place_replicas_spread(rc, rm, sel, R, dom, D, np.ones(T))
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), (fc, fm)))
        after = snap.select(rc, rm, sel)
        assert np.array_equal(after.node_idx, before.node_idx) and np.array_equal(after.score, before.score)
        for t in range(T):
            a = int(off[t])
            p = int(rows["placed"][t])
            load(ks, snap, fc, fm, ac, am, lab)
            acc = snap.commit_claims(node[a:a + p], np.repeat(rc[t], p), np.repeat(rm[t], p))
            assert acc.all(), t
    assert rows["placed"].sum() > 1000


def test_limits(ks):
    """T = 4096 specs, and 65 536 copies of one spec (hostname domains, so m rises once per round)."""
    rng = np.random.default_rng(0x11)
    N, W = 40, 1
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    dom, D = domains(rng, N, 3)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        T = ks.capi.KS_REPLICAS_MAX_SPECS
        rc, rm, sel = _specs(rng, T, W, cpu=(0, 300), mem=(0, 1 << 30))
        R = rng.integers(0, 6, T).astype(np.uint32)
        check(snap, fc, fm, ac, am, lab, rc, rm, sel, R, dom, D, rng.integers(1, 4, T).astype(np.uint32),
              policy=1)
        big = np.array([ks.capi.KS_REPLICAS_MAX], np.uint32)
        z = np.zeros(1, np.int64)
        for policy in (0, 4):
            got = check(snap, fc, fm, ac, am, lab, z, z, np.zeros((1, W), np.uint64), big,
                        np.arange(N, dtype=np.int32), N, [1], policy=policy)
            assert got[0]["placed"][0] == big[0] and got[0]["min_count"][0] == big[0] // N


def test_staging_shared_with_other_calls(ks):
    """Interleaved with ks_place_replicas and ks_scaleup_estimate on one snapshot, each result equals the same call on a
    fresh snapshot."""
    rng = np.random.default_rng(0x5A)
    N, T, W = 3000, 64, 2
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    rc, rm, sel = _specs(rng, T, W)
    dom, D = domains(rng, N, 5)
    R = rng.integers(0, 3000, T).astype(np.uint32)
    ex = rng.integers(0, 5, (T, D)).astype(np.uint32)
    spread = lambda s: s.place_replicas_spread(rc, rm, sel, R, dom, D, np.full(T, 2), None, ex, 1)
    rep = lambda s: s.place_replicas(rc, rm, sel, R * 4, 0)
    scale = lambda s: s.scaleup_estimate(rc, rm, sel, ac[:8], am[:8], ac[:8], am[:8], lab[:8], np.full(8, 20, np.uint32))

    def fresh(fn):
        with ks.Snapshot(0) as s:
            load(ks, s, fc, fm, ac, am, lab)
            return fn(s)

    want = {k: fresh(f) for k, f in (("spread", spread), ("rep", rep), ("scale", scale))}
    with ks.Snapshot(0) as s:
        load(ks, s, fc, fm, ac, am, lab)
        for step in range(2):
            for name, fn in (("spread", spread), ("rep", rep), ("spread", spread), ("scale", scale), ("spread", spread)):
                got = fn(s)
                assert all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(got, want[name])), (step, name)


def test_empty_snapshot_and_errors(ks):
    T, W = 3, 1
    rc, rm, sel = np.ones(T, np.int64), np.ones(T, np.int64), np.zeros((T, W), np.uint64)
    R = np.array([2, 0, 3], np.uint32)
    ex = np.arange(T * 2, dtype=np.uint32).reshape(T, 2)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, W), np.uint64))
        rows, node, score, _, cnt = snap.place_replicas_spread(rc, rm, sel, R, np.zeros(0, np.int32), 2, np.ones(T),
                                                               existing=ex)
        assert (rows["blocked_domain"] == -1).all() and (rows["placed"] == 0).all() and (node == -1).all()
        assert (score == 0).all() and np.array_equal(cnt, ex)
        N = 4
        fc = np.full(N, 1000, np.int64)
        load(ks, snap, fc, fc << 20, fc, fc << 20, np.zeros((N, W), np.uint64))
        dom = np.array([0, 1, -1, 0], np.int32)

        def code(**kw):
            a = dict(node_domain=dom, n_domains=2, max_skew=np.ones(T), existing=None, policy=0)
            a.update(kw)
            with pytest.raises(ks.KsError) as e:
                snap.place_replicas_spread(rc, rm, sel, R, **a)
            return e.value.code

        assert code(n_domains=0) == ks.capi.KS_ERR_RANGE
        assert code(n_domains=(1 << 20) + 1, node_domain=np.zeros(N, np.int32)) == ks.capi.KS_ERR_RANGE
        assert code(max_skew=np.array([1, 0, 1])) == ks.capi.KS_ERR_RANGE
        assert code(existing=np.full((T, 2), (1 << 24) + 1)) == ks.capi.KS_ERR_RANGE
        big_t = 65  # 65 specs x 2^20 domains of counts > 2^26
        b_rc, b_sel, b_rep = np.zeros(big_t, np.int64), np.zeros((big_t, W), np.uint64), np.ones(big_t, np.uint32)
        zeros, b_skew = np.zeros(N, np.int32), np.ones(big_t, np.uint32)
        b_out, counts = (ks.capi.ks_spread_plan * big_t)(), np.zeros(4, np.uint32)
        b_pods = ks.capi.ks_pods(big_t, b_rc.ctypes.data, b_rc.ctypes.data, b_sel.ctypes.data, ks.KS_MEM_HOST)
        b_sp = ks.capi.ks_spread(1 << 20, zeros.ctypes.data, b_skew.ctypes.data, None, None)
        assert ks.lib.ks_place_replicas_spread(snap._h, C.byref(b_pods), b_rep.ctypes.data, C.byref(b_sp), 0, b_out,
                                               None, None, counts.ctypes.data) == ks.capi.KS_ERR_RANGE
        assert (counts == 0).all()
        assert code(node_domain=np.array([0, 2, 0, 0], np.int32)) == ks.capi.KS_ERR_INVALID
        assert code(node_domain=np.array([0, -2, 0, 0], np.int32)) == ks.capi.KS_ERR_INVALID
        assert code(policy=2) == ks.capi.KS_ERR_INVALID
        out = (ks.capi.ks_spread_plan * T)()
        pods = ks.capi.ks_pods(T, rc.ctypes.data, rm.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
        assert ks.lib.ks_place_replicas_spread(snap._h, C.byref(pods), R.ctypes.data, None, 0, out, None, None,
                                               None) == ks.capi.KS_ERR_INVALID
        skew = np.ones(T, np.uint32)
        sp = ks.capi.ks_spread(2, dom.ctypes.data, skew.ctypes.data, None, None)
        dev = ks.capi.ks_pods(T, rc.ctypes.data, rm.ctypes.data, sel.ctypes.data, ks.KS_MEM_DEVICE)
        assert ks.lib.ks_place_replicas_spread(snap._h, C.byref(dev), R.ctypes.data, C.byref(sp), 0, out, None, None,
                                               None) == ks.capi.KS_ERR_INVALID
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), (fc, fc << 20)))


ZONE = "topology.kubernetes.io/zone"


def _gv1_zoned():
    g = load_golden("gv1.json")
    nodes = []
    for i, n in enumerate(g["nodes"]):
        n = dict(n)
        labels = dict(n["labels"] or {})
        if i < 4:
            labels[ZONE] = "ab"[i // 2]
        n["labels"] = labels
        nodes.append(n)
    return g, nodes


def test_host_layer_after_node_and_pod_events(ks):
    """Plans over objects equal the packed call on the exported arrays with ksh_context_topology_domains' domains, after
    node and pod events; existing-pod names that are unknown or lack the key are not counted."""
    g, nodes = _gv1_zoned()
    arena = ks.objects.ObjectArena()
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(nodes), len(nodes))
        pods = arena.pods(g["pods"])
        n = len(g["pods"])
        R = np.arange(n, dtype=np.uint32) % 7 + 1
        skew = np.arange(n, dtype=np.uint32) % 2 + 1
        for step in range(3):
            names = [ctx.node_name(i) for i in range(ctx.n_nodes)]
            existing = [[names[t % len(names)], "no-such-node", names[-1]] for t in range(n)]
            got = ctx.place_replicas_spread(pods, n, R, ZONE, skew, None, existing, step % 2)
            dom, values = ctx.topology_domains(ZONE)
            D = len(values)
            ex = np.zeros((n, D), np.uint32)
            for t, lst in enumerate(existing):
                for name in lst:
                    if name in names and dom[names.index(name)] >= 0:
                        ex[t, dom[names.index(name)]] += 1
            ac, am, lab, bn, bc, bm = ctx.export_packed()
            rc, rm, sel = ctx.pack_pods(pods, n)
            with ks.Snapshot(0) as s:
                s.set_nodes(ac, am, lab)
                s.set_bound(bn, bc, bm)
                want = s.place_replicas_spread(rc, rm, sel, R, dom, D, skew, None, ex, step % 2)
            for a, b in zip(got, want):
                assert np.array_equal(a, b), step
            if step == 0:
                ctx.remove_node(ctx.node_name(0))
            elif step == 1 and got[1][0] >= 0:
                bound = dict(g["pods"][1])
                bound["name"] = "replica-0"
                bound["node_name"] = ctx.node_name(int(got[1][0]))
                ctx.pod_bound(arena.pods([bound]))
        no_key = ctx.place_replicas_spread(pods, n, R, "no/such-key", skew)
        assert (no_key[0]["placed"] == 0).all() and (no_key[0]["blocked_domain"] == -1).all() and no_key[4] is None
