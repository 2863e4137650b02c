"""Soft constraints when binding (ks_profile_bind) on the H100: node, total, parts, both refusals, hard and soft
counts and the final free[] bit for bit against tests/profile_bind_oracle.py across label widths, policies 1, 3 and 4,
1 to 4 keys with hard, soft and both on one key, node counts at the CTA-slice edges, existing pods, duplicate and self
terms of all four kinds, 4 096 groups and 150 000 nodes; J1 and J2 against ks_affinity_bind on the device; errors
leaving free[] unchanged; the empty snapshot; and a following ks_select on both kernel paths."""
import numpy as np
import pytest

from affinity_bind_oracle import AFFINITY, ANTI
from profile_bind_oracle import ANTI_PREFERRED, PREFERRED, profile_bind_packed
from test_replicas_gpu import _nodes, _specs, load
from test_spread_bind_gpu import key_set, mixed_queue
from test_spread_gpu import D_SEED, zone_labels

pytestmark = pytest.mark.gpu

POLICIES = (1, 3, 4)


def check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms=(), ex_pods=None, skew=None, mind=None,
          ex=None, policy=4, **scoring):
    got = snap.profile_bind(rc, rm, sel, group, G, keys, terms, ex_pods, skew, mind, ex, policy, **scoring)
    ofc, ofm = fc.copy(), fm.copy()
    want = profile_bind_packed(ofc, ofm, ac, am, lab, rc, rm, sel, group, G, keys, terms, ex_pods, skew, mind, ex,
                               policy, **scoring)
    for i in range(4):
        assert np.array_equal(got[i], want[i]), (i, np.nonzero((got[i] != want[i]).reshape(len(rc), -1))[0][:8])
    for i in (4, 5):
        if got[i] is not None:
            assert all(np.array_equal(a, b) for a, b in zip(got[i], want[i])), i
    gfc, gfm = snap.free()
    assert np.array_equal(gfc, ofc) and np.array_equal(gfm, ofm)
    return got


def random_terms(rng, G, K, T, hot=4):
    """T terms of all four kinds over the first `hot` groups mostly, self and cross targets, with weights; then one
    exact duplicate and one self preferred anti-affinity term."""
    terms, weights = [], []
    for _ in range(T):
        owner = int(rng.integers(0, min(G, hot))) if rng.random() < 0.8 else int(rng.integers(0, G))
        kind = int(rng.choice([AFFINITY, ANTI, PREFERRED, ANTI_PREFERRED], p=[0.1, 0.2, 0.35, 0.35]))
        tg = sorted(set(rng.integers(0, min(G, hot), int(rng.integers(1, 3))).tolist()))
        terms.append((owner, kind, int(rng.integers(0, K)), tg))
        weights.append(int(rng.integers(1, 101)) if kind >= PREFERRED else 0)
    if terms:
        terms.append(terms[0])
        weights.append(weights[0])
        terms.append((0, ANTI_PREFERRED, K - 1, [0]))
        weights.append(100)
    return terms, weights


def soft_setup(rng, G, K):
    soft = np.array([0, 1, 3, 5], np.uint32)[rng.integers(0, 4, (G, K))]
    soft[rng.random(G) < 0.25] = 0  # some groups without soft constraints
    return soft, (rng.random(G) < 0.5).astype(np.uint8)


CASES = [  # (W, N, key modes, groups, pods, terms)
    (1, 1, (1,), 3, 20, 3),
    (2, 127, (3, "host"), 4, 100, 5),
    (4, 128, (3,), 5, 100, 6),
    (8, 129, ("host",), 3, 80, 4),
    (1, 2100, ("edge", "host"), 6, 100, 6),
    (2, 3000, (3, 7, "host"), 6, 100, 8),
    (4, 16896, (7, 3, 5, "host"), 6, 60, 8),
    (8, 16897, (3,), 6, 60, 5),
]


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("case", CASES, ids=[f"W{c[0]}-N{c[1]}-" + "+".join(map(str, c[2])) for c in CASES])
def test_against_the_oracle(ks, case, policy):
    W, N, modes, G, P, T = case
    rng = np.random.default_rng([W, N, len(modes), policy, 0x50F] + [D_SEED.get(str(m), 5) for m in modes])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, modes)
    lab = zone_labels(lab, *keys[0])
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 3000), mem=(0, 12 << 30))
    terms, tw = random_terms(rng, G, len(keys), T)
    soft, soft_all = soft_setup(rng, G, len(keys))
    E = int(rng.integers(0, 2 * G + 1))
    ex_pods = (rng.integers(0, G, E), rng.integers(0, N, E))
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got = check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms, ex_pods, skew, mind, ex, policy,
                    soft_skew=soft, soft_all_keys=soft_all, term_weight=tw, hard_affinity_weight=int(rng.integers(0, 3)))
        load(ks, snap, fc, fm, ac, am, lab)  # soft only, on the same keys as the hard constraints
        check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, [], None, None, None, ex, policy,
              soft_skew=skew, soft_all_keys=np.zeros(G, np.uint8))
    if N > 1:
        assert (got[0] >= 0).any() and (got[2][:, 1] != 100).any()


def test_many_groups(ks):
    rng = np.random.default_rng(0x50F10)
    N, W, G, P = 400, 2, 4096, 120
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (5, "host"))
    hot = rng.choice(G, 12, replace=False)
    group = hot[rng.integers(0, 12, P)].astype(np.int32)
    group[rng.random(P) < 0.1] = -1
    rc, rm, _ = _specs(rng, P, W, cpu=(0, 3000), mem=(0, 8 << 30))
    sel = np.zeros((P, W), np.uint64)
    terms = [(int(hot[i]), (ANTI, PREFERRED, ANTI_PREFERRED)[i % 3], i % 2, [int(hot[(i + 1) % 12]), int(hot[i])])
             for i in range(12)]
    tw = [0 if t[1] < 2 else 37 for t in terms]
    soft = np.zeros((G, 2), np.uint32)
    soft[hot] = [5, 3]
    ex_pods = (rng.integers(0, G, 300), rng.integers(0, N, 300))
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms, ex_pods, policy=4, soft_skew=soft,
              soft_all_keys=np.zeros(G, np.uint8), term_weight=tw)


def test_150k_nodes(ks):
    rng = np.random.default_rng(0x50F11)
    N, W, G, P = 150_000, 1, 6, 30
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3, "host"))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P)
    terms = [(0, ANTI_PREFERRED, 1, [0]), (1, PREFERRED, 0, [0]), (2, ANTI, 0, [3]), (4, AFFINITY, 0, [4])]
    soft = np.tile(np.array([[5, 3]], np.uint32), (G, 1))
    ex_pods = (np.array([0, 3, 0]), np.array([5, 149_999, 77_777]))
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms, ex_pods, skew, None, ex, 1,
              soft_skew=soft, soft_all_keys=np.zeros(G, np.uint8), term_weight=[100, 40, 0, 0])


@pytest.mark.parametrize("policy", POLICIES)
def test_j1_j2_against_affinity_bind(ks, policy):
    """J1: no soft term and hard_affinity_weight 0 is ks_affinity_bind (parts = (score, 0, 0)).  J2: soft terms on a
    one-domain key bind the same nodes, 100 * weight_spread higher for a group with soft keys."""
    rng = np.random.default_rng(0x50F12 + policy)
    N, W, G, P = 3000, 2, 5, 120
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (4, "host")) + [(np.zeros(N, np.int32), 1)]
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 3000), mem=(0, 12 << 30))
    terms = [(0, ANTI, 1, [0]), (1, AFFINITY, 0, [1, 2])]
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        want = snap.affinity_bind(rc, rm, sel, group, G, keys, terms, None, skew, mind, ex, policy)
        want_free = snap.free()
        load(ks, snap, fc, fm, ac, am, lab)
        got = snap.profile_bind(rc, rm, sel, group, G, keys, terms, None, skew, mind, ex, policy,
                                hard_affinity_weight=0)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert np.array_equal(got[3], want[2]) and all(np.array_equal(a, b) for a, b in zip(got[4], want[3]))
        assert np.array_equal(got[2][:, 0], np.where(got[0] >= 0, got[1], 0)) and not got[2][:, 1:].any()
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), want_free))
        soft = np.zeros((G, 3), np.uint32)
        soft[:, 2] = rng.integers(0, 3, G)
        load(ks, snap, fc, fm, ac, am, lab)
        got = snap.profile_bind(rc, rm, sel, group, G, keys, terms + [(2, PREFERRED, 2, [3])], None, skew, mind, ex,
                                policy, soft_skew=soft, term_weight=[0, 0, 60], hard_affinity_weight=0)
        has = np.array([g >= 0 and soft[g].any() for g in group]) & (got[0] >= 0)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1] + 200 * has)
        assert not got[2][:, 2].any()


def test_errors_leave_free_unchanged(ks):
    rng = np.random.default_rng(0x50F13)
    N, W, G, P = 200, 1, 3, 10
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3,))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P)
    bad = [
        dict(policy=0), dict(policy=2),
        dict(weight_spread=101), dict(weight_affinity=101), dict(hard_affinity_weight=101),
        dict(terms=[(0, 4, 0, [1])], term_weight=[1]),
        dict(terms=[(0, PREFERRED, 0, [1])], term_weight=[0]),
        dict(terms=[(0, PREFERRED, 0, [1])], term_weight=[101]),
        dict(terms=[(0, ANTI, 0, [1])], term_weight=[5]),
        dict(soft_all_keys=np.full(G, 2, np.uint8)),
    ]
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        for kw in bad:
            kw = dict(kw)
            terms = kw.pop("terms", ())
            policy = kw.pop("policy", 4)
            with pytest.raises(ks.KsError) as e:
                snap.profile_bind(rc, rm, sel, group, G, keys, terms, None, skew, None, None, policy, **kw)
            assert e.value.code == ks.capi.KS_ERR_INVALID, kw
            got = snap.free()
            assert np.array_equal(got[0], fc) and np.array_equal(got[1], fm), kw
        # kinds 2 and 3 stay refused by ks_affinity_bind
        with pytest.raises(ks.KsError) as e:
            snap.affinity_bind(rc, rm, sel, group, G, keys, [(0, PREFERRED, 0, [1])], None, skew)
        assert e.value.code == ks.capi.KS_ERR_INVALID


def test_empty_snapshot_and_following_select(ks, orc):
    rng = np.random.default_rng(0x50F14)
    N, W, G, P = 1000, 1, 3, 40
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (3, "host"))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P)
    soft = np.full((G, 2), 2, np.uint32)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac[:0], am[:0], lab[:0])
        got = snap.profile_bind(rc, rm, sel, group, G, [(d[:0], n) for d, n in keys], (), None, skew, None, ex, 4,
                                soft_skew=soft)
        assert (got[0] == -1).all() and not got[1].any() and not got[2].any() and not got[3].any()
        for c in (got[4], got[5]):
            assert all(np.array_equal(a, np.asarray(b, np.uint32)) for a, b in zip(c, ex))
        for flags in (ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR):
            load(ks, snap, fc, fm, ac, am, lab)
            check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, [], None, skew, None, ex, 3,
                  soft_skew=soft)
            ofc, ofm = snap.free()
            want = orc.run_packed(ofc, ofm, ac, am, lab, rc, rm, sel, policy=1, want_mask=False)[:2]
            r = snap.select(rc, rm, sel, policy=ks.KS_SCORE_LEAST_ALLOCATED, flags=flags)
            assert np.array_equal(r.node_idx, want[0]) and np.array_equal(r.score, want[1]), r.path


from test_profile_bind import assert_golden, golden_runs, run_oracle  # noqa: E402


@pytest.mark.parametrize("run", list(golden_runs()), ids=lambda r: r[0])
def test_golden_on_the_device(ks, run):
    """The hand-derived queues of tests/golden/gv1_profile_bind.json: the .5 round, the empty-value domain, the ignored
    node, the self term counted twice, hard_affinity_weight and soft/hard counts diverging, on the kernel."""
    name, a, scoring, want = run
    with ks.Snapshot(0) as snap:
        load(ks, snap, a["fc"], a["fm"], a["ac"], a["am"], a["lab"])
        got = snap.profile_bind(a["rc"], a["rm"], a["sel"], a["group"], a["G"], a["keys"], a["terms"], a["ex_pods"],
                                a["skew"], None, a["ex"], a["policy"], **scoring)
        assert_golden([got[0], got[1], got[2], None, got[4], got[5]], want, name)
        ofc, ofm = run_oracle(a, scoring)[1]
        assert all(np.array_equal(x, y) for x, y in zip(snap.free(), (ofc, ofm)))


def rack_keys(rng, N, racks):
    """A rack-like key of `racks` domains per 3 nodes or fewer, none per node, and about 3% of nodes without it."""
    d = (np.arange(N) // 3 % racks).astype(np.int32) if racks * 3 < N else (np.arange(N) // 3).astype(np.int32)
    d[rng.random(N) < 0.03] = -1
    return d, int(d.max()) + 1


@pytest.mark.parametrize("soft_all", (0, 1))
@pytest.mark.parametrize("policy", (1, 4))
def test_many_domain_soft_keys(ks, soft_all, policy):
    """Distinct-domain counting on keys that are not one node per domain: about 100 rack domains (shared-bitmap words
    0-3), and N = 16 897 with d = n // 3 (5 633 domains: shared words 0-63 and the direct global bitmap above 2 047),
    60 pods so both bitmap parities are cleared and reused many times."""
    rng = np.random.default_rng([0x50F20, soft_all, policy])
    N, W, G, P = 16_897, 1, 5, 60
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = [rack_keys(rng, N, 100), rack_keys(rng, N, N), key_set(rng, N, (3,))[0]]
    assert keys[0][1] == 100 and keys[1][1] > 5000
    group = rng.integers(-1, G, P).astype(np.int32)
    rc, rm, _ = _specs(rng, P, W, cpu=(0, 3000), mem=(0, 12 << 30))
    sel = np.zeros((P, W), np.uint64)
    soft = rng.choice(np.array([0, 1, 3], np.uint32), (G, 3))
    soft[:, :2] = np.maximum(soft[:, :2], 1)  # every group spreads softly over both rack keys
    ex = [rng.integers(0, 3, (G, D)).astype(np.uint32) for _, D in keys]
    terms = [(0, ANTI_PREFERRED, 1, [0]), (1, PREFERRED, 0, [2])]
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got = check(snap, fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, terms, None, None, None, ex, policy,
                    soft_skew=soft, soft_all_keys=np.full(G, soft_all, np.uint8), term_weight=[60, 30])
    assert (got[0] >= 0).sum() > P // 2 and len(set(got[2][:, 1].tolist())) > 2


@pytest.mark.parametrize("policy", POLICIES)
def test_j3_on_the_device(ks, policy):
    """J3: "g preferred-(anti-)affine to h" and "h preferred-(anti-)affine to g" bind the queue the same way."""
    rng = np.random.default_rng(0x50F21 + policy)
    N, W, G, P = 3000, 1, 4, 100
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (5, "host"))
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 3000), mem=(0, 12 << 30))
    ex_pods = (rng.integers(0, G, 6), rng.integers(0, N, 6))
    for kind, k in ((PREFERRED, 0), (ANTI_PREFERRED, 1)):
        runs = []
        for t in ((1, kind, k, [2]), (2, kind, k, [1])):
            with ks.Snapshot(0) as snap:
                load(ks, snap, fc, fm, ac, am, lab)
                got = snap.profile_bind(rc, rm, sel, group, G, keys, [t], ex_pods, skew, None, ex, policy,
                                        term_weight=[77])
                runs.append(got[:4] + (snap.free(),))
        for x, y in zip(*runs):
            if isinstance(x, tuple):
                assert all(np.array_equal(a, b) for a, b in zip(x, y))
            else:
                assert np.array_equal(x, y)
        assert runs[0][2][:, 2].any()


def test_count_cap_leaves_free_unchanged(ks):
    """KS_ERR_RANGE for groups x domains above 2^26 (the bound that also caps the IPA counter words, which never exceed
    groups x domains), before free[] changes."""
    rng = np.random.default_rng(0x50F22)
    N, W, G = 100, 1, 65
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    D = 1 << 20
    keys = [(np.arange(N, dtype=np.int32), D)]
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        with pytest.raises(ks.KsError) as e:
            snap.profile_bind([1000], [1 << 30], np.zeros((1, 1), np.uint64), [0], G, keys,
                              [(g, PREFERRED, 0, [g]) for g in range(G)], term_weight=[1] * G, want_counts=False)
        assert e.value.code == ks.capi.KS_ERR_RANGE
        got = snap.free()
        assert np.array_equal(got[0], fc) and np.array_equal(got[1], fm)


def test_host_layer(ks):
    """ksh_reconcile_profile equals ks_profile_bind on the packed arrays over the pods that go to the device, with the
    statuses of ksh_reconcile_affinity, Binding bodies, the bound list and the charged snapshot."""
    import json
    from test_affinity_bind_gpu import HOST, ZONE, _objects
    from test_spread_gpu import _gv1_zoned
    g, nodes = _gv1_zoned()
    nodes, objs = _objects(g, nodes)
    group = np.array([i % 3 for i in range(12)], np.int32)
    skew = np.array([[1, 0], [0, 0], [0, 0]], np.uint32)
    terms = [(0, ANTI_PREFERRED, 1, [0]), (1, ANTI, 1, [1]), (2, PREFERRED, 0, [0])]
    tw = [100, 0, 50]
    soft = np.array([[5, 3], [5, 3], [0, 0]], np.uint32)
    sall = np.array([0, 0, 1], np.uint8)
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
            want = s.profile_bind(rc, rm, sel, group[todo], 3, keys, terms, ([1] * 4, list(range(4))), skew,
                                  soft_skew=soft, soft_all_keys=sall, term_weight=tw)
            want_free = s.free()
        bound0 = ctx.num_bound
        status, node, bodies = ctx.reconcile_profile(arena.pods(objs), 12, group, 3, [ZONE, HOST], terms,
                                                     existing_pods, skew, soft_skew=soft, soft_all_keys=sall,
                                                     term_weight=tw)
        assert status[4] == ks.host.KSH_RECONCILE_OK and node[4] == -1 and bodies[4] is None
        assert status[7] == ks.host.KSH_RECONCILE_BINDING_OBJECT_FAILED and node[7] == -1
        assert np.array_equal(node[todo], want[0])
        for k, i in enumerate(todo):
            if want[0][k] >= 0:
                assert status[i] == ks.host.KSH_RECONCILE_OK
                body = json.loads(bodies[i])
                assert body["kind"] == "Binding" and body["target"]["name"] == names[want[0][k]]
            elif want[3][k, 0] > 0:
                assert status[i] == ks.host.KSH_RECONCILE_SPREAD_UNSATISFIED
            elif want[3][k, 1] > 0:
                assert status[i] == ks.host.KSH_RECONCILE_AFFINITY_UNSATISFIED
            else:
                assert status[i] == ks.host.KSH_RECONCILE_NO_NODE_FOUND
        placed = int((want[0] >= 0).sum())
        assert ctx.num_bound == bound0 + placed and placed > 0
        exp = ctx.export_packed()
        with ks.Snapshot(0) as s:
            s.set_nodes(*exp[:3])
            s.set_bound(*exp[3:])
            f = s.free()
        assert np.array_equal(f[0], want_free[0]) and np.array_equal(f[1], want_free[1])
