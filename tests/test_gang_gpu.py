"""Pod groups on the GPU (-m gpu): k_gang_batch through ks_gang_bind / Snapshot.gang_bind and the host layer's
ksh_reconcile_gangs, bit-exact against the CPU restatement of tests/gang_oracle.py (nodes, scores, placed, rounds and
free[] after the call), plus the equivalences the definition implies."""
import json

import numpy as np
import pytest

from gang_oracle import gang_bind_packed, groups
from helpers import load_golden

pytestmark = pytest.mark.gpu

W_KEYS = {1: 8, 2: 16, 4: 32, 8: 64}  # label words -> synth n_keys


def _cluster(ks, P, N, seed, W=1, bound_per_node=3):
    cl = ks.synth.make(P, N, seed=seed, n_keys=W_KEYS[W], bound_per_node=bound_per_node)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    return ac, am, lab, bn, bc, bm, rc, rm, sel


def _minimums(rng, off):
    """min_member per group, cycling through 0, 1, the size and a random value"""
    size = np.diff(off).astype(np.int64)
    kind = np.arange(len(size)) % 4
    rand = (rng.random(len(size)) * (size + 1)).astype(np.int64)
    return np.choose(kind, [np.zeros_like(size), np.ones_like(size), size, rand]).astype(np.uint32)


def _run_and_check(ks, orc, snap, ac, am, lab, rc, rm, sel, off, mm, policy, what=""):
    fc, fm = snap.free()
    want = gang_bind_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, off, mm, policy)
    got = snap.gang_bind(rc, rm, sel, off, mm, policy)
    for name, g, w in zip(("node_idx", "score", "placed", "rounds"), got, want):
        assert g.dtype == w.dtype and np.array_equal(g, w), f"{name} {what}"
    gc, gm = snap.free()
    assert np.array_equal(gc, fc) and np.array_equal(gm, fm), f"free {what}"
    return want


@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("N", [1, 1023, 1025, 10_007])
def test_gang_matches_restatement(ks, orc, W, N):
    P = 3000
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, P, N, 12000 + 17 * W + N, W)
    assert lab.shape[1] == W
    rng = np.random.default_rng(W * 100_003 + N)
    scale = max(1, (4 * P) // (3 * N))  # few nodes: groups compete for them and some roll back
    rc, rm = rc * min(scale, 8), rm * min(scale, 8)
    for policy in (ks.KS_SCORE_LEFTOVER, ks.KS_SCORE_LEAST_ALLOCATED):
        off = groups(rng, P, 1, 200)
        mm = _minimums(rng, off)
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            snap.set_bound(bn, bc, bm)
            _run_and_check(ks, orc, snap, ac, am, lab, rc, rm, sel, off, mm, policy, f"W={W} N={N} policy={policy}")


@pytest.mark.parametrize("policy", [0, 1])
def test_two_thousand_mixed_groups(ks, orc, policy):
    """About 100 000 pods in about 2 000 groups of 1 to 1024 pods, every kind of min_member."""
    P, N = 100_000, 2048
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, P, N, 12500 + policy)
    rng = np.random.default_rng(77 + policy)
    big = rng.random(4000) < 0.03
    sizes = np.where(big, rng.integers(65, 1025, 4000), rng.integers(1, 65, 4000))
    off = np.concatenate([[0], np.cumsum(sizes)])
    off = np.concatenate([off[off < P], [P]]).astype(np.uint64)
    assert 1500 < len(off) - 1 < 2500 and np.diff(off).max() <= 1024 and np.diff(off).min() >= 1
    mm = _minimums(rng, off)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        idx, _, placed, _ = _run_and_check(ks, orc, snap, ac, am, lab, rc, rm, sel, off, mm, policy)
    committed = placed >= mm
    assert committed.any() and (~committed).any() and (idx >= 0).any()


def test_tight_cluster_most_groups_roll_back(ks, orc):
    P, N = 4000, 300
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, P, N, 12600)
    rc, rm = rc * 8, rm * 8
    off = groups(np.random.default_rng(5), P, 4, 64)
    mm = np.diff(off).astype(np.uint32)  # all or nothing
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        _, _, placed, _ = _run_and_check(ks, orc, snap, ac, am, lab, rc, rm, sel, off, mm, 0)
    rolled = placed < mm
    assert rolled.mean() > 0.5 and (~rolled).any()


def test_all_rolled_back_leaves_free_unchanged(ks, orc):
    P, N = 2048, 1025
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, P, N, 12700)
    off = groups(np.random.default_rng(6), P, 2, 300)
    rc = rc.copy()
    rc[off[1:].astype(np.int64) - 1] = 1 << 35  # the last pod of every group fits no node
    mm = np.diff(off).astype(np.uint32)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        fc, fm = snap.free()
        idx, score, placed, rounds = snap.gang_bind(rc, rm, sel, off, mm)
        gc, gm = snap.free()
    assert (idx == -1).all() and (score == 0).all() and (placed < mm).all() and (placed > 0).any()
    assert np.array_equal(gc, fc) and np.array_equal(gm, fm)


@pytest.mark.parametrize("policy", [0, 1])
def test_one_group_without_minimum_is_stream_bind(ks, orc, policy):
    P, N = 1024, 200
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, P, N, 12800 + policy)
    rc, rm = rc * 3, rm * 3
    out = []
    for gang in (True, False):
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            snap.set_bound(bn, bc, bm)
            if gang:
                idx, score, placed, rounds = snap.gang_bind(rc, rm, sel, [0, P], [0], policy)
                r = int(rounds[0])
                assert placed[0] == (idx >= 0).sum()
            else:
                idx, score, r = snap.stream_bind(rc, rm, sel, policy)
            out.append((idx, score, r) + snap.free())
    assert out[0][2] == out[1][2] > 1
    for a, b in zip(out[0], out[1]):
        assert np.array_equal(np.asarray(a), np.asarray(b))


def test_select_after_gang_bind_sees_the_new_free(ks, orc):
    """free[] changes on the device: the bit-parallel index must be rebuilt before the next select."""
    P, N = 4096, 5000
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, P, N, 12900)
    off = groups(np.random.default_rng(9), P, 8, 256)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        before = snap.select(rc, rm, sel, flags=ks.capi.KS_SELECT_FORCE_BITPAR)  # builds the index
        idx, _, _, _ = snap.gang_bind(rc * 4, rm * 4, sel, off, np.diff(off).astype(np.uint32) // 2)
        assert (idx >= 0).sum() > 100
        fc, fm = snap.free()
        want = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, 0, want_mask=False)
        for flags in (ks.capi.KS_SELECT_FORCE_DIRECT, ks.capi.KS_SELECT_FORCE_BITPAR):
            r = snap.select(rc, rm, sel, flags=flags)
            assert np.array_equal(r.node_idx, want[0]) and np.array_equal(r.score, want[1])
            assert np.array_equal(r.feasible_cnt, want[2])
        assert not np.array_equal(before.score, want[1])


def test_empty_snapshot_places_nothing(ks):
    with ks.Snapshot(0) as snap:
        snap.set_nodes(np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 1), np.uint64))
        rc = np.ones(5, np.int64)
        idx, score, placed, rounds = snap.gang_bind(rc, rc, np.zeros((5, 1), np.uint64), [0, 2, 5], [0, 1])
    assert (idx == -1).all() and (score == 0).all() and placed.tolist() == [0, 0] and rounds.tolist() == [1, 1]


def test_gv1_golden_on_the_device(ks):
    g = load_golden("gv1.json")
    names = [p["name"] for p in g["pods"]]
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as pk:
        pk.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        pk.set_cluster_pods(arena.pods(g["bound_pods"]), len(g["bound_pods"]))
        rc, rm, sel = pk.pack_pods(arena.pods(g["pods"]), len(g["pods"]))
        ac, am, lab, bn, bc, bm = pk.export_packed()
    for case in load_golden("gv1_gang.json")["cases"]:
        order = [names.index(p) for grp in case["groups"] for p in grp["pods"]]
        off = np.cumsum([0] + [len(grp["pods"]) for grp in case["groups"]]).astype(np.uint64)
        mm = [grp["min_member"] for grp in case["groups"]]
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            snap.set_bound(bn, bc, bm)
            idx, score, placed, rounds = snap.gang_bind(rc[order], rm[order], sel[order], off, mm)
            assert idx.tolist() == case["node_idx"] and score.tolist() == case["score"], case["name"]
            assert placed.tolist() == case["placed"] and rounds.tolist() == case["rounds"], case["name"]
            fc, fm = snap.free()
            assert fc.tolist() == case["free_cpu"] and fm.tolist() == case["free_mem"], case["name"]


def _ctx_free(ks, ctx):
    h = ks.lib.ksh_context_snapshot(ctx._h)
    n = ks.lib.ks_snapshot_num_nodes(h)
    fc, fm = np.empty(n, np.int64), np.empty(n, np.int64)
    assert ks.lib.ks_snapshot_get_free(h, fc.ctypes.data, fm.ctypes.data) == 0
    return fc, fm


def _bad(ks, snap, rc, off, mm):
    with pytest.raises(ks.KsError) as e:
        snap.gang_bind(rc, rc, np.zeros((len(rc), 1), np.uint64), off, mm)
    return e.value.code


def test_argument_errors(ks):
    E = ks.capi
    with ks.Snapshot(0) as snap:
        snap.set_nodes(np.full(4, 1000, np.int64), np.full(4, 1000, np.int64), np.zeros((4, 1), np.uint64))
        rc = np.full(1025, 1000, np.int64)  # one pod fills a node
        assert _bad(ks, snap, rc[:4], [0, 2, 2, 4], [0, 0, 0]) == E.KS_ERR_RANGE  # empty group
        assert _bad(ks, snap, rc, [0, 1025], [0]) == E.KS_ERR_RANGE  # 1025 pods
        assert _bad(ks, snap, rc[:4], [0, 3, 2, 4], [0, 0, 0]) == E.KS_ERR_INVALID  # decreasing
        assert _bad(ks, snap, rc[:4], [1, 4], [0]) == E.KS_ERR_INVALID  # offset[0] != 0
        assert _bad(ks, snap, rc[:4], [0, 3], [0]) == E.KS_ERR_INVALID  # does not end at P
        assert _bad(ks, snap, rc[:4], [0, 2, 4], [3, 0]) == E.KS_ERR_RANGE  # min_member > size
        fc, fm = snap.free()
        assert fc.tolist() == [1000] * 4  # nothing ran
        idx, _, placed, rounds = snap.gang_bind(rc, rc, np.zeros((1025, 1), np.uint64), [0, 1024, 1025], [1, 1])
        assert placed.tolist() == [4, 0] and (idx >= 0).sum() == 4


def test_host_layer_matches_restatement(ks, orc):
    """ksh_reconcile_gangs on objects: bound members count toward min_member, nameless pods do not; committed pods get
    Binding bodies and join the bound list, rolled-back pods change nothing; pod_deleted returns their capacity."""
    cl = ks.synth.make(600, 30, seed=13000, bound_per_node=2)
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    pods_s = [dict(p) for p in pods_s]
    rng = np.random.default_rng(3)
    off = groups(rng, len(pods_s), 2, 30)
    G = len(off) - 1
    mm = np.diff(off).astype(np.uint32)
    mm[::3] //= 2
    first = off[:-1].astype(np.int64)
    running = first[1::4]
    for i in running:  # a running member: skipped, counts toward its group
        pods_s[i] = dict(pods_s[i], node_name="node-1")
    nameless = first[2::4] + 1
    nameless = nameless[nameless < off[1:][2::4].astype(np.int64)]
    for i in nameless:
        pods_s[i] = {"name": None, "ns": None, "containers": [{"cpu": "1m"}]}
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(nodes_s), arena.pods(bound_s), arena.pods(pods_s)
    # expectation: per group, the schedulable pods with min_member minus running members, via the restatement
    sched = [i for i in range(len(pods_s)) if i not in set(running.tolist()) | set(nameless.tolist())]
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as pk:
        pk.set_nodes(nodes, cl.N)
        pk.set_cluster_pods(bound, cl.B)
        rc, rm, sel = pk.pack_pods(arena.pods([pods_s[i] for i in sched]), len(sched))
        ac, am, lab, bn, bc, bm = pk.export_packed()
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    grp = np.searchsorted(off, np.array(sched), side="right") - 1
    s_off = np.searchsorted(grp, np.arange(G + 1)).astype(np.uint64)
    need = np.array([max(0, int(mm[g]) - int(np.isin(running, np.arange(off[g], off[g + 1])).sum())) for g in range(G)])
    status_w = np.zeros(len(pods_s), np.int32)
    node_w = np.full(len(pods_s), -1, np.int32)
    status_w[nameless] = ks.host.KSH_RECONCILE_BINDING_OBJECT_FAILED
    for g in range(G):
        a, b = int(s_off[g]), int(s_off[g + 1])
        if a == b:
            continue
        members = np.array(sched[a:b])
        if need[g] > b - a:
            status_w[members] = ks.host.KSH_RECONCILE_GANG_UNSATISFIED
            continue
        i, _, placed, _ = gang_bind_packed(orc, fc, fm, ac, am, lab, rc[a:b], rm[a:b], sel[a:b], [0, b - a], [need[g]])
        if placed[0] < need[g]:
            status_w[members] = ks.host.KSH_RECONCILE_GANG_UNSATISFIED
        else:
            node_w[members] = i
            status_w[members] = np.where(i >= 0, 0, ks.host.KSH_RECONCILE_NO_NODE_FOUND)
    assert (status_w == ks.host.KSH_RECONCILE_GANG_UNSATISFIED).any() and (node_w >= 0).any()
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, cl.N)
        ctx.set_cluster_pods(bound, cl.B)
        b0 = ctx.num_bound
        status, node, bodies, placed = ctx.reconcile_gangs(pods, len(pods_s), off, mm)
        assert np.array_equal(status, status_w) and np.array_equal(node, node_w)
        assert ctx.num_bound == b0 + (node_w >= 0).sum()
        for i in np.nonzero(node_w >= 0)[0][:40]:
            assert json.loads(bodies[i]) == {"apiVersion": "v1", "kind": "Binding",
                                             "metadata": {"name": pods_s[i]["name"], "namespace": pods_s[i].get("ns", "default")},
                                             "target": {"name": ctx.node_name(int(node_w[i]))}}
        assert all(bodies[i] is None for i in np.nonzero(node_w < 0)[0])
        assert np.array_equal(np.stack(_ctx_free(ks, ctx)), np.stack((fc, fm)))
        # deleting the committed pods returns their capacity
        done = np.nonzero(node_w >= 0)[0]
        for i in done:
            spec = dict(pods_s[i], node_name=ctx.node_name(int(node_w[i])))
            ctx.pod_deleted(arena.pods([spec]), 0)
        assert ctx.num_bound == b0
        f0 = orc.free_reduce(ac, am, bn, bc, bm)
        ctx.select_nodes(arena.pods([pods_s[sched[0]]]), 1)  # refreshes the device from the host list
        assert np.array_equal(np.stack(_ctx_free(ks, ctx)), np.stack(f0))


def test_staging_reuse_across_call_sizes(ks, orc):
    """The pinned staging block is reused while it is large enough: calls whose sizes step around a reused block (the
    output half starts 8-byte aligned after the input half) must all stay exact."""
    N = 64
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, 4096, N, 13100)
    rng = np.random.default_rng(11)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        for P, G in [(1, 1), (6, 5), (5, 5), (7, 6), (2, 1), (40, 9), (33, 33), (4096, 300), (1, 1), (4095, 301)]:
            cuts = np.sort(rng.choice(np.arange(1, P), G - 1, replace=False)) if G > 1 else np.zeros(0, np.int64)
            off = np.concatenate([[0], cuts, [P]]).astype(np.uint64)
            mm = _minimums(rng, off)
            _run_and_check(ks, orc, snap, ac, am, lab, rc[:P], rm[:P], sel[:P], off, mm, 0, f"P={P} G={G}")


def test_group_arrays_must_agree(ks):
    with ks.Snapshot(0) as snap:
        snap.set_nodes(np.full(4, 1000, np.int64), np.full(4, 1000, np.int64), np.zeros((4, 1), np.uint64))
        rc = np.ones(4, np.int64)
        sel = np.zeros((4, 1), np.uint64)
        for off, mm in (([0, 2, 4], [1]), ([0, 4], [1, 1]), ([], [])):
            with pytest.raises(ValueError):
                snap.gang_bind(rc, rc, sel, off, mm)


def test_requeued_pod_loses_its_old_charge_whatever_its_group_does(ks):
    """A pod this context bound earlier comes back unbound (its POST failed): its earlier charge is dropped whether its
    group reaches the device or is refused up front for having too few schedulable members."""
    nodes_s = [{"name": f"n{i}", "allocatable": {"cpu": "4", "memory": "8Gi"}} for i in range(2)]
    pods_s = [{"name": f"p{i}", "ns": "w", "containers": [{"cpu": "1", "memory": "1Gi"}]} for i in range(3)]
    arena = ks.objects.ObjectArena()
    nodes = arena.nodes(nodes_s)
    for refused in (False, True):
        with ks.host.Context(0) as ctx:
            ctx.set_nodes(nodes, 2)
            st, nd, _, _ = ctx.reconcile_gangs(arena.pods(pods_s), 3, [0, 3], [3])
            assert (st == 0).all() and (nd >= 0).all() and ctx.num_bound == 3
            # p0 comes back unbound.  With a member that fits no node its group goes to the device and rolls back;
            # with a nameless member it has one schedulable pod for a minimum of 2 and is refused before the device.
            other = ({"name": None, "ns": None, "containers": [{"cpu": "1m"}]} if refused else
                     {"name": "huge", "ns": "w", "containers": [{"cpu": "64", "memory": "1Gi"}]})
            st, nd, _, placed = ctx.reconcile_gangs(arena.pods([pods_s[0], other]), 2, [0, 2], [2])
            want = ks.host.KSH_RECONCILE_BINDING_OBJECT_FAILED if refused else ks.host.KSH_RECONCILE_GANG_UNSATISFIED
            assert st.tolist() == [ks.host.KSH_RECONCILE_GANG_UNSATISFIED, want] and (nd == -1).all()
            assert placed.tolist() == [0 if refused else 1]
            assert ctx.num_bound == 2, f"refused={refused}"
