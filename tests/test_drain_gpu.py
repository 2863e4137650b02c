"""Drain simulation on the GPU (-m gpu): k_drain_scan / k_drain_commit through ks_drain_check / Snapshot.drain_check and
the host layer's ksh_drain_nodes, bit-exact against the CPU restatement of tests/drain_oracle.py (placed, nodes and
scores).  After every call free[] is unchanged and ks_select on both kernel paths gives what it gave before."""
import numpy as np
import pytest

from drain_oracle import bound_candidates, drain_packed
from helpers import load_golden

pytestmark = pytest.mark.gpu

W_KEYS = {1: 8, 2: 16, 4: 32, 8: 64}  # label words -> synth n_keys
LC, LM = 1 << 36, 1 << 55


def _cluster(ks, N, seed, W=1, bound_per_node=3, P=2000):
    cl = ks.synth.make(P, N, seed=seed, n_keys=W_KEYS[W], bound_per_node=bound_per_node)
    return cl.packed()


def _candidates(rng, N, D, pods_max, P, dup=True):
    """D random candidate nodes (duplicates when dup), sizes 0..pods_max, pods drawn from P pending pods."""
    node = rng.integers(0, N, D).astype(np.int32)
    if dup and D > 1:
        node[D // 2] = node[0]
    size = rng.integers(0, pods_max + 1, D)
    off = np.concatenate([[0], np.cumsum(size)]).astype(np.uint64)
    pick = rng.integers(0, P, int(off[-1]))
    return node, off, pick


def _select_state(ks, snap, rc, rm, sel):
    out = []
    for policy in (0, 1):
        for flags in (ks.capi.KS_SELECT_FORCE_DIRECT, ks.capi.KS_SELECT_FORCE_BITPAR):
            if policy == 1 and flags == ks.capi.KS_SELECT_FORCE_BITPAR:
                continue
            r = snap.select(rc, rm, sel, policy=policy, flags=flags)
            out.append((r.node_idx, r.score, r.feasible_cnt))
    return out


def _check(ks, orc, snap, ac, am, lab, rc, rm, sel, node, off, policy, flags=0, which=None, what=""):
    fc, fm = snap.free()
    probe = slice(0, min(len(rc), 300))
    before = _select_state(ks, snap, rc[probe], rm[probe], sel[probe])
    got = snap.drain_check(rc, rm, sel, node, off, policy, flags)
    want = drain_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, node, off, policy,
                        bool(flags & ks.capi.KS_DRAIN_EXCLUDE_CANDIDATES), which)
    if which is not None:  # compare the sampled candidates only
        pods = np.concatenate([np.arange(int(off[d]), int(off[d + 1])) for d in which] + [np.zeros(0, np.int64)])
        got_c = (got[0][which], got[1][pods], got[2][pods])
        want_c = (want[0][which], want[1][pods], want[2][pods])
    else:
        got_c, want_c = got, want
    for name, g, w in zip(("placed", "node_idx", "score"), got_c, want_c):
        assert g.dtype == w.dtype and np.array_equal(g, w), f"{name} {what}"
    gc, gm = snap.free()
    assert np.array_equal(gc, fc) and np.array_equal(gm, fm), f"free changed {what}"
    after = _select_state(ks, snap, rc[probe], rm[probe], sel[probe])
    for a, b in zip(before, after):
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), f"select changed {what}"
    return got


@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("N", [1, 1023, 1025, 10_007])
def test_drain_matches_restatement(ks, orc, W, N):
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, N, 21000 + 17 * W + N, W)
    rng = np.random.default_rng(W * 1009 + N)
    rc, rm = rc * 3, rm * 3  # some candidates stop
    D = 60 if N > 1 else 4
    node, off, pick = _candidates(rng, N, D, 40, len(rc))
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        for policy in (0, 1):
            for flags in (0, ks.capi.KS_DRAIN_EXCLUDE_CANDIDATES):
                placed, _, _ = _check(ks, orc, snap, ac, am, lab, rc[pick], rm[pick], sel[pick], node, off, policy, flags,
                                      what=f"W={W} N={N} policy={policy} flags={flags}")
                if N > 1 and flags == 0:
                    size = np.diff(off)
                    assert (placed == size).any() and (placed < size).any()


def test_chunk_edges_from_the_sm_count(ks, orc):
    """One-candidate rounds split the nodes into chunks of whole tiles: N such that the last chunk holds one node, and
    such that the chunks are exact."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for N in (2 * sms * 1024 + 1, 2 * sms * 1024, 1024 * 7 + 1):
        ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, N, 21500 + N, bound_per_node=1, P=200)
        rng = np.random.default_rng(N)
        node = np.array([N - 1, 0, N // 2], np.int32)
        off = np.array([0, 6, 9, 9], np.uint64)
        pick = rng.integers(0, len(rc), 9)
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            snap.set_bound(bn, bc, bm)
            for policy in (0, 1):
                _check(ks, orc, snap, ac, am, lab, rc[pick], rm[pick], sel[pick], node, off, policy, what=f"N={N}")


@pytest.mark.parametrize("policy", [0, 1])
def test_twenty_thousand_candidates(ks, orc, policy):
    """D = 20 000 with sizes 0 to 1024 (a few large ones), checked on a seeded sample that includes the largest."""
    N = 2048
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, N, 22000 + policy, P=20000)
    rng = np.random.default_rng(5 + policy)
    D = 20_000
    size = np.where(rng.random(D) < 0.002, rng.integers(200, 1025, D), rng.integers(0, 12, D))
    size[7] = 1024
    off = np.concatenate([[0], np.cumsum(size)]).astype(np.uint64)
    node = rng.integers(0, N, D).astype(np.int32)
    pick = rng.integers(0, len(rc), int(off[-1]))
    which = sorted(set(rng.choice(D, 40, replace=False).tolist()) | {7, int(np.argmax(size[8:])) + 8})
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        placed, _, _ = _check(ks, orc, snap, ac, am, lab, rc[pick] * 2, rm[pick] * 2, sel[pick], node, off, policy,
                              ks.capi.KS_DRAIN_EXCLUDE_CANDIDATES if policy else 0, which=which)
    assert (placed == size).sum() > 1000 and (placed < size).any()


def _table(N, W, fc, fm, seed):
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, 1 << 62, (N, W), dtype=np.uint64) & ~np.uint64(1 << 63)  # bit 63 is never set
    return np.asarray(fc, np.int64), np.asarray(fm, np.int64), lab


@pytest.mark.parametrize("policy", [0, 1])
def test_deep_overlay_on_two_nodes(ks, orc, policy):
    """A 1024-pod candidate whose pods all land on the two large nodes: the overlay is deep on few nodes."""
    N = 3000
    ac = np.full(N, 1000, np.int64)
    am = np.full(N, 1 << 30, np.int64)
    ac[[5, 2900]] = 1 << 30
    am[[5, 2900]] = 1 << 45
    ac, am, lab = _table(N, 1, ac, am, 1)
    rng = np.random.default_rng(policy)
    P = 1024 + 300
    rc = rng.integers(0, 2_000_000, P)
    rm = rng.integers(1 << 31, 1 << 34, P)  # more memory than a small node has
    rc[:1024:97] = 0  # zero requests: the overlay entry keeps free[]'s cpu and ties with untouched values
    sel = (lab[rng.integers(0, N, P)] & rng.integers(0, 1 << 62, (P, 1), dtype=np.uint64))
    sel[:1024] = 0
    node = np.array([17, 2900, 17], np.int32)
    off = np.array([0, 1024, 1024 + 150, P], np.uint64)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        placed, idx, _ = _check(ks, orc, snap, ac, am, lab, rc, rm, sel, node, off, policy)
    assert placed[0] > 500 and set(idx[:int(placed[0])].tolist()) <= {5, 2900}


@pytest.mark.parametrize("policy", [0, 1])
def test_ties_across_chunks_and_overlays(ks, orc, policy):
    """Equal free values on every node, so every choice is a tie that the lower index breaks, with moves that bring an
    overlay node back level with untouched ones (requests of 0), on both sides of tile and chunk boundaries."""
    N = 9 * 1024 + 3
    ac = np.full(N, 8000, np.int64)
    am = np.full(N, 8 << 30, np.int64)
    ac, am, lab = _table(N, 2, ac, am, 2)
    lab[:] = 0
    rng = np.random.default_rng(10 + policy)
    D = 300
    node = rng.choice(np.array([0, 1, 1023, 1024, 1025, 2047, 2048, N - 1]), D).astype(np.int32)
    size = rng.integers(0, 30, D)
    off = np.concatenate([[0], np.cumsum(size)]).astype(np.uint64)
    P = int(off[-1])
    rc = rng.choice(np.array([0, 0, 1000, 4000, 8000]), P)
    rm = rng.choice(np.array([0, 0, 1 << 30, 8 << 30]), P)
    sel = np.zeros((P, 2), np.uint64)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        for flags in (0, ks.capi.KS_DRAIN_EXCLUDE_CANDIDATES):
            _check(ks, orc, snap, ac, am, lab, rc, rm, sel, node, off, policy, flags)


@pytest.mark.parametrize("policy", [0, 1])
def test_edge_values(ks, orc, policy):
    """Free at +-limit, allocatable <= 0 (LeastAllocated scores 0 for that resource), requests at the limit, and
    selectors with a bit no node carries (the candidate stops at that pod)."""
    N = 2500
    rng = np.random.default_rng(30 + policy)
    ac = rng.choice(np.array([-LC, -1, 0, 1, 1000, LC]), N)
    am = rng.choice(np.array([-LM, -1, 0, 1, 1 << 30, LM]), N)
    ac, am, lab = _table(N, 1, ac, am, 3)
    D = 120
    node, off, _ = _candidates(rng, N, D, 12, 1)
    P = int(off[-1])
    rc = rng.choice(np.array([0, 1, 1000, LC]), P)
    rm = rng.choice(np.array([0, 1, 1 << 30, LM]), P)
    sel = lab[rng.integers(0, N, P)] & rng.integers(0, 1 << 62, (P, 1), dtype=np.uint64)
    sel[rng.random(P) < 0.05, 0] |= np.uint64(1 << 63)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        placed, _, _ = _check(ks, orc, snap, ac, am, lab, rc, rm, sel, node, off, policy)
    assert (placed < np.diff(off)).any() and (placed == np.diff(off)).any()


def test_full_sweep_c2(ks, orc):
    """Every c2 node a candidate with its bound pods (each given a seeded pending pod's selector); a seeded sample against
    the restatement, and every drainable candidate's moves applied to a snapshot without its pods must fit."""
    cl = ks.synth.config("c2")
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    N = len(ac)
    order, node, off = bound_candidates(bn, N)
    rng = np.random.default_rng(0xC2)
    prc, prm = bc[order], bm[order]
    psel = np.ascontiguousarray(sel[rng.integers(0, len(rc), len(order))])
    which = sorted(rng.choice(N, 60, replace=False).tolist())
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        placed, idx, _ = _check(ks, orc, snap, ac, am, lab, prc, prm, psel, node, off, 0, which=which)
        size = np.diff(off).astype(np.uint32)
        drainable = np.nonzero(placed == size)[0]
        assert 0 < len(drainable) < N
        for d in rng.choice(drainable, 20, replace=False):
            a, b = int(off[d]), int(off[d + 1])
            keep = np.ones(len(bn), bool)
            keep[order[a:b]] = False
            snap.set_bound(bn[keep], bc[keep], bm[keep])  # the candidate's pods evicted
            for p in range(a, b):
                snap.apply_bind(int(idx[p]), int(prc[p]), int(prm[p]))
            fc, fm = snap.free()
            dest = idx[a:b]
            assert (fc[dest] >= 0).all() and (fm[dest] >= 0).all() and int(d) not in set(dest.tolist())
        snap.set_bound(bn, bc, bm)


def test_gv1_golden_on_the_device(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as pk:
        pk.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        pk.set_cluster_pods(arena.pods(g["bound_pods"]), len(g["bound_pods"]))
        specs = g["bound_pods"] + g["pods"]
        rc, rm, sel = pk.pack_pods(arena.pods(specs), len(specs))
        ac, am, lab, bn, bc, bm = pk.export_packed()
    names = [p["name"] for p in specs]
    for case in load_golden("gv1_drain.json")["cases"]:
        pick = [names.index(p) for c in case["candidates"] for p in c["pods"]]
        node = [c["node"] for c in case["candidates"]]
        off = np.cumsum([0] + [len(c["pods"]) for c in case["candidates"]]).astype(np.uint64)
        flags = ks.capi.KS_DRAIN_EXCLUDE_CANDIDATES if case["exclude_candidates"] else 0
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            snap.set_bound(bn, bc, bm)
            for policy, key in ((0, "leftover"), (1, "least_allocated")):
                placed, idx, score = snap.drain_check(rc[pick], rm[pick], sel[pick], node, off, policy, flags)
                want = case[key]
                assert placed.tolist() == want["placed"] and idx.tolist() == want["node_idx"], case["name"]
                assert score.tolist() == want["score"], case["name"]


def test_argument_errors(ks):
    E = ks.capi
    with ks.Snapshot(0) as snap:
        snap.set_nodes(np.full(4, 1000, np.int64), np.full(4, 1000, np.int64), np.zeros((4, 1), np.uint64))

        def bad(rc, node, off, policy=0, flags=0):
            with pytest.raises(ks.KsError) as e:
                snap.drain_check(rc, rc, np.zeros((len(rc), 1), np.uint64), node, off, policy, flags)
            return e.value.code

        one = np.ones(1025, np.int64)
        assert bad(one, [0], [0, 1025]) == E.KS_ERR_RANGE  # 1025 pods
        assert bad(one[:2], [0], [0, 2], flags=2) == E.KS_ERR_INVALID  # unknown flag
        assert bad(one[:2], [0], [0, 2], policy=7) == E.KS_ERR_INVALID
        assert bad(one[:2], [4], [0, 2]) == E.KS_ERR_INVALID  # node index >= N
        assert bad(one[:2], [-1], [0, 2]) == E.KS_ERR_INVALID
        assert bad(one[:3], [0, 1], [0, 2, 1]) == E.KS_ERR_INVALID  # decreasing
        assert bad(one[:2], [0], [1, 2]) == E.KS_ERR_INVALID  # offset[0] != 0
        assert bad(one[:2], [0], [0, 1]) == E.KS_ERR_INVALID  # does not end at P
        assert bad(np.array([1, -1]), [0], [0, 2]) == E.KS_ERR_RANGE  # request below 0
        assert bad(np.array([1, LC + 1]), [0], [0, 2]) == E.KS_ERR_RANGE
        with pytest.raises(ValueError):
            snap.drain_check(one[:2], one[:2], np.zeros((2, 1), np.uint64), [0, 1], [0, 2])
        fc, _ = snap.free()
        assert fc.tolist() == [1000] * 4
        placed, idx, score = snap.drain_check(one[:0], one[:0], np.zeros((0, 1), np.uint64), [], [0])
        assert len(placed) == 0 and len(idx) == 0
        # 1024 is allowed; candidates without pods are drainable
        placed, idx, _ = snap.drain_check(np.full(1024, 1, np.int64), np.full(1024, 1, np.int64),
                                          np.zeros((1024, 1), np.uint64), [0, 1, 2], [0, 1024, 1024, 1024])
        assert placed.tolist() == [1024, 0, 0] and set(idx.tolist()) == {1, 2, 3}


def _objects(ks, N=40, seed=23000):
    cl = ks.synth.make(300, N, seed=seed, bound_per_node=4)
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    return cl, nodes_s, bound_s, pods_s


def _grouped(bound_s, names):
    """The bound pods of the named nodes, grouped by node, and the offsets"""
    specs, off = [], [0]
    for n in names:
        specs += [b for b in bound_s if b["node_name"] == n]
        off.append(len(specs))
    return specs, np.array(off, np.uint64)


def test_host_layer_matches_packed_call(ks, orc):
    """ksh_drain_nodes over objects equals ks_drain_check on the same packed pods, also after node and pod events; it
    refuses pods bound elsewhere and unknown node names."""
    cl, nodes_s, bound_s, pods_s = _objects(ks)
    arena = ks.objects.ObjectArena()
    names = [f"node-{i}" for i in (3, 0, 17, 3, 39)]
    specs, off = _grouped(bound_s, names)
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(nodes_s), cl.N)
        ctx.set_cluster_pods(arena.pods(bound_s), cl.B)

        def both(flags=0):
            pods = arena.pods(specs)
            placed, node = ctx.drain_nodes(names, pods, off, 0, flags)
            rc, rm, sel = ctx.pack_pods(pods, len(specs))
            snap_h = ks.lib.ksh_context_snapshot(ctx._h)
            by_name = {ctx.node_name(i): i for i in range(ctx.n_nodes)}
            idx_map = [by_name[n] for n in names]
            n_nodes = ks.lib.ks_snapshot_num_nodes(snap_h)
            fc, fm = np.empty(n_nodes, np.int64), np.empty(n_nodes, np.int64)
            assert ks.lib.ks_snapshot_get_free(snap_h, fc.ctypes.data, fm.ctypes.data) == 0
            ac, am, lab, bn, bc, bm = ctx.export_packed()
            want = drain_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, idx_map, off, 0,
                                bool(flags & ks.capi.KS_DRAIN_EXCLUDE_CANDIDATES))
            assert np.array_equal(placed, want[0]) and np.array_equal(node, want[1])
            return placed, node

        both()
        both(ks.capi.KS_DRAIN_EXCLUDE_CANDIDATES)
        # events: a node grows, a pod binds to node-0, a bound pod of node-17 goes away
        grown = dict(nodes_s[5], allocatable={"cpu": "512", "memory": str(1 << 40)})
        ctx.upsert_node(arena.nodes([grown]), 0)
        extra = {"name": "late", "ns": "load", "node_name": "node-0", "containers": [{"cpu": "100m", "memory": "1Mi"}]}
        ctx.pod_bound(arena.pods([extra]), 0)
        gone = [b for b in bound_s if b["node_name"] == "node-17"][0]
        ctx.pod_deleted(arena.pods([gone]), 0)
        bound_s = [b for b in bound_s if b is not gone] + [extra]
        specs, off = _grouped(bound_s, names)
        placed, node = both()
        assert 5 in set(node.tolist())  # the grown node is the best destination now
        # mis-grouped pods and unknown names
        with pytest.raises(ks.KsError) as e:
            ctx.drain_nodes(names[:2], arena.pods(specs), np.array([0, int(off[2]) - 1, int(off[2])], np.uint64))
        assert e.value.code == ks.capi.KS_ERR_INVALID and "spec.nodeName" in str(e.value)
        with pytest.raises(ks.KsError) as e:
            ctx.drain_nodes(["node-3", "no-such-node"], arena.pods(specs), np.array([0, int(off[1]), int(off[1])], np.uint64))
        assert e.value.code == ks.capi.KS_ERR_INVALID and "no-such-node" in str(e.value)
