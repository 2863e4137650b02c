"""The GPU tests of KS_SCORE_MOST_ALLOCATED (3, bin-packing) and KS_SCORE_LEAST_BALANCED (4, upstream's default resource
scoring), written once for both policies: every call that takes a policy, bit for bit against the CPU restatement of
tests/policy_oracle.py: ks_select (per-cell kernel, the bit-parallel k_most_alloc / k_least_balanced, AUTO),
ks_select_topk, ks_stream_bind on both loops, the ks_stream surface, ks_gang_bind with rollback, ks_drain_check,
ks_place_replicas (prefix fill under 3, one copy at a time under 4) and the object-level host layer; and the walk of
k_most_alloc / k_least_balanced at its exits, at its length extremes and across graph replays and policy changes.

tests/test_most_allocated_gpu.py and tests/test_least_balanced_gpu.py collect these tests under their policy (a
`policy` fixture) and add the tests that hold for one policy only."""
import numpy as np
import pytest

from drain_oracle import bound_candidates, drain_packed
from gang_oracle import gang_bind_packed, groups
from gang_oracle import sequential_packed as one_at_a_time
from policy_oracle import (EDGES, LEAST_BALANCED, MOST_ALLOCATED, PLAN, Oracle, exit_tie_cluster, topk_packed,
                           walk_extreme_clusters)

__all__ = ["pytestmark", "o", "cluster", "snapshot", "assert_refused"]  # + every test_ function, below
pytestmark = pytest.mark.gpu
SCORE_MAX = {MOST_ALLOCATED: 100, LEAST_BALANCED: 200}


def cluster(seed, N, P, W=1, family="mixed"):
    """Random packed cluster: (free_cpu, free_mem, alloc_cpu, alloc_mem, labels[N,W], req_cpu, req_mem, sel[P,W])."""
    rng = np.random.default_rng(seed)
    ac = rng.choice([4000, 8000, 16000, 32000, 96000], N).astype(np.int64)  # c3-like 4 to 96 cores
    am = rng.choice([4, 16, 64, 384], N).astype(np.int64) << 30
    fc = (ac * rng.integers(0, 17, N) // 16).astype(np.int64)
    fm = (am * rng.integers(0, 17, N) // 16).astype(np.int64)
    rc = rng.choice([0, 100, 250, 500, 1000, 4000], P).astype(np.int64)
    rm = rng.choice([0, 1 << 27, 1 << 30, 1 << 32], P).astype(np.int64)
    if family == "ties":  # few distinct nodes: many equal scores, ties to the lowest index
        k = rng.integers(0, 3, N)
        ac, am, fc, fm = ac[k], am[k], fc[k], fm[k]
    elif family == "edges":  # allocatable <= 0, free above allocatable, free at the limits, zero requests
        ac[rng.random(N) < 0.1] = 0
        am[rng.random(N) < 0.1] = -(1 << 20)
        over = rng.random(N) < 0.15
        fc[over], fm[over] = ac[over] + 4000, am[over] + (1 << 33)
        top = rng.random(N) < 0.05
        fc[top], fm[top], ac[top], am[top] = 1 << 36, 1 << 55, 1 << 36, 1 << 55
        rc[rng.random(P) < 0.3] = 0
        rm[rng.random(P) < 0.3] = 0
    lab = rng.integers(0, 1 << 16, (N, W)).astype(np.uint64) | (rng.integers(0, 1 << 16, (N, W)).astype(np.uint64) << 40)
    sel = np.zeros((P, W), np.uint64)
    w = rng.random(P) < 0.4
    sel[w, rng.integers(0, W, int(w.sum()))] = np.uint64(1) << rng.integers(0, 16, int(w.sum())).astype(np.uint64)
    return fc, fm, ac, am, lab, rc, rm, sel


def snapshot(ks, fc, fm, ac, am, lab):
    """A snapshot whose free[] is fc / fm: one bound pod per node carries alloc - free."""
    s = ks.Snapshot(0)
    s.set_nodes(ac, am, lab)
    s.set_bound(np.arange(len(ac), dtype=np.int32), ac - fc, am - fm)
    got = s.free()
    assert np.array_equal(got[0], fc) and np.array_equal(got[1], fm)
    return s


@pytest.fixture(scope="module")
def o(orc):
    return Oracle(orc)


CASES = [  # (seed, N, P, W, family)
    (1, 1, 1, 1, "mixed"), (2, 1023, 1, 1, "mixed"), (3, 1025, 7, 2, "edges"), (4, 3000, 40, 4, "ties"),
    (5, 5001, 130, 8, "mixed"), (6, 777, 1500, 1, "edges"), (7, 20000, 3, 1, "ties"), (8, 4097, 600, 2, "mixed"),
    (9, 10000, 512, 1, "mixed"),  # C2's node count
    (10, 150_000, 300, 1, "mixed"),  # more column blocks than SMs: every CTA walks several column blocks
    (12, 12_000, 200, 8, "edges"),  # W = 8 over 6 column blocks of 8 tiles
]


@pytest.mark.parametrize("seed,N,P,W,family", CASES)
def test_select_both_paths_and_auto(ks, o, policy, seed, N, P, W, family):
    fc, fm, ac, am, lab, rc, rm, sel = cl = cluster(seed, N, P, W, family)
    w_idx, w_score, w_cnt, w_mask, _ = o.run_packed(*cl, policy)
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        for flags in (ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR, ks.KS_SELECT_AUTO,
                      ks.KS_SELECT_FORCE_BITPAR | ks.KS_SELECT_NO_GRAPH):
            r = s.select(rc, rm, sel, policy=policy, flags=flags, want_mask=True)
            if flags & (ks.KS_SELECT_FORCE_DIRECT | ks.KS_SELECT_FORCE_BITPAR):
                assert r.path == ("direct" if flags & ks.KS_SELECT_FORCE_DIRECT else "bitpar")
            assert np.array_equal(r.node_idx, w_idx) and np.array_equal(r.score, w_score), flags
            assert np.array_equal(r.feasible_cnt, w_cnt) and np.array_equal(r.mask, w_mask), flags
            lo = s.select(rc, rm, sel, policy=ks.KS_SCORE_LEFTOVER, flags=flags, want_mask=True)
            assert np.array_equal(r.mask, lo.mask) and np.array_equal(r.feasible_cnt, lo.feasible_cnt)
        if N > 1000 and family == "mixed":
            assert (w_idx >= 0).sum() > 0
        assert np.array_equal(s.free()[0], fc) and np.array_equal(s.free()[1], fm)  # nothing charged


def test_negative_requests_scan_every_tile(ks, o, policy):
    """A negative request voids the early-exit bound of the bit-parallel walk: the pod scans every tile, still exact."""
    fc, fm, ac, am, lab, rc, rm, sel = cl = cluster(13, 6000, 300, 2, "edges")
    rng = np.random.default_rng(13)
    rc[rng.random(300) < 0.2] = -500
    rm[rng.random(300) < 0.2] = -(1 << 30)
    w = o.run_packed(*cl, policy, want_mask=False)
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        for flags in (ks.KS_SELECT_FORCE_BITPAR, ks.KS_SELECT_FORCE_DIRECT):
            r = s.select(rc, rm, sel, policy=policy, flags=flags)
            assert np.array_equal(r.node_idx, w[0]) and np.array_equal(r.score, w[1]) and np.array_equal(r.feasible_cnt, w[2])


def _both_paths(ks, s, cl, want, policy, tag):
    rc, rm, sel = cl[5:]
    for flags in (ks.KS_SELECT_FORCE_BITPAR, ks.KS_SELECT_FORCE_DIRECT):
        r = s.select(rc, rm, sel, policy=policy, flags=flags)
        assert r.path == ("bitpar" if flags == ks.KS_SELECT_FORCE_BITPAR else "direct")
        assert np.array_equal(r.node_idx, want[0]) and np.array_equal(r.score, want[1]), (tag, r.path)
        assert np.array_equal(r.feasible_cnt, want[2]), (tag, r.path)


@pytest.mark.parametrize("edge", list(EDGES))
def test_exit_ties(ks, o, policy, edge):
    """Ties exactly at the walk's early exit (exit_tie_cluster; tests/policy_suite.py shows with the walk model that each
    cluster reaches its boundary): Y comes right after X in bound order, has the lower index, and scores as X and as the
    limit of its tile, so the walk must not stop in front of Y's tile and Y wins.  Mirror: Y scores one lower, the walk
    stops there and X wins."""
    for mirror in (False, True):
        cl, x, y = exit_tie_cluster(policy, edge, mirror, seed=EDGES[edge][1])
        w = o.run_packed(*cl, policy, want_mask=False)
        assert (w[0] == (x if mirror else y)).all()
        with snapshot(ks, *cl[:5]) as s:
            _both_paths(ks, s, cl, w, policy, (edge, mirror))


def test_walk_length_extremes(ks, o, policy):
    """walk_extreme_clusters: pods that walk every window, nodes stored at 2^62 scattered through the table, allocatables
    <= 0, a saturated D (exhaustive walks) and the tightest D (all allocatables equal)."""
    for name, cl in walk_extreme_clusters(policy, seed=policy):
        w = o.run_packed(*cl, policy, want_mask=False)
        assert (w[0] >= 0).sum() > 40, name
        with snapshot(ks, *cl[:5]) as s:
            _both_paths(ks, s, cl, w, policy, name)


def test_graph_replay_and_alternating_policies(ks, o, policy):
    """The bound orders of policies 3 and 4 are built outside the captured CUDA graph (bitpar_prepare_order).  A
    replayed call sees a bind and new pod values in the same device buffers, and calls under policies 1, 3, 4, 3, 4 on
    one snapshot, with binds between them, each see the current free[]: every result against the oracle."""
    import torch
    fc, fm, ac, am, lab, rc, rm, sel = cluster(90, 6000, 2000, 2)
    P = len(rc)
    dev = torch.device("cuda:0")
    t = [torch.from_numpy(np.ascontiguousarray(a.view(np.int64))).to(dev) for a in (rc, rm, sel)]
    idx = torch.empty(P, dtype=torch.int32, device=dev)
    score = torch.empty(P, dtype=torch.int64, device=dev)
    cnt = torch.empty(P, dtype=torch.int32, device=dev)
    st = torch.cuda.Stream()
    with snapshot(ks, fc, fm, ac, am, lab) as s:

        def check(q, req_cpu, tag):
            s.select_raw(P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, idx, score, cnt, ks.KS_MEM_DEVICE, policy=q,
                         flags=ks.KS_SELECT_FORCE_BITPAR, stream=st.cuda_stream)
            st.synchronize()
            assert s.last_path() == "bitpar"
            f = s.free()
            w = o.run_packed(f[0], f[1], ac, am, lab, req_cpu, rm, sel, q, want_mask=False)
            got = idx.cpu().numpy(), score.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)
            assert all(np.array_equal(a, b) for a, b in zip(got, w[:3])), tag
            return w[0]

        first = None
        for it in range(3):  # capture, replay, replay
            first = check(policy, rc, ("replay", it))
        s.apply_bind(int(first[first >= 0][0]), 10_000_000, 1 << 40)
        assert not np.array_equal(check(policy, rc, "after a bind"), first)
        rc2 = rc.copy()
        rc2[::2] += 50
        t[0].copy_(torch.from_numpy(rc2))
        torch.cuda.synchronize()
        check(policy, rc2, "new pod values")
        t[0].copy_(torch.from_numpy(rc))
        torch.cuda.synchronize()
        for step, q in enumerate((ks.KS_SCORE_LEAST_ALLOCATED, MOST_ALLOCATED, LEAST_BALANCED, MOST_ALLOCATED,
                                  LEAST_BALANCED)):
            got = check(q, rc, ("alternating", step, q))
            if step in (1, 2):  # a bind between the calls of 3 and 4, and of 4 and 3
                s.apply_bind(int(got[got >= 0][step]), 4000 * step, 1 << 32)


def test_index_follows_snapshot_changes(ks, o, policy):
    """The policy's bound order is rebuilt after each change of free[]: binds between calls are seen."""
    fc, fm, ac, am, lab, rc, rm, sel = cluster(14, 4000, 500)
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        for step in range(3):
            r = s.select(rc, rm, sel, policy=policy, flags=ks.KS_SELECT_FORCE_BITPAR)
            f = s.free()
            w = o.run_packed(f[0], f[1], ac, am, lab, rc, rm, sel, policy, want_mask=False)
            assert np.array_equal(r.node_idx, w[0]) and np.array_equal(r.score, w[1]), step
            p = int(np.nonzero(r.node_idx >= 0)[0][0])
            s.apply_bind(int(r.node_idx[p]), int(rc[p]) * 4 + 1000, int(rm[p]) * 4 + (1 << 30))


def assert_refused(ks, bad):
    """Every call that takes a policy refuses `bad' before any device work."""
    fc, fm, ac, am, lab, rc, rm, sel = cluster(11, 300, 20)
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        for call in (lambda: s.select(rc, rm, sel, policy=bad), lambda: s.select_topk(rc, rm, sel, 4, bad),
                     lambda: s.stream_bind(rc, rm, sel, bad), lambda: s.place_replicas(rc, rm, sel, np.ones(20), bad),
                     lambda: s.gang_bind(rc, rm, sel, np.arange(21, dtype=np.uint64), np.ones(20, np.uint32), bad)):
            with pytest.raises(ks.KsError) as e:
                call()
            assert e.value.code == -1


def test_full_c2(ks, o, policy):
    """The c2 workload of bench.py (100k pods x 10k nodes, same seed): both kernel paths and AUTO return the same
    bindings, counts and mask for every pod; 4096 seeded pods are checked against the restatement."""
    P, N = ks.synth.SHAPES["c2"]
    cl = ks.synth.make(P, N, ks.synth.SEEDS["c2"])
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    with ks.Snapshot(0) as s:
        s.set_nodes(ac, am, lab)
        s.set_bound(bn, bc, bm)
        fc, fm = s.free()
        d = s.select(rc, rm, sel, policy=policy, flags=ks.KS_SELECT_FORCE_DIRECT, want_mask=True)
        for flags in (ks.KS_SELECT_FORCE_BITPAR, ks.KS_SELECT_AUTO):
            r = s.select(rc, rm, sel, policy=policy, flags=flags, want_mask=True)
            assert np.array_equal(r.node_idx, d.node_idx) and np.array_equal(r.score, d.score), flags
            assert np.array_equal(r.feasible_cnt, d.feasible_cnt) and np.array_equal(r.mask, d.mask), flags
    pick = np.random.default_rng(0xC2).choice(P, 4096, replace=False)
    w = o.run_packed(fc, fm, ac, am, lab, rc[pick], rm[pick], sel[pick], policy)
    assert np.array_equal(d.node_idx[pick], w[0]) and np.array_equal(d.score[pick], w[1])
    assert np.array_equal(d.feasible_cnt[pick], w[2]) and np.array_equal(d.mask[pick], w[3])
    assert (d.node_idx >= 0).mean() > 0.5


@pytest.mark.parametrize("k", [1, 2, 7, 31, 32])
def test_select_topk(ks, o, policy, k):
    for seed, N, P, W, fam in ((20, 2500, 300, 1, "ties"), (21, 700, 9, 4, "edges"), (22, 9000, 2, 2, "mixed")):
        fc, fm, ac, am, lab, rc, rm, sel = cl = cluster(seed + k, N, P, W, fam)
        want = topk_packed(o, *cl, k, policy)
        with snapshot(ks, fc, fm, ac, am, lab) as s:
            got = s.select_topk(rc, rm, sel, k, policy)
            r = s.select(rc, rm, sel, policy=policy)
            assert all(np.array_equal(a, b) for a, b in zip(got, want)), (seed, k)
            assert np.array_equal(got[0][:, 0], r.node_idx) and np.array_equal(got[1][:, 0], r.score)
            assert np.array_equal(s.free()[0], fc)


@pytest.mark.parametrize("P", [1, 300, 1024, 1500])
def test_stream_bind_both_loops(ks, o, policy, P):
    """Up to 1024 pods the device loop, above it the host loop through the per-cell select."""
    fc, fm, ac, am, lab, rc, rm, sel = cl = cluster(30 + P, 900, P, 2)
    wf, wm = fc.copy(), fm.copy()
    want = o.stream_bind_packed(wf, wm, ac, am, lab, rc, rm, sel, policy)
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        got = s.stream_bind(rc, rm, sel, policy)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[2] == want[2]
        f = s.free()
        assert np.array_equal(f[0], wf) and np.array_equal(f[1], wm)
    assert (want[0] >= 0).any()


def test_stream_surface(ks, o, policy):
    fc, fm, ac, am, lab, rc, rm, sel = cluster(40, 600, 700)
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        with ks.Stream(s, policy, max_batch=256) as q:
            q.submit(rc, rm, sel, np.arange(len(rc), dtype=np.uint64))
            q.flush()
            t, i, sc = q.poll()
        assert sorted(t.tolist()) == list(range(len(rc)))
        wf, wm = fc.copy(), fm.copy()
        order = np.argsort(t, kind="stable")
        got_i, got_s = i[order], sc[order]
        f = s.free()
    placed = got_i >= 0
    # free[] is charged exactly the binds reported, and every score lies in the policy's range
    np.subtract.at(wf, got_i[placed], rc[placed])
    np.subtract.at(wm, got_i[placed], rm[placed])
    assert np.array_equal(f[0], wf) and np.array_equal(f[1], wm)
    assert placed.any() and (got_s[placed] >= 0).all() and (got_s[placed] <= SCORE_MAX[policy]).all()


def test_stream_surface_single_batch_equals_stream_bind(ks, o, policy):
    fc, fm, ac, am, lab, rc, rm, sel = cl = cluster(41, 600, 200)
    wf, wm = fc.copy(), fm.copy()
    want = o.stream_bind_packed(wf, wm, ac, am, lab, rc, rm, sel, policy)
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        with ks.Stream(s, policy, max_batch=1024) as q:
            q.submit(rc, rm, sel, np.arange(len(rc), dtype=np.uint64))
            q.flush()
            t, i, sc = q.poll()
            batches = q.stats()[0]
        order = np.argsort(t)
        assert batches == 1  # one submit of fewer than max_batch pods is one micro-batch: exactly ks_stream_bind
        assert np.array_equal(i[order], want[0]) and np.array_equal(sc[order], want[1])
        assert np.array_equal(s.free()[0], wf) and np.array_equal(s.free()[1], wm)


def test_gang_bind_with_rollback(ks, o, policy):
    fc, fm, ac, am, lab, rc, rm, sel = cl = cluster(50, 400, 900, 1)
    rc, rm = rc * 8, rm * 8
    off = groups(np.random.default_rng(50), len(rc), 1, 60)
    mm = np.diff(off).astype(np.uint32)  # all members: groups fail once the cluster fills
    wf, wm = fc.copy(), fm.copy()
    want = gang_bind_packed(o, wf, wm, ac, am, lab, rc, rm, sel, off, mm, policy)
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        got = s.gang_bind(rc, rm, sel, off, mm, policy)
        assert all(np.array_equal(a, b) for a, b in zip(got, want))
        f = s.free()
        assert np.array_equal(f[0], wf) and np.array_equal(f[1], wm)  # rolled-back groups restored bit for bit
    assert (want[2] < mm).any() and (want[2] >= mm).any()


@pytest.mark.parametrize("exclude", [0, 1])
def test_drain_check(ks, o, policy, exclude):
    fc, fm, ac, am, lab, _, _, _ = cluster(60 + exclude, 500, 1)
    rng = np.random.default_rng(60)
    B = 2500
    bn = rng.integers(0, 500, B).astype(np.int32)
    bc, bm = rng.choice([500, 2000, 8000], B).astype(np.int64), rng.choice([1 << 30, 1 << 33], B).astype(np.int64)
    order, node, off = bound_candidates(bn, 500)
    pc, pm = bc[order], bm[order]
    psel = np.zeros((len(order), 1), np.uint64)
    psel[::7, 0] = np.uint64(1) << np.uint64(63)  # a pair no node carries: that pod's candidate stops there
    want = drain_packed(o, fc, fm, ac, am, lab, pc, pm, psel, node, off, policy, exclude=bool(exclude))
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        got = s.drain_check(pc, pm, psel, node, off, policy, exclude)
        assert all(np.array_equal(a, b) for a, b in zip(got, want))
        assert np.array_equal(s.free()[0], fc) and np.array_equal(s.free()[1], fm)
    size = np.diff(off)
    assert (want[0] == size).any() and (want[0] < size).any()


def test_place_replicas(ks, o, policy):
    fc, fm, ac, am, lab, rc, rm, sel = cluster(70, 3000, 64, 2, "edges")
    rc[rc == 0] = 250
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        cap = s.place_replicas(rc, rm, sel, np.zeros(64), policy, want_nodes=False)[0]["capacity"].astype(np.int64)
        R = np.array([0, 1, 2, 65536] + [max(0, min(int(c) + d, 65536)) for c, d in zip(cap[4:], [-1, 0, 1] * 20)],
                     np.uint32)
        got = s.place_replicas(rc, rm, sel, R, policy)
        want = PLAN[policy](fc, fm, ac, am, lab, rc, rm, sel, R)
        for f in want[0].dtype.names:
            assert np.array_equal(got[0][f], want[0][f]), f
        assert all(np.array_equal(a, b) for a, b in zip(got[1:], want[1:]))
        assert np.array_equal(s.free()[0], fc) and np.array_equal(s.free()[1], fm)
        assert (got[0]["placed"] > 0).sum() > 30 and (got[0]["max_per_node"] > 1).any()
        rows = s.place_replicas(rc, rm, sel, R, policy, want_nodes=False)[0]  # the rows alone are the same
        assert all(np.array_equal(rows[f], got[0][f]) for f in rows.dtype.names)
        # a shorter request is a prefix of the longer plan
        short = s.place_replicas(rc, rm, sel, R // 2, policy)
        for t in range(len(R)):
            a, b, c = int(got[3][t]), int(short[3][t]), int(short[3][t + 1])
            n = int(short[0]["placed"][t])
            assert np.array_equal(short[1][b:b + n], got[1][a:a + n]) and np.array_equal(short[2][b:b + n], got[2][a:a + n])
            assert (short[1][b + n:c] == -1).all()


def test_place_replicas_equals_singleton_gangs_and_commits(ks, o, policy):
    fc, fm, ac, am, lab, rc, rm, sel = cluster(71, 800, 6, 1)
    rc[rc == 0], rm[rm == 0] = 500, 1 << 30
    R = np.array([1, 5, 40, 200, 1000, 3], np.uint32)
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        rows, node, score, off = s.place_replicas(rc, rm, sel, R, policy)
        for t in range(len(R)):
            a, b = int(off[t]), int(off[t + 1])
            n = int(R[t])
            gi, gs, _, _ = s.gang_bind(np.repeat(rc[t], n), np.repeat(rm[t], n), np.repeat(sel[t:t + 1], n, 0),
                                       np.arange(n + 1, dtype=np.uint64), np.zeros(n, np.uint32), policy)
            assert np.array_equal(gi, node[a:b]) and np.array_equal(gs, score[a:b]), t
            gf = s.free()
            s.set_bound(np.arange(len(ac), dtype=np.int32), ac - fc, am - fm)  # back to the start
            placed = node[a:b][node[a:b] >= 0]
            acc = s.commit_claims(placed, np.repeat(rc[t], len(placed)), np.repeat(rm[t], len(placed)))
            assert acc.all()
            cf = s.free()
            assert np.array_equal(cf[0], gf[0]) and np.array_equal(cf[1], gf[1])
            s.set_bound(np.arange(len(ac), dtype=np.int32), ac - fc, am - fm)
        # the restatements agree with one copy at a time on this cluster too
        want = PLAN[policy](fc, fm, ac, am, lab, rc, rm, sel, R)
        assert all(np.array_equal(a, b) for a, b in zip((node, score), want[1:3]))


def test_host_layer(ks, o, policy):
    """ksh_select_nodes, ksh_rank_nodes, ksh_place_replicas, ksh_drain_nodes, ksh_reconcile_gangs and
    ksh_reconcile_batch under the policy equal the packed calls on the context's own packed state."""
    cl = ks.synth.make(300, 400, seed=0x3A11, bound_per_node=2)
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(nodes_s), arena.pods(bound_s), arena.pods(pods_s)
    P, gp = len(pods_s), 120
    R = (np.arange(P) % 9).astype(np.uint32)
    offg = groups(np.random.default_rng(3), gp, 1, 12)
    mm = (np.diff(offg) // 2).astype(np.uint32)
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, cl.N)
        ctx.set_cluster_pods(bound, len(bound_s))
        h_sel = ctx.select_nodes(pods, P, policy=policy)
        h_rank = ctx.rank_nodes(pods, P, 6, policy=policy)
        h_rep = ctx.place_replicas(pods, P, R, policy=policy)
        ac, am, lab, bn, bc, bm = ctx.export_packed()
        order, node, off = bound_candidates(bn, cl.N)
        dp = arena.pods([bound_s[i] for i in order])
        h_drain = ctx.drain_nodes([ctx.node_name(n) for n in range(cl.N)], dp, off, policy=policy)
        rc, rm, sel = ctx.pack_pods(pods, P)
        dc, dm, dsel = ctx.pack_pods(dp, len(order))
        assert all(np.array_equal(a, b) for a, b in zip(ctx.export_packed(), (ac, am, lab, bn, bc, bm)))  # nothing bound
        h_gang = ctx.reconcile_gangs(pods, gp, offg, mm, policy=policy)
        h_batch = ctx.reconcile_batch(arena.pods(pods_s[gp:]), P - gp, policy=policy)
    with ks.Snapshot(0) as s:
        s.set_nodes(ac, am, lab)
        s.set_bound(bn, bc, bm)
        r = s.select(rc, rm, sel, policy=policy)
        assert np.array_equal(h_sel[0], r.node_idx) and np.array_equal(h_sel[1], r.score)
        assert np.array_equal(h_sel[2], r.feasible_cnt)
        fc, fm = s.free()
        w = o.run_packed(fc, fm, ac, am, lab, rc, rm, sel, policy, want_mask=False)
        assert np.array_equal(r.node_idx, w[0]) and (w[0] >= 0).any() and (w[0] < 0).any()
        assert all(np.array_equal(a, b) for a, b in zip(h_rank, s.select_topk(rc, rm, sel, 6, policy)))
        want = s.place_replicas(rc, rm, sel, R, policy)
        assert all(np.array_equal(a, b) for a, b in zip(h_rep, want))
        want = s.drain_check(dc, dm, dsel, node, off, policy)
        assert np.array_equal(h_drain[0], want[0]) and np.array_equal(h_drain[1], want[1])
        want = s.gang_bind(rc[:gp], rm[:gp], sel[:gp], offg, mm, policy)
        assert np.array_equal(h_gang[1], want[0]) and np.array_equal(h_gang[3], want[2])
        want = s.stream_bind(rc[gp:], rm[gp:], sel[gp:], policy)
        assert np.array_equal(h_batch[1], want[0])


def test_sequential_singletons_equal_restatement(ks, o, policy):
    """Singleton groups: every pod sees the binds of all earlier pods."""
    fc, fm, ac, am, lab, rc, rm, sel = cluster(80, 200, 300, 1)
    wf, wm = fc.copy(), fm.copy()
    want = one_at_a_time(o, wf, wm, ac, am, lab, rc, rm, sel, policy)
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        got = s.gang_bind(rc, rm, sel, np.arange(len(rc) + 1, dtype=np.uint64), np.ones(len(rc), np.uint32), policy)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert np.array_equal(s.free()[0], wf)


def test_place_replicas_large_plans_and_many_specs(ks, o, policy):
    """65 536 copies of one spec, and 300 specs on a node count past one shared block of the sequential kernel's
    1024-node block maxima (policy 4), against the restatement of the policy's plan."""
    fc, fm, ac, am, lab, rc, rm, sel = cluster(72, 2600, 300, 1)
    rc[rc == 0] = 100
    R = (np.arange(300) * 37 % 900).astype(np.uint32)
    R[0] = 65536
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        got = s.place_replicas(rc, rm, sel, R, policy)
    want = PLAN[policy](fc, fm, ac, am, lab, rc, rm, sel, R)
    for f in want[0].dtype.names:
        assert np.array_equal(got[0][f], want[0][f]), f
    assert all(np.array_equal(a, b) for a, b in zip(got[1:], want[1:]))
    assert got[0]["placed"][0] > 1000


def test_full_c3_argmax_paths_agree(ks, policy):
    """The c3 workload of bench.py: the bit-parallel walk and the per-cell kernel return the same bindings."""
    P, N = ks.synth.SHAPES["c3"]
    cl = ks.synth.make(P, N, ks.synth.SEEDS["c3"])
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    with ks.Snapshot(0) as s:
        s.set_nodes(ac, am, lab)
        s.set_bound(bn, bc, bm)
        d = s.select(rc, rm, sel, policy=policy, flags=ks.KS_SELECT_FORCE_DIRECT)
        b = s.select(rc, rm, sel, policy=policy, flags=ks.KS_SELECT_FORCE_BITPAR)
        assert b.path == "bitpar" and d.path == "direct"
        assert np.array_equal(b.node_idx, d.node_idx) and np.array_equal(b.score, d.score)
        assert np.array_equal(b.feasible_cnt, d.feasible_cnt)


__all__ += [n for n in dir() if n.startswith("test_")]
