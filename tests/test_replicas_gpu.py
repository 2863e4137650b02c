"""Replica placement (ks_place_replicas) on the GPU: rows, copy nodes and copy scores bit for bit against the merge
restatement of tests/replicas_oracle.py across label widths, node counts around the chunk edges, spec counts up to the
limit, replica counts around the capacity and up to the limits, both policies, tie-heavy clusters, LEAST_ALLOCATED
plateaus, zero requests and values at the limits; the plan against the device's own one-copy-at-a-time paths
(ks_gang_bind with singleton groups, ks_snapshot_commit_claims, ks_select on both kernel paths); nothing charged; the
shared staging between other calls; and the host layer."""
import ctypes as C

import numpy as np
import pytest

from helpers import load_golden
from replicas_oracle import U64_MAX, merge_packed, node_copies

pytestmark = pytest.mark.gpu

LIM_C, LIM_M = 1 << 36, 1 << 55
KS_ERR_PARSE = -3  # include/ksched.h
FIELDS = ("capacity", "placed", "nodes", "feasible_cnt", "max_per_node", "last_score")


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def chunk_geometry(N, T, sms):
    """replica_chunks of ks_replicas.cu: (n_chunks, chunk_len)."""
    tiles = max(1, (N + 255) // 256)
    want = min(tiles, max(1, (4 * sms + T - 1) // T))
    per = (tiles + want - 1) // want
    return (tiles + per - 1) // per, per * 256


def _nodes(rng, N, W, dense=0.7):
    ac = rng.choice([2000, 4000, 8000, 16000, 64000], N).astype(np.int64)
    am = rng.choice([8, 16, 32, 64, 256], N).astype(np.int64) << 30
    fc = ac - rng.integers(0, 2000, N)
    fm = am - rng.integers(0, 8 << 30, N)
    lab = np.zeros((N, W), np.uint64)
    on = rng.random((N, 64 * W)) < dense
    for w in range(W):
        lab[:, w] = (on[:, 64 * w:64 * w + 64].astype(np.uint64) << np.arange(64, dtype=np.uint64)).sum(1, dtype=np.uint64)
    return fc, fm, ac, am, lab


def _specs(rng, T, W, cpu=(0, 4000), mem=(0, 16 << 30), sel_p=0.3):
    rc = rng.integers(cpu[0], cpu[1] + 1, T).astype(np.int64)
    rm = rng.integers(mem[0], mem[1] + 1, T).astype(np.int64)
    sel = np.zeros((T, W), np.uint64)
    for t in np.nonzero(rng.random(T) < sel_p)[0]:
        b = int(rng.integers(0, 64 * W))
        sel[t, b // 64] |= np.uint64(1) << np.uint64(b % 64)
    return rc, rm, sel


def load(ks, snap, fc, fm, ac, am, lab):
    """Nodes with allocatable ac/am and free fc/fm (one bound pod per node carries the difference)."""
    snap.set_nodes(ac, am, lab)
    n = len(ac)
    snap.set_bound(np.arange(n, dtype=np.int32), ac - fc, am - fm)
    got = snap.free()
    assert np.array_equal(got[0], fc) and np.array_equal(got[1], fm)


def check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, R, policy, want_nodes=True):
    got = snap.place_replicas(rc, rm, sel, R, policy, want_nodes=want_nodes)
    want = merge_packed(fc, fm, ac, am, lab, rc, rm, sel, R, policy)
    for f in FIELDS:
        assert np.array_equal(got[0][f], want[0][f]), (f, got[0][f][:8], want[0][f][:8])
    if want_nodes:
        assert np.array_equal(got[1], want[1]), np.nonzero(got[1] != want[1])[0][:8]
        assert np.array_equal(got[2], want[2]), np.nonzero(got[2] != want[2])[0][:8]
    assert np.array_equal(got[3], want[3])
    return got


@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("policy", [0, 1])
def test_label_widths(ks, W, policy):
    rng = np.random.default_rng(10 * W + policy)
    fc, fm, ac, am, lab = _nodes(rng, 3000, W)
    rc, rm, sel = _specs(rng, 40, W)
    R = rng.integers(0, 3000, 40).astype(np.uint32)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        rows = check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, R, policy)[0]
        check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, R, policy, want_nodes=False)
    assert (rows["placed"] > 0).any() and (rows["nodes"] > 1).any()


def test_node_counts_around_the_chunk_edges(ks):
    sms = _sms()
    rng = np.random.default_rng(3)
    for T in (1, 7):
        sizes = {1, 255, 256, 257}
        for N in (5000, 70000):
            n_chunks, clen = chunk_geometry(N, T, sms)
            sizes |= {clen - 1, clen, clen + 1, (n_chunks - 1) * clen, (n_chunks - 1) * clen + 1}
        for N in sorted(s for s in sizes if s > 0):
            fc, fm, ac, am, lab = _nodes(rng, N, 1)
            rc, rm, sel = _specs(rng, T, 1, cpu=(500, 4000), mem=(1 << 30, 16 << 30))
            R = rng.integers(0, 5000, T).astype(np.uint32)
            with ks.Snapshot(0) as snap:
                load(ks, snap, fc, fm, ac, am, lab)
                for policy in (0, 1):
                    check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, R, policy)


def test_largest_cluster(ks):
    rng = np.random.default_rng(4)
    N = 270337
    fc, fm, ac, am, lab = _nodes(rng, N, 2)
    rc, rm, sel = _specs(rng, 3, 2, cpu=(1000, 4000), mem=(4 << 30, 16 << 30))
    R = np.array([1, 20000, 65536], np.uint32)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        for policy in (0, 1):
            check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, R, policy)


def test_spec_counts_up_to_the_limit(ks):
    rng = np.random.default_rng(5)
    fc, fm, ac, am, lab = _nodes(rng, 300, 1)
    for T in (1, 2, 1000, 4096):
        rc, rm, sel = _specs(rng, T, 1)
        R = rng.integers(0, 40, T).astype(np.uint32)
        with ks.Snapshot(0) as snap:
            load(ks, snap, fc, fm, ac, am, lab)
            check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, R, T % 2)


def test_replicas_around_the_capacity(ks):
    rng = np.random.default_rng(6)
    fc, fm, ac, am, lab = _nodes(rng, 900, 1)
    rc, rm, sel = _specs(rng, 6, 1, cpu=(200, 3000), mem=(1 << 30, 8 << 30))
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        caps = [node_copies(fc, fm, lab, int(rc[t]), int(rm[t]), sel[t])[1] for t in range(6)]
        for policy in (0, 1):
            for delta in (-1, 0, 1):
                R = np.array([min(65536, max(0, c + delta)) for c in caps], np.uint32)
                rows = check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, R, policy)[0]
                assert np.array_equal(rows["placed"], np.minimum(R, rows["capacity"]))
            check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, np.array([0, 1, 65536, 0, 1, 65536], np.uint32), policy)


def test_total_replicas_at_the_limit(ks):
    """256 specs of 65536 copies: 2^24 copies in one call, each spec's plan against one restatement."""
    rng = np.random.default_rng(7)
    N = 40
    fc, fm, ac, am, lab = _nodes(rng, N, 1, dense=0.0)
    fc, fm = fc * 8, fm * 8  # room for a few thousand copies per node
    T = 256
    rc, rm = np.full(T, 7, np.int64), np.full(T, 1 << 24, np.int64)
    rc[1::2], rm[1::2] = 5, 3 << 23
    sel = np.zeros((T, 1), np.uint64)
    R = np.full(T, 65536, np.uint32)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac * 8, am * 8, lab)
        snap.set_bound(np.arange(N, dtype=np.int32), ac * 8 - fc, am * 8 - fm)
        for policy in (0, 1):
            rows, node, score, off = snap.place_replicas(rc, rm, sel, R, policy)
            assert int(off[-1]) == 1 << 24
            for t in (0, 1):
                w = merge_packed(fc, fm, ac * 8, am * 8, lab, rc[t:t + 1], rm[t:t + 1], sel[t:t + 1], R[t:t + 1], policy)
                for u in range(t, T, 2):
                    a, b = int(off[u]), int(off[u + 1])
                    assert all(rows[f][u] == w[0][f][0] for f in FIELDS)
                    assert np.array_equal(node[a:b], w[1]) and np.array_equal(score[a:b], w[2])


def test_tie_heavy_clusters_across_chunk_edges(ks):
    sms = _sms()
    for T in (1, 3):
        n_chunks, clen = chunk_geometry(4 * 4096, T, sms)
        N = max(n_chunks, 2) * clen
        N = min(N, 4 * 4096)
        fc = np.full(N, 4000, np.int64)
        fm = np.full(N, 16 << 30, np.int64)
        lab = np.zeros((N, 1), np.uint64)
        rc, rm, sel = np.full(T, 1000, np.int64), np.full(T, 4 << 30, np.int64), np.zeros((T, 1), np.uint64)
        with ks.Snapshot(0) as snap:
            load(ks, snap, fc, fm, fc, fm, lab)
            for policy in (0, 1):
                # every node takes 4 copies with equal scores per copy: the tie boundary falls at node clen + 5 etc.
                for R in (clen + 5, 2 * clen - 1, N + clen + 3, 4 * N - 1):
                    Rs = np.full(T, min(R, 65536), np.uint32)
                    check(ks, snap, fc, fm, fc, fm, lab, rc, rm, sel, Rs, policy)


def test_least_allocated_plateaus(ks):
    rng = np.random.default_rng(8)
    N = 2000
    ac = np.full(N, 1 << 20, np.int64)  # a request of 1000 m moves the percentage by 0 or 1: long plateaus
    am = np.full(N, 1 << 50, np.int64)
    fc = ac - rng.integers(0, 1 << 19, N)
    fm = am - rng.integers(0, 1 << 49, N)
    lab = np.zeros((N, 1), np.uint64)
    rc, rm, sel = np.array([1000, 3000, 0], np.int64), np.array([1 << 30, 0, 1 << 40], np.int64), np.zeros((3, 1), np.uint64)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, np.array([65536, 40000, 777], np.uint32), 1)


def test_zero_requests(ks):
    rng = np.random.default_rng(9)
    fc, fm, ac, am, lab = _nodes(rng, 5000, 1, dense=0.0)
    rc, rm, sel = np.zeros(2, np.int64), np.zeros(2, np.int64), np.zeros((2, 1), np.uint64)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        for policy in (0, 1):
            rows, node, score, _ = check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, np.array([65536, 3], np.uint32),
                                         policy)
            assert (rows["capacity"] == U64_MAX).all() and (rows["nodes"] == 1).all()
            assert rows["max_per_node"].tolist() == [65536, 3] and len(set(node.tolist())) == 1


def test_limits_negative_free_nonpositive_allocatable_and_selectors(ks):
    rng = np.random.default_rng(10)
    N, W = 4000, 2
    fc = rng.choice([-LIM_C // 2, -1, 0, 1, 1000, LIM_C // 2, LIM_C // 3], N).astype(np.int64)
    fm = rng.choice([-LIM_M // 2, -1, 0, 1, 1 << 30, LIM_M // 2, LIM_M // 3], N).astype(np.int64)
    ac = np.where(rng.random(N) < 0.2, rng.choice([-5, 0], N), fc + rng.integers(0, 1000, N)).astype(np.int64)
    am = np.where(rng.random(N) < 0.2, rng.choice([-5, 0], N), fm + rng.integers(0, 1 << 20, N)).astype(np.int64)
    lab = np.zeros((N, W), np.uint64)
    lab[:, 0] = rng.integers(0, 1 << 62, N, dtype=np.int64).astype(np.uint64)  # dense selectors
    lab[:, 1] = np.where(rng.random(N) < 0.5, ~np.uint64(0) >> np.uint64(1), 0).astype(np.uint64)
    T = 24
    rc = rng.choice([0, 1, 1000, LIM_C // 4, LIM_C], T).astype(np.int64)
    rm = rng.choice([0, 1, 1 << 30, LIM_M // 4, LIM_M], T).astype(np.int64)
    sel = np.zeros((T, W), np.uint64)
    sel[:, 0] = rng.integers(0, 4, T).astype(np.uint64)
    sel[::5, 1] = np.uint64(1) << np.uint64(63)  # the never-set bit: capacity 0
    R = rng.integers(0, 65537, T).astype(np.uint32)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(np.arange(N, dtype=np.int32), ac - fc, am - fm)
        for policy in (0, 1):
            rows = check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, R, policy)[0]
            assert (rows["capacity"][::5] == 0).all()


def _cluster(ks, seed, N=600):
    cl = ks.synth.make(N, 10, seed=seed, bound_per_node=2)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    return ac, am, lab, bn, bc, bm, rc, rm, sel


@pytest.mark.parametrize("policy", [0, 1])
def test_one_copy_at_a_time_on_the_device(ks, orc, policy):
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, 0xAB + policy)
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    for t in range(4):
        spec = rc[t:t + 1] * 3, rm[t:t + 1] * 3, np.ascontiguousarray(sel[t:t + 1])
        R = 700
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            snap.set_bound(bn, bc, bm)
            rows, node, score, _ = snap.place_replicas(*spec, [R], policy)
            first = snap.select(*spec, policy=policy)
            assert node[0] == first.node_idx[0] and rows["feasible_cnt"][0] == first.feasible_cnt[0]
            if node[0] >= 0:
                assert score[0] == first.score[0]
            for r in (0, 1, 5, int(rows["placed"][0])):  # a shorter request plans the prefix
                p = snap.place_replicas(*spec, [r], policy)
                assert np.array_equal(p[1], node[:r]) and np.array_equal(p[2], score[:r])
            gang_node, gang_score, _, _ = snap.gang_bind(np.repeat(spec[0], R), np.repeat(spec[1], R),
                                                         np.repeat(spec[2], R, axis=0), np.arange(R + 1, dtype=np.uint64),
                                                         np.zeros(R, np.uint32), policy)
            gang_free = snap.free()
        assert np.array_equal(gang_node, node) and np.array_equal(gang_score, score)
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            snap.set_bound(bn, bc, bm)
            acc = snap.commit_claims(node, np.repeat(spec[0], R), np.repeat(spec[1], R))
            assert acc.all() if rows["placed"][0] == R else acc[:rows["placed"][0]].all()
            f = snap.free()
            assert np.array_equal(f[0], gang_free[0]) and np.array_equal(f[1], gang_free[1])
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            snap.set_bound(bn, bc, bm)
            done = 0
            for r in sorted({1, 2, 17, 300, int(rows["placed"][0])}):
                if r > rows["placed"][0]:
                    continue
                snap.commit_claims(node[done:r], np.repeat(spec[0], r - done), np.repeat(spec[1], r - done))
                done = r
                for flags in (ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR):
                    if flags == ks.KS_SELECT_FORCE_BITPAR and policy:
                        continue  # the bit-parallel kernel is LEFTOVER only
                    s = snap.select(*spec, policy=policy, flags=flags)
                    want = (node[r], score[r]) if r < R else (-1, 0)
                    assert (s.node_idx[0], s.score[0] if s.node_idx[0] >= 0 else 0) == want, (r, flags)


def test_nothing_is_charged_and_errors_change_nothing(ks, orc):
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, 0xC0)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        before, pick = snap.free(), snap.select(rc, rm, sel)
        snap.place_replicas(rc, rm, sel, np.full(len(rc), 100, np.uint32), 0)
        snap.place_replicas(rc, rm, sel, np.full(len(rc), 100, np.uint32), 1, want_nodes=False)
        for kw, code in ((dict(policy=7), ks.capi.KS_ERR_INVALID),
                         (dict(rc=np.array([-1] + [0] * (len(rc) - 1))), ks.capi.KS_ERR_RANGE),
                         (dict(rm=np.array([LIM_M + 1] + [0] * (len(rc) - 1))), ks.capi.KS_ERR_RANGE),
                         (dict(R=np.array([65537] + [1] * (len(rc) - 1))), ks.capi.KS_ERR_RANGE)):
            with pytest.raises(ks.KsError) as e:
                snap.place_replicas(kw.get("rc", rc), kw.get("rm", rm), sel, kw.get("R", np.ones(len(rc))),
                                    kw.get("policy", 0))
            assert e.value.code == code
        big = np.full(4097, 1, np.uint32)
        with pytest.raises(ks.KsError) as e:
            snap.place_replicas(np.zeros(4097), np.zeros(4097), np.zeros((4097, snap.label_words)), big)
        assert e.value.code == ks.capi.KS_ERR_RANGE
        with pytest.raises(ks.KsError) as e:
            snap.place_replicas(np.zeros(257), np.zeros(257), np.zeros((257, snap.label_words)),
                                np.full(257, 65536, np.uint32))
        assert e.value.code == ks.capi.KS_ERR_RANGE  # more than 2^24 copies
        out = (ks.capi.ks_replica_plan * 1)()
        pods = ks.capi.ks_pods(1, rc.ctypes.data, rm.ctypes.data, sel.ctypes.data, ks.KS_MEM_DEVICE)
        one = np.ones(1, np.uint32)
        assert ks.lib.ks_place_replicas(snap._h, C.byref(pods), one.ctypes.data, 0, out, None, None) == ks.capi.KS_ERR_INVALID
        pods.mem_space = ks.KS_MEM_HOST
        assert ks.lib.ks_place_replicas(snap._h, C.byref(pods), None, 0, out, None, None) == ks.capi.KS_ERR_INVALID
        assert ks.lib.ks_place_replicas(snap._h, C.byref(pods), one.ctypes.data, 0, None, None, None) == ks.capi.KS_ERR_INVALID
        pods.n = 0
        assert ks.lib.ks_place_replicas(snap._h, C.byref(pods), None, 0, None, None, None) == ks.KS_OK
        after = snap.free()
        assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
        again = snap.select(rc, rm, sel)
        assert np.array_equal(pick.node_idx, again.node_idx) and np.array_equal(pick.score, again.score)


def test_empty_snapshot(ks):
    with ks.Snapshot(0) as snap:
        snap.set_nodes(np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 1), np.uint64))
        rows, node, score, _ = snap.place_replicas([1, 0], [1, 0], np.zeros((2, 1)), [3, 2])
        assert (rows["capacity"] == 0).all() and (rows["placed"] == 0).all() and (node == -1).all() and (score == 0).all()


def test_staging_shared_with_other_calls(ks, orc):
    """A large call grows the shared device blocks between scale-up, drain, gang and cached-graph selects; every result
    equals the same call on a fresh snapshot."""
    import torch
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, 0xD0, N=2000)
    W = lab.shape[1]
    T = 64
    rs = np.resize(rc, T), np.resize(rm, T), np.resize(sel, (T, W))
    big = np.full(T, 60000, np.uint32)

    def fresh(fn):
        with ks.Snapshot(0) as s:
            s.set_nodes(ac, am, lab)
            s.set_bound(bn, bc, bm)
            return fn(s)

    rep = lambda s: s.place_replicas(*rs, big, 1)
    small = lambda s: s.place_replicas(rc, rm, sel, np.full(len(rc), 3, np.uint32), 0)
    tac, tam = ac[:8], am[:8]
    scale = lambda s: s.scaleup_estimate(rc, rm, sel, tac, tam, tac, tam, lab[:8], np.full(8, 20, np.uint32))
    off = np.arange(0, 11, dtype=np.uint64)
    drain = lambda s: s.drain_check(rc[:10], rm[:10], sel[:10], np.arange(10, dtype=np.int32), off)
    want = {k: fresh(f) for k, f in (("rep", rep), ("small", small), ("scale", scale), ("drain", drain))}
    d = torch.device("cuda:0")
    t_rc, t_rm = torch.from_numpy(rc).to(d), torch.from_numpy(rm).to(d)
    t_sel = torch.from_numpy(sel.view(np.int64)).to(d)
    P = len(rc)
    with ks.Snapshot(0) as s:
        s.set_nodes(ac, am, lab)
        s.set_bound(bn, bc, bm)
        idx0 = torch.empty(P, dtype=torch.int32, device=d)
        sc0 = torch.empty(P, dtype=torch.int64, device=d)
        cnt0 = torch.empty(P, dtype=torch.int32, device=d)
        for step in range(2):
            for name, fn in (("small", small), ("scale", scale), ("rep", rep), ("drain", drain), ("small", small)):
                got = fn(s)
                assert all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(got, want[name])), (step, name)
                s.select_raw(P, t_rc, t_rm, t_sel, ks.KS_MEM_DEVICE, idx0, sc0, cnt0, ks.KS_MEM_DEVICE)
                torch.cuda.synchronize()
                host = s.select(rc, rm, sel)
                assert np.array_equal(idx0.cpu().numpy(), host.node_idx), (step, name)
        g = s.gang_bind(rc[:1000], rm[:1000], sel[:1000], np.array([0, 1000], np.uint64), np.zeros(1, np.uint32))
        assert len(g[0]) == 1000
        after_gang = s.place_replicas(*rs, big, 1)  # after a charging call: equals a fresh snapshot with that free[]
        with ks.Snapshot(0) as f:
            f.set_nodes(ac, am, lab)
            f.set_bound(np.concatenate([bn, g[0][g[0] >= 0]]), np.concatenate([bc, rc[:1000][g[0] >= 0]]),
                        np.concatenate([bm, rm[:1000][g[0] >= 0]]))
            want_gang = f.place_replicas(*rs, big, 1)
        assert all(np.array_equal(a, b) for a, b in zip(after_gang, want_gang))


def test_host_layer_after_node_and_pod_events(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    nodes = arena.nodes(g["nodes"])
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        pods = arena.pods(g["pods"])
        n = len(g["pods"])
        R = np.arange(n, dtype=np.uint32) % 7 + 1
        for step in range(3):
            before = ctx.export_packed()
            got = ctx.place_replicas(pods, n, R, step % 2)
            ac, am, lab, bn, bc, bm = ctx.export_packed()
            rc, rm, sel = ctx.pack_pods(pods, n)
            with ks.Snapshot(0) as s:
                s.set_nodes(ac, am, lab)
                s.set_bound(bn, bc, bm)
                want = s.place_replicas(rc, rm, sel, R, step % 2)
            for a, b in zip(got, want):
                assert np.array_equal(a, b), step
            assert all(np.array_equal(a, b) for a, b in zip(ctx.export_packed(), before))  # nothing bound or changed
            if step == 0:  # a node event: the first node goes, then a pod event binds a copy of pod 0
                ctx.remove_node(ctx.node_name(0))
            elif step == 1 and got[1][0] >= 0:
                bound = dict(g["pods"][0])
                bound["name"] = "replica-0"
                bound["node_name"] = ctx.node_name(int(got[1][0]))
                ctx.pod_bound(arena.pods([bound]))


def test_host_layer_errors_and_absent_pairs(ks):
    """Packing errors of the object-level call on a device context, before any device work and with nothing changed:
    an unparsable quantity (KS_ERR_PARSE), NULL pods, replicas or out with n > 0 (KS_ERR_INVALID), a replica count above
    the limit (KS_ERR_RANGE).  A selector pair no node carries maps to the never-set bit: capacity 0."""
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        ctx.set_cluster_pods(arena.pods(g["bound_pods"]), len(g["bound_pods"]))
        before = ctx.export_packed()
        good = [{"name": "a", "containers": [{"cpu": "500m", "memory": "1073741824"}]}]
        bad = good + [{"name": "bad", "containers": [{"cpu": "1", "memory": "12Qi"}]}]
        with pytest.raises(ks.KsError) as e:
            ctx.place_replicas(arena.pods(bad), 2, [1, 1])
        assert e.value.code == KS_ERR_PARSE
        with pytest.raises(ks.KsError) as e:
            ctx.place_replicas(arena.pods(good), 1, [65537])
        assert e.value.code == ks.capi.KS_ERR_RANGE
        rows = np.zeros(1, ks.capi.REPLICA_PLAN_DTYPE)
        one = np.ones(1, np.uint32)
        pods = arena.pods(good)
        lib = ks.lib
        assert lib.ksh_place_replicas(ctx._h, None, 1, one.ctypes.data, 0, rows.ctypes.data, None, None) == ks.capi.KS_ERR_INVALID
        assert lib.ksh_place_replicas(ctx._h, C.addressof(pods), 1, None, 0, rows.ctypes.data, None, None) == ks.capi.KS_ERR_INVALID
        assert lib.ksh_place_replicas(ctx._h, C.addressof(pods), 1, one.ctypes.data, 0, None, None, None) == ks.capi.KS_ERR_INVALID
        assert lib.ksh_place_replicas(ctx._h, None, 0, None, 0, None, None, None) == ks.KS_OK
        assert all(np.array_equal(a, b) for a, b in zip(ctx.export_packed(), before))
        absent = [dict(good[0], selector={"zone": "nowhere"}), dict(good[0], name="b", selector={"zone": "a"})]
        rows, node, score, off = ctx.place_replicas(arena.pods(absent), 2, [3, 3])
        assert rows["capacity"][0] == 0 and (node[:3] == -1).all() and rows["capacity"][1] > 0 and rows["placed"][1] == 3


@pytest.mark.parametrize("policy", [0, 1])
def test_smallest_allocatable_and_largest_free(ks, policy):
    """Allocatable of 1 to 3 millicores / bytes with free near 2^36 / 2^55: LEAST_ALLOCATED scores near 100 * 2^55 / 2,
    the widest threshold range the search has to close; next to ordinary nodes so the threshold falls between them."""
    rng = np.random.default_rng(11 + policy)
    N = 300
    fc, fm, ac, am, lab = _nodes(rng, N, 1, dense=0.0)
    k = np.arange(0, N, 3)
    ac[k] = rng.integers(1, 4, len(k))
    am[k] = rng.integers(1, 4, len(k))
    fc[k] = LIM_C - rng.integers(0, 1 << 20, len(k))
    fm[k] = LIM_M - rng.integers(0, 1 << 40, len(k))
    T = 8
    rc = np.array([100, 0, 1000, 1 << 20, 1 << 30, 7, 0, 4000], np.int64)
    rm = np.array([1 << 20, 1 << 30, 0, 1 << 40, 1 << 50, 1 << 45, 0, 16 << 30], np.int64)
    sel = np.zeros((T, 1), np.uint64)
    R = np.array([15, 65536, 65536, 40000, 3000, 65536, 5, 900], np.uint32)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        check(ks, snap, fc, fm, ac, am, lab, rc, rm, sel, R, policy)
    # three nodes: one with a 1-byte memory allocatable and 2^55 bytes free, two ordinary ones
    fc, fm = np.array([1000, 1000, 1000], np.int64), np.array([LIM_M, 1 << 30, 1 << 30], np.int64)
    ac, am = np.array([1000, 1000, 1000], np.int64), np.array([1, 1 << 30, 1 << 30], np.int64)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, np.zeros((3, 1), np.uint64))
        for r in (1, 14, 15, 16, 30):
            check(ks, snap, fc, fm, ac, am, np.zeros((3, 1), np.uint64), np.array([100], np.int64),
                  np.array([1 << 20], np.int64), np.zeros((1, 1), np.uint64), np.array([r], np.uint32), policy)
