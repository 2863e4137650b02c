"""The calls that change free[] on the device (-m gpu): ks_snapshot_apply_bind, ks_snapshot_commit_claims (K3
k_stream_resolve), ks_stream_bind (the cooperative k_stream_batch and the host-driven loop above 1024 pods), ks_gang_bind
(k_gang_batch) and the ks_stream queue, bit for bit against the oracle's restatements (orc.stream_bind_packed,
orc.commit_claims, tests/gang_oracle.py) at edge values and at the kernels' internal boundaries: the per-CTA node
slices of k_stream_batch, its 4-pod loser strips, the power-of-two padding of the claim sort, the 4096-claim launches of
commit_claims and the max_rounds bound.

Every node's free stays within +-2^36 millicores / +-2^55 bytes after every mutating call (the range that keeps scores
inside int64), and a request that could take it outside is refused with KS_ERR_RANGE before anything changes.  After the
commits, ks_select (both kernel paths, both policies), ks_select_topk and ks_explain must equal the oracle on the
committed free[]: the bit-parallel index is rebuilt after every kind of commit."""
import numpy as np
import pytest

from explain_oracle import explain_packed
from gang_oracle import gang_bind_packed, groups
from test_least_alloc_float_model import _families

pytestmark = pytest.mark.gpu

LIM_C, LIM_M = 1 << 36, 1 << 55
KS_ERR_RANGE = -5
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
TOP = np.uint64(1 << 63)     # bit 63 of a label word; in the last word, bit 64W-1
ABSENT = np.uint64(1 << 62)  # bit 62 of word 0: no node carries it
DIRECT, BITPAR = 1, 2        # KS_SELECT_FORCE_DIRECT / KS_SELECT_FORCE_BITPAR

FAMILIES = ("adversarial", "homogeneous", "rising", "negative free", "tiny allocatable", "limits", "slice ties")
P_DEVICE = (1, 4, 5, 255, 256, 257, 1023, 1024)
N_DEVICE = (1, 127, 128, 129, 1023, 1025)


@pytest.fixture(scope="module")
def sms(ks):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _slices(N, sms):
    """k_stream_batch's node slices: grid = min(SMs, ceil(N/128)) CTAs of ceil(N/grid) nodes, the last ones maybe empty"""
    grid = max(1, min(sms, (N + 127) // 128))
    chunk = (N + grid - 1) // grid
    return grid, chunk


def _slice_edges(N, sms):
    grid, chunk = _slices(N, sms)
    e = {0, N - 1}
    for s in range(1, grid):
        e.update((s * chunk - 1, s * chunk))
    return np.array(sorted(x for x in e if 0 <= x < N), np.int64)


def _labels(rng, N, W, same):
    lab = rng.integers(0, 1 << 63, (N, W), dtype=np.uint64) | (rng.integers(0, 2, (N, W), dtype=np.uint64) << np.uint64(63))
    lab &= ~ABSENT
    if same:
        lab[:] = lab[0] | TOP
    return lab


def _selectors(rng, lab, P):
    """no selector; every pair some node carries; a sparse subset of them; bit 63 of every word; bit 64W-1 alone; a
    bit no node carries"""
    N, W = lab.shape
    kind = rng.integers(0, 6, P)
    src = lab[rng.integers(0, N, P)]
    sub = src & rng.integers(0, 1 << 63, (P, W), dtype=np.uint64) & rng.integers(0, 1 << 63, (P, W), dtype=np.uint64)
    sub &= rng.integers(0, 1 << 63, (P, W), dtype=np.uint64)
    sel = np.zeros((P, W), np.uint64)
    sel[kind == 1] = src[kind == 1]
    sel[kind == 2] = sub[kind == 2]
    sel[kind == 3] = TOP
    sel[kind == 4, W - 1] = TOP
    sel[kind == 5, 0] = ABSENT | sub[kind == 5, 0]
    return sel


def _family(name, rng, N, P, W, sms):
    """(ac, am, lab, fc, fm, rc, rm, sel): allocatable, labels, free[] and P pods; requests within [0, limit], as the
    committing calls require them"""
    def pick(vals, n):
        return rng.choice(np.array(vals, np.int64), n)

    lab = _labels(rng, N, W, same=name in ("homogeneous", "slice ties"))
    i = np.arange(N, dtype=np.int64)
    if name == "adversarial":  # the pools of test_gpu_parity.py::test_adversarial_values, requests made non-negative
        ac = pick([-5, 0, 1, 250, 1000, 1000, 4000, 64000, LIM_C // 2], N)
        am = pick([-1, 0, 1, 1 << 20, 1 << 30, 1 << 30, 1 << 34, LIM_M // 2], N)
        fc, fm = ac.copy(), am.copy()
        bn = rng.integers(0, N, 3 * N)
        np.subtract.at(fc, bn, pick([0, 0, 100, 1000, -100], 3 * N))
        np.subtract.at(fm, bn, pick([0, 1, 1 << 20, 1 << 28, -1], 3 * N))
        rc = pick([0, 0, 1, 250, 1000, 1001, 4000, 63999, LIM_C], P)
        rm = pick([0, 1, (1 << 20) - 1, 1 << 20, 1 << 30, (1 << 30) + 1, LIM_M], P)
    elif name == "homogeneous":  # one key everywhere: the lowest-index rule decides every choice
        ac, am = np.full(N, 4000, np.int64), np.full(N, 1 << 34, np.int64)
        fc, fm = ac.copy(), am.copy()
        rc = pick([0, 250, 500, 1000], P)
        rm = pick([0, 1 << 28, 1 << 30, 1 << 32], P)
    elif name == "rising":  # the score rises with the node index: the best node is N-1, last slice, last lane
        ac, am = np.full(N, 1 << 20, np.int64), np.full(N, 1 << 40, np.int64)
        fc = i * ((1 << 20) - (1 << 15)) // N
        fm = i * ((1 << 40) - (1 << 35)) // N
        fc[-1], fm[-1] = ac[-1], am[-1]
        rc = pick([0, 1, 100, 250], P)
        rm = pick([0, 1, 1 << 20, 1 << 24], P)
    elif name == "negative free":  # and zero requests against it
        ac, am = pick([0, 1000, 4000], N), pick([0, 1 << 30], N)
        fc = pick([-LIM_C, -1000, -1, 0, 0, 500, 4000], N)
        fm = pick([-LIM_M, -1, 0, 1 << 20, 1 << 30], N)
        rc, rm = pick([0, 0, 0, 1, 500], P), pick([0, 0, 1, 1 << 20], P)
    elif name == "tiny allocatable":  # allocatable <= 0 or a few units (LeastAllocated divides by it)
        ac, am = pick([-5, -1, 0, 1, 2, 3], N), pick([-3, 0, 1, 2, 1 << 20], N)
        fc = pick([-2, 0, 1, 2, 3, 1000, 4000], N)
        fm = pick([-1, 0, 1, 2, 1 << 20, 1 << 30], N)
        rc, rm = pick([0, 1, 2, 100], P), pick([0, 1, 2, 1 << 19], P)
    elif name == "limits":  # free, allocatable and requests at exactly the limits: (free - req) * 100 is largest here
        ac, am = pick([LIM_C, 1, -LIM_C, 0], N), pick([LIM_M, 1, -LIM_M, 0], N)
        fc = pick([LIM_C, LIM_C - 1, -LIM_C, 0, 1], N)
        fm = pick([LIM_M, LIM_M - 1, -LIM_M, 0, 1], N)
        rc, rm = pick([0, 1, LIM_C - 1, LIM_C], P), pick([0, 1, LIM_M - 1, LIM_M], P)
    elif name == "slice ties":  # the best key sits on both sides of every CTA slice boundary, tied
        ac, am = np.full(N, 4000, np.int64), np.full(N, 1 << 34, np.int64)
        fc, fm = np.full(N, 1000, np.int64), np.full(N, 1 << 32, np.int64)
        e = _slice_edges(N, sms)
        fc[e], fm[e] = 4000, 1 << 34
        rc, rm = pick([0, 1000, 1000, 1000], P), pick([0, 1 << 30], P)
    else:
        raise ValueError(name)
    return ac, am, lab, fc, fm, rc, rm, _selectors(rng, lab, P)


def _load(snap, ac, am, lab, fc, fm):
    """set_nodes + set_bound with two bound pods per node that leave exactly fc / fm (each pod within the limits)"""
    N = len(ac)
    dc, dm = ac - fc, am - fm
    bc = np.stack([dc // 2, dc - dc // 2], 1).reshape(-1)
    bm = np.stack([dm // 2, dm - dm // 2], 1).reshape(-1)
    snap.set_nodes(ac, am, lab)
    snap.set_bound(np.repeat(np.arange(N, dtype=np.int32), 2), bc, bm)
    gc, gm = snap.free()
    assert np.array_equal(gc, fc) and np.array_equal(gm, fm)


def _free_in_range(snap):
    fc, fm = snap.free()
    assert ((fc >= -LIM_C) & (fc <= LIM_C)).all(), "free_cpu outside +-2^36"
    assert ((fm >= -LIM_M) & (fm <= LIM_M)).all(), "free_mem outside +-2^55"
    return fc, fm


def _warm_index(snap, rc, rm, sel):
    """one bit-parallel select, so the index exists before the commit and a stale one would be used after it"""
    k = min(len(rc), 64)
    snap.select(rc[:k], rm[:k], sel[:k], flags=BITPAR)


def _check_derived(orc, snap, ac, am, lab, rc, rm, sel, tag):
    """ks_select on both paths and both policies, ks_select_topk entry 0 and ks_explain against the oracle on the
    snapshot's current free[]"""
    k = min(len(rc), 256)
    rc, rm, sel = rc[:k], rm[:k], sel[:k]
    fc, fm = snap.free()
    for policy in (0, 1):
        oidx, oscore, ocnt, _, _ = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, policy=policy, want_mask=False)
        for path, flag in (("direct", DIRECT), ("bitpar", BITPAR)):
            r = snap.select(rc, rm, sel, policy=policy, flags=flag)
            assert r.path == path
            assert np.array_equal(r.node_idx, oidx), f"select node_idx {path} policy {policy} {tag}"
            assert np.array_equal(r.score, oscore), f"select score {path} policy {policy} {tag}"
            assert np.array_equal(r.feasible_cnt, ocnt), f"select feasible_cnt {path} policy {policy} {tag}"
        ti, ts, tc = snap.select_topk(rc, rm, sel, 1, policy)
        assert np.array_equal(ti[:, 0], oidx) and np.array_equal(ts[:, 0], oscore), f"topk policy {policy} {tag}"
        assert np.array_equal(tc, ocnt), f"topk count policy {policy} {tag}"
    assert np.array_equal(snap.explain(rc, rm, sel), explain_packed(orc, fc, fm, lab, rc, rm, sel)), f"explain {tag}"


def _stream_case(orc, snap, fam, policy, path, tag):
    ac, am, lab, fc, fm, rc, rm, sel = fam
    _load(snap, ac, am, lab, fc, fm)
    _warm_index(snap, rc, rm, sel)
    ofc, ofm = fc.copy(), fm.copy()
    oidx, oscore, orounds = orc.stream_bind_packed(ofc, ofm, ac, am, lab, rc, rm, sel, policy=policy)
    idx, score, rounds = snap.stream_bind(rc, rm, sel, policy=policy)
    assert snap.last_path() == path, tag
    assert np.array_equal(idx, oidx), f"node_idx {tag}"
    assert np.array_equal(score, oscore), f"score {tag}"
    assert rounds == orounds, f"rounds {tag}"
    gfc, gfm = _free_in_range(snap)
    assert np.array_equal(gfc, ofc) and np.array_equal(gfm, ofm), f"free {tag}"
    _check_derived(orc, snap, ac, am, lab, rc, rm, sel, tag)
    return idx, rounds


# ---------------------------------------------------------------------------------------------------- ks_stream_bind
@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("P", P_DEVICE)
def test_stream_bind_device_loop(ks, orc, sms, P, W, policy):
    """k_stream_batch at every N of N_DEVICE (one, and around one 128-node slice and a thousand), a value family per
    shape; P around the 4-pod loser strips and the power-of-two padding of the claim sort"""
    rng = np.random.default_rng(P * 1009 + W * 31 + policy)
    with ks.Snapshot(0) as snap:
        for j, N in enumerate(N_DEVICE):
            fam_name = FAMILIES[(j + P + W + policy) % len(FAMILIES)]
            fam = _family(fam_name, rng, N, P, W, sms)
            _stream_case(orc, snap, fam, policy, "stream_batch", f"P={P} N={N} W={W} policy={policy} {fam_name}")


def _sm_derived_n(sms):
    """the smallest N with sms CTAs whose last slice is empty, and the smallest whose last slice holds one node"""
    empty = single = None
    for N in range(128 * (sms - 1) + 1, 128 * (sms + 2)):
        grid, chunk = _slices(N, sms)
        if grid != sms:
            continue
        if empty is None and (grid - 1) * chunk >= N:
            empty = N
        if single is None and (grid - 1) * chunk == N - 1:
            single = N
    assert empty is not None and single is not None
    return empty, single


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("which", ["last slice empty", "last slice one node"])
def test_stream_bind_sm_derived_slices(ks, orc, sms, which, W, policy):
    """N chosen from the device's SM count so that k_stream_batch's last CTA scans no node, or exactly one (132 SMs:
    N = 16 897 and 16 769); the best node sits at the end (rising), ties straddle every slice boundary, and one key is
    everywhere (homogeneous)"""
    empty, single = _sm_derived_n(sms)
    N = empty if which == "last slice empty" else single
    grid, chunk = _slices(N, sms)
    assert grid == sms and ((grid - 1) * chunk >= N if N == empty else (grid - 1) * chunk == N - 1)
    rng = np.random.default_rng(N + 7 * W + policy)
    with ks.Snapshot(0) as snap:
        for fam_name, P in (("rising", 1024), ("slice ties", 257), ("homogeneous", 257)):
            fam = _family(fam_name, rng, N, P, W, sms)
            idx, _ = _stream_case(orc, snap, fam, policy, "stream_batch", f"{which} N={N} W={W} policy={policy} {fam_name}")
            if fam_name == "rising":
                assert (idx == N - 1).any()


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("W", [2, 8])
@pytest.mark.parametrize("P", [1025, 5000])
def test_stream_bind_host_loop(ks, orc, sms, P, W, policy):
    """above 1024 pods: per-cell select + commit_claims per round.  Identical nodes make every pod of the first round
    claim the same node, so its claims span the 4096-claim launches of commit_claims and arrival order must survive
    the cut"""
    rng = np.random.default_rng(P + W + policy)
    with ks.Snapshot(0) as snap:
        for fam_name, N in (("homogeneous", 300), ("adversarial", 700), ("limits", 129)):
            fam = list(_family(fam_name, rng, N, P, W, sms))
            if fam_name == "homogeneous":  # about 64 pods per node: tens of rounds, not thousands
                fam[0] = fam[3] = np.full(N, 32000, np.int64)
                fam[1] = fam[4] = np.full(N, 1 << 36, np.int64)
            _stream_case(orc, snap, tuple(fam), policy, "direct", f"host loop P={P} N={N} W={W} policy={policy} {fam_name}")


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("N", [1024, 1023])
def test_stream_bind_worst_case_rounds(ks, N, policy):
    """1024 identical pods on identical nodes that each fit exactly one: every round all pending pods claim the lowest
    free node and only the first wins, so pod i gets node i in round i + 1; with one node too few the last pod gets
    -1 in round 1024.  Pins max_rounds = n + 1 and the loser order through every CTA slice, without an oracle."""
    P = 1024
    for W in (1, 8):
        ac, am = np.full(N, 1000, np.int64), np.full(N, 1 << 30, np.int64)
        lab = np.zeros((N, W), np.uint64)
        rc, rm = np.full(P, 1000, np.int64), np.full(P, 1 << 30, np.int64)
        sel = np.zeros((P, W), np.uint64)
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            idx, score, rounds = snap.stream_bind(rc, rm, sel, policy=policy)
            assert snap.last_path() == "stream_batch"
            fc, fm = _free_in_range(snap)
        want = np.arange(P, dtype=np.int32)
        want[want >= N] = -1
        assert np.array_equal(idx, want) and (score == 0).all() and rounds == 1024, f"N={N} W={W}"
        assert (fc == 0).all() and (fm == 0).all()


# ------------------------------------------------------------------------------------------ ks_snapshot_commit_claims
@pytest.mark.parametrize("n", [1, 2, 3, 4095, 4096, 4097, 8192, 8193, 12288])
def test_commit_claims_edges(ks, orc, sms, n):
    """every claim to one node (a single segment spans the whole sort and every 4096-claim launch), then claims over
    all nodes mixed with indices that name no node (-1, -2, INT32_MIN, N, INT32_MAX: never accepted)"""
    rng = np.random.default_rng(n)
    N = 1025
    with ks.Snapshot(0) as snap:
        for fam_name in ("adversarial", "negative free", "limits", "homogeneous", "tiny allocatable"):
            ac, am, lab, fc, fm, rc, rm, sel = _family(fam_name, rng, N, n, 2, sms)
            if fam_name == "homogeneous":
                rc, rm = rc // 100, rm // 100  # hundreds of claims fit before the node runs out
            _load(snap, ac, am, lab, fc, fm)
            _warm_index(snap, rc, rm, sel)
            one = np.full(n, int(np.argmax(fc)), np.int32)
            mixed = rng.integers(0, N, n).astype(np.int32)
            bad = rng.random(n) < 0.2
            mixed[bad] = rng.choice(np.array([-1, -2, INT32_MIN, N, INT32_MAX], np.int64), int(bad.sum()))
            for claims, what in ((one, "one node"), (mixed, "mixed")):
                tag = f"n={n} {fam_name} {what}"
                acc = snap.commit_claims(claims, rc, rm)
                oacc = orc.commit_claims(fc, fm, claims, rc, rm)
                assert np.array_equal(acc, oacc), f"accepted {tag}"
                assert not acc[(claims < 0) | (claims >= N)].any(), tag
                gfc, gfm = _free_in_range(snap)
                assert np.array_equal(gfc, fc) and np.array_equal(gfm, fm), f"free {tag}"
                _check_derived(orc, snap, ac, am, lab, rc, rm, sel, tag)


# ------------------------------------------------------------------------------------------------------ ks_gang_bind
def _gang_case(orc, snap, fam, off, mm, policy, tag):
    ac, am, lab, fc, fm, rc, rm, sel = fam
    ofc, ofm = snap.free()
    want = gang_bind_packed(orc, ofc, ofm, ac, am, lab, rc, rm, sel, off, mm, policy)
    got = snap.gang_bind(rc, rm, sel, off, mm, policy)
    assert snap.last_path() == "gang_batch"
    for name, g, w in zip(("node_idx", "score", "placed", "rounds"), got, want):
        assert g.dtype == w.dtype and np.array_equal(g, w), f"{name} {tag}"
    gfc, gfm = _free_in_range(snap)
    assert np.array_equal(gfc, ofc) and np.array_equal(gfm, ofm), f"free {tag}"
    return got


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("fam_name", FAMILIES)
def test_gang_edge_families_w8(ks, orc, sms, fam_name, policy):
    """k_gang_batch at W = 8 on every value family, with min_member = size on every group, then with mixed minimums"""
    rng = np.random.default_rng(FAMILIES.index(fam_name) * 10 + policy)
    P, N = 2000, 1025
    fam = _family(fam_name, rng, N, P, 8, sms)
    ac, am, lab, fc, fm, rc, rm, sel = fam
    off = groups(rng, P, 1, 200)
    size = np.diff(off).astype(np.uint32)
    with ks.Snapshot(0) as snap:
        _load(snap, ac, am, lab, fc, fm)
        _warm_index(snap, rc, rm, sel)
        _, _, placed, _ = _gang_case(orc, snap, fam, off, size, policy, f"{fam_name} policy={policy} min=size")
        _check_derived(orc, snap, ac, am, lab, rc, rm, sel, f"{fam_name} after min=size")
        mm = (rng.random(len(size)) * (size + 1)).astype(np.uint32)
        _gang_case(orc, snap, fam, off, mm, policy, f"{fam_name} policy={policy} mixed min")
        _check_derived(orc, snap, ac, am, lab, rc, rm, sel, f"{fam_name} after mixed min")


@pytest.mark.parametrize("policy", [0, 1])
def test_gang_zero_request_groups_are_placed(ks, orc, sms, policy):
    """groups made only of zero-request pods fit every matching node with free >= 0: all placed, all committed,
    free[] unchanged - also on a cluster where most nodes have negative free"""
    rng = np.random.default_rng(40 + policy)
    P, N = 1500, 1025
    fam = list(_family("negative free", rng, N, P, 8, sms))
    fam[3][-1], fam[4][-1] = 0, 0  # at least one node with free >= 0
    fam[5], fam[6] = np.zeros(P, np.int64), np.zeros(P, np.int64)
    fam[7] = np.zeros((P, 8), np.uint64)
    ac, am, lab, fc, fm, rc, rm, sel = fam
    off = groups(rng, P, 1, 300)
    size = np.diff(off).astype(np.uint32)
    with ks.Snapshot(0) as snap:
        _load(snap, ac, am, lab, fc, fm)
        idx, _, placed, _ = _gang_case(orc, snap, tuple(fam), off, size, policy, f"zero requests policy={policy}")
        assert np.array_equal(placed, size) and (idx >= 0).all()
        gfc, gfm = snap.free()
        assert np.array_equal(gfc, fc) and np.array_equal(gfm, fm)


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("fam_name", ["negative free", "limits"])
def test_gang_rollbacks_restore_free_bit_for_bit(ks, orc, sms, fam_name, policy):
    """group by group, all or nothing: after a group that rolls back free[] is exactly what it was before it (the
    atomics add back values up to 2^55), after one that commits it is the oracle's"""
    rng = np.random.default_rng(50 + policy + (fam_name == "limits"))
    P, N = 1200, 257
    fam = _family(fam_name, rng, N, P, 8, sms)
    ac, am, lab, fc, fm, rc, rm, sel = fam
    off = groups(rng, P, 2, 40)
    size = np.diff(off).astype(np.uint32)
    mm = np.where(np.arange(len(size)) % 2 == 0, size, 1).astype(np.uint32)  # all or nothing / at least one
    rolled = committed = 0
    with ks.Snapshot(0) as snap:
        _load(snap, ac, am, lab, fc, fm)
        for g in range(len(size)):
            a, b = int(off[g]), int(off[g + 1])
            one = (rc[a:b], rm[a:b], sel[a:b])
            before = snap.free()
            _, _, placed, _ = _gang_case(orc, snap, (ac, am, lab, fc, fm) + one, np.array([0, b - a], np.uint64),
                                         mm[g:g + 1], policy, f"{fam_name} group {g}")
            if placed[0] < mm[g]:
                rolled += placed[0] > 0  # something was charged and had to be given back
                after = snap.free()
                assert np.array_equal(after[0], before[0]) and np.array_equal(after[1], before[1]), f"group {g}"
            else:
                committed += 1
        _check_derived(orc, snap, ac, am, lab, rc, rm, sel, f"{fam_name} after the groups")
    assert rolled > 0 and committed > 0


# ------------------------------------------------------------------------------------------------------- ks_stream
@pytest.mark.parametrize("max_batch", [1, 3, 1024])
def test_async_queue_w8_least_allocated(ks, orc, sms, max_batch):
    """the queue at W = 8 under LeastAllocated: with a flush after every submit the dispatcher cuts each submit into
    max_batch-pod micro-batches in arrival order, so the results equal the oracle's stream loop batch by batch"""
    rng = np.random.default_rng(60 + max_batch)
    P, N = 1400, 500
    ac, am, lab, fc, fm, rc, rm, sel = _family("adversarial", rng, N, P, 8, sms)
    with ks.Snapshot(0) as snap:
        _load(snap, ac, am, lab, fc, fm)
        _warm_index(snap, rc, rm, sel)
        ofc, ofm = fc.copy(), fm.copy()
        with ks.Stream(snap, policy=ks.KS_SCORE_LEAST_ALLOCATED, max_batch=max_batch) as q:
            lo = 0
            for size in (1, 7, 300, 2, 1024 - 334 + 1, 66):
                hi = min(P, lo + size)
                q.submit(rc[lo:hi], rm[lo:hi], sel[lo:hi], np.arange(lo, hi, dtype=np.uint64))
                q.flush()
                t, i, s = q.poll()
                assert sorted(t.tolist()) == list(range(lo, hi))
                order = np.argsort(t)
                for a in range(lo, hi, max_batch):
                    b = min(hi, a + max_batch)
                    oidx, oscore, _ = orc.stream_bind_packed(ofc, ofm, ac, am, lab, rc[a:b], rm[a:b], sel[a:b], policy=1)
                    assert np.array_equal(i[order][a - lo:b - lo], oidx), f"batch [{a}, {b})"
                    assert np.array_equal(s[order][a - lo:b - lo], oscore), f"batch [{a}, {b})"
                lo = hi
            batches, _, max_seen = q.stats()
            assert max_seen == min(max_batch, 691) and batches >= 6
        gfc, gfm = _free_in_range(snap)
        assert np.array_equal(gfc, ofc) and np.array_equal(gfm, ofm)
        _check_derived(orc, snap, ac, am, lab, rc, rm, sel, f"queue max_batch={max_batch}")


# --------------------------------------------------------------------------------------- the range of free[] is kept
def test_apply_bind_refuses_to_leave_the_limits(ks, orc):
    """A node with free_mem = 2^55: a negative-request bind that would raise it to 2^56 (and a second one to 3*2^55,
    where the bit-parallel and the per-cell select used to disagree) is refused and free[] is unchanged; binds and
    releases that stay within the limits, up to exactly the limits, go through."""
    N = 4
    ac = np.array([1000, 1000, LIM_C, 1000], np.int64)
    am = np.array([LIM_M, 1 << 30, 1 << 30, 1 << 30], np.int64)
    lab = np.zeros((N, 1), np.uint64)
    rc, rm, sel = np.array([0, 1], np.int64), np.array([0, 1], np.int64), np.zeros((2, 1), np.uint64)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        _warm_index(snap, rc, rm, sel)

        def refused(*binds):
            before = snap.free()
            for node, c, m in binds:
                with pytest.raises(ks.KsError) as e:
                    snap.apply_bind(node, c, m)
                assert e.value.code == KS_ERR_RANGE, (node, c, m)
                after = _free_in_range(snap)
                assert np.array_equal(after[0], before[0]) and np.array_equal(after[1], before[1]), (node, c, m)

        refused((0, 0, -LIM_M), (0, 0, -LIM_M), (2, -1, 0), (1, -LIM_C, 0), (3, -LIM_C, -LIM_M))
        _check_derived(orc, snap, ac, am, lab, rc, rm, sel, "after refused binds")
        snap.apply_bind(1, 100, 1 << 20)  # a bind ...
        snap.apply_bind(1, -100, -(1 << 20))  # ... and its release by the negated request
        snap.apply_bind(0, 0, LIM_M)  # down to 0
        snap.apply_bind(0, 0, LIM_M)  # to exactly -2^55
        snap.apply_bind(2, LIM_C, 0)  # 0
        snap.apply_bind(2, LIM_C, 0)  # exactly -2^36
        fc, fm = _free_in_range(snap)
        assert fc.tolist() == [1000, 1000, -LIM_C, 1000] and fm.tolist() == [-LIM_M, 1 << 30, 1 << 30, 1 << 30]
        refused((0, 0, 1), (2, 1, 0), (2, LIM_C, LIM_M))
        _check_derived(orc, snap, ac, am, lab, rc, rm, sel, "after binds at the limits")


BAD_REQUESTS = [(-1, 0), (0, -1), (LIM_C + 1, 0), (0, LIM_M + 1), (INT64_MIN, 0), (0, INT64_MAX)]


@pytest.mark.parametrize("bad", BAD_REQUESTS, ids=["cpu -1", "mem -1", "cpu 2^36+1", "mem 2^55+1", "cpu INT64_MIN",
                                                   "mem INT64_MAX"])
@pytest.mark.parametrize("call", ["commit_claims", "stream_bind", "stream_bind host loop", "gang_bind", "Stream.submit"])
def test_committing_calls_refuse_out_of_range_requests(ks, orc, sms, call, bad):
    """one request outside [0, limit] fails the whole call with KS_ERR_RANGE before any device work: free[] unchanged,
    nothing of the call committed.  (A negative request always fits and raises free[]; one above the limit fits a
    negative-free node in the oracle's terms but leaves the range.)"""
    rng = np.random.default_rng(70)
    P = 1025 if call == "stream_bind host loop" else 40
    N = 64
    ac, am, lab, fc, fm, rc, rm, sel = _family("homogeneous", rng, N, P, 1, sms)
    rc, rm = rc.copy(), rm.copy()
    rc[P // 2], rm[P // 2] = bad
    with ks.Snapshot(0) as snap:
        _load(snap, ac, am, lab, fc, fm)
        if call == "Stream.submit":
            with ks.Stream(snap) as q:
                with pytest.raises(ks.KsError) as e:
                    q.submit(rc, rm, sel, np.arange(P, dtype=np.uint64))
                q.flush()
                t, _, _ = q.poll()
                assert len(t) == 0  # the refused submit queued nothing
                # and the queue keeps working
                q.submit(rc[:3], rm[:3], sel[:3], np.arange(3, dtype=np.uint64))
                q.flush()
                t, i, s = q.poll()
            order = np.argsort(t)
            oidx, oscore, _ = orc.stream_bind_packed(fc, fm, ac, am, lab, rc[:3], rm[:3], sel[:3])
            assert np.array_equal(t[order], np.arange(3)) and np.array_equal(i[order], oidx)
            assert np.array_equal(s[order], oscore)
        else:
            with pytest.raises(ks.KsError) as e:
                if call == "commit_claims":
                    snap.commit_claims(np.zeros(P, np.int32), rc, rm)
                elif call.startswith("stream_bind"):
                    snap.stream_bind(rc, rm, sel)
                else:
                    snap.gang_bind(rc, rm, sel, np.array([0, P // 2, P], np.uint64), np.zeros(2, np.uint32))
        assert e.value.code == KS_ERR_RANGE
        gfc, gfm = _free_in_range(snap)
        assert np.array_equal(gfc, fc) and np.array_equal(gfm, fm)


# ------------------------------------------------------------------------------ LeastAllocated single-precision guards
FLOAT_FAMILIES = ("realistic", "round fills", "api limits", "tiny allocatable", "zero and negative allocatable",
                  "24-bit edge", "quotient near 2^24")


@pytest.mark.parametrize("family", FLOAT_FAMILIES)
def test_least_allocated_float_families_on_both_paths(ks, orc, family):
    """the value families of the CPU model in test_least_alloc_float_model.py through the kernels themselves: the
    guards of k_least_alloc's float shortcut (x < 2^24, pc < 4e6, |qm| + em < 4e6) on the bit-parallel path, and the
    per-cell kernel, both equal to the oracle's integers"""
    rng = np.random.default_rng(3)
    N, P = 1500, 300
    fams = {f[0]: f[1:] for f in _families(rng, N, P)}
    assert set(fams) == set(FLOAT_FAMILIES)
    fc, fm, ac, am, rc, rm = (np.asarray(a, np.int64) for a in fams[family])
    lab = np.zeros((N, 1), np.uint64)
    sel = np.zeros((P, 1), np.uint64)
    o = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, policy=1)
    with ks.Snapshot(0) as snap:
        _load(snap, ac, am, lab, fc, fm)
        for path, flag in (("direct", DIRECT), ("bitpar", BITPAR)):
            r = snap.select(rc, rm, sel, policy=ks.KS_SCORE_LEAST_ALLOCATED, flags=flag, want_mask=True)
            assert r.path == path
            for name, g, w in zip(("node_idx", "score", "feasible_cnt", "mask"), (r.node_idx, r.score, r.feasible_cnt,
                                                                                   r.mask), o):
                assert np.array_equal(g, w), f"{family} {path} {name}"
        assert (o[0] >= 0).any()
