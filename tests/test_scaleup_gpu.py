"""Scale-up estimate (ks_scaleup_estimate) on the GPU: every row, node ordinal and reason count bit for bit against the
restatement of tests/scaleup_oracle.py, across label widths, template and pod counts up to the limits, max_nodes from 0
to 1024, tie-heavy orders, zero requests, empty and negative capacities, values at the template limits and selectors;
the snapshot untouched; templates split over calls; and the argument and range errors."""
import ctypes as C

import numpy as np
import pytest

from explain_oracle import explain_packed
from helpers import load_golden
from scaleup_oracle import best_template, packed_from_specs, scaleup_packed
from test_scaleup import _host_case

pytestmark = pytest.mark.gpu

LC, LM = 1 << 26, 1 << 45  # template limits: KS_MAX_CPU_MILLI >> 10, KS_MAX_MEM_BYTES >> 10


def _setup(ks, W=1, seed=0):
    cl = ks.synth.make(50, 200, seed=0x5C00 + seed, bound_per_node=2)
    ac, am, lab, bn, bc, bm, _, _, _ = cl.packed()
    return ac, am, lab, bn, bc, bm


def _pods(rng, P, W, cpu_hi=8000, mem_hi=32 << 30, sel_p=0.3, bits=None):
    rc = rng.integers(0, cpu_hi + 1, P).astype(np.int64)
    rm = rng.integers(0, mem_hi + 1, P).astype(np.int64)
    sel = np.zeros((P, W), np.uint64)
    bits = bits if bits is not None else 64 * W
    for p in np.nonzero(rng.random(P) < sel_p)[0]:
        for b in rng.choice(bits, rng.integers(1, 3), replace=False):
            sel[p, b // 64] |= np.uint64(1) << np.uint64(b % 64)
    return rc, rm, sel


def _templates(rng, T, W, max_nodes=None, dense=0.5):
    ac = rng.choice([2000, 4000, 8000, 16000, 32000, 64000], T).astype(np.int64)
    am = rng.choice([8, 16, 32, 64, 128, 256], T).astype(np.int64) << 30
    ds_c = rng.integers(0, 500, T)
    ds_m = rng.integers(0, 1 << 30, T)
    fc, fm = ac - ds_c, am - ds_m
    lab = np.zeros((T, W), np.uint64)
    on = rng.random((T, W * 64)) < dense
    for t in range(T):
        for b in np.nonzero(on[t])[0]:
            lab[t, b // 64] |= np.uint64(1) << np.uint64(b % 64)
    mx = rng.integers(0, 40, T).astype(np.uint32) if max_nodes is None else np.full(T, max_nodes, np.uint32)
    return ac, am, fc, fm, lab, mx


def _check(ks, orc, rc, rm, sel, ac, am, fc, fm, lab, mx, snap=None):
    def run(s):
        return s.scaleup_estimate(rc, rm, sel, ac, am, fc, fm, lab, mx)
    if snap is None:
        with ks.Snapshot(0) as s:
            got = run(s)
    else:
        got = run(snap)
    want = scaleup_packed(orc, ac, am, fc, fm, lab, mx, rc, rm, sel)
    rows, best, node, why = got
    w_rows, w_best, w_node, w_why = want
    for f in w_rows.dtype.names:
        assert np.array_equal(rows[f], w_rows[f]), f
    assert best == w_best
    assert np.array_equal(node, w_node)
    assert np.array_equal(why, w_why)
    # not_enough_resources + node_selector_mismatch + (templates the pod is eligible for) = T, summed over the pods
    assert (len(ac) - why[:, 2].astype(np.int64) - why[:, 3]).sum() == rows["eligible"].sum()
    return got


@pytest.mark.parametrize("W", [1, 2, 4, 8])
def test_label_widths(ks, orc, W):
    rng = np.random.default_rng(100 + W)
    rc, rm, sel = _pods(rng, 700, W)
    ac, am, fc, fm, lab, mx = _templates(rng, 37, W)
    rows = _check(ks, orc, rc, rm, sel, ac, am, fc, fm, lab, mx)[0]
    assert rows["placed"].sum() > 0 and (rows["placed"] < rows["eligible"]).any()


@pytest.mark.parametrize("T,P", [(1, 1), (1, 65536), (4096, 1), (4096, 64), (300, 2000), (133, 257)])
def test_sizes(ks, orc, T, P):
    rng = np.random.default_rng(T * 7 + P)
    rc, rm, sel = _pods(rng, P, 1, cpu_hi=4000, mem_hi=8 << 30, sel_p=0.1)
    ac, am, fc, fm, lab, mx = _templates(rng, T, 1, dense=0.8)
    if T == 1:
        mx[:] = 1024
    _check(ks, orc, rc, rm, sel, ac, am, fc, fm, lab, mx)


def test_max_nodes_0_1_small_and_1024_exactly(ks, orc):
    rng = np.random.default_rng(7)
    rc, rm, sel = _pods(rng, 3000, 1, sel_p=0.0)
    ac, am, fc, fm, lab, _ = _templates(rng, 4, 1)
    lab[:] = 0
    for m in (0, 1, 3):
        rows = _check(ks, orc, rc, rm, sel, ac, am, fc, fm, lab, np.full(4, m, np.uint32))[0]
        assert (rows["nodes"] == m).all() if m else (rows["placed"] == 0).all()
    # 2048 identical pods that each fill a node: ordinals 0..1023 across every warp of the walk, then the limit
    rc = np.full(2048, 4000, np.int64)
    rm = np.full(2048, 16 << 30, np.int64)
    sel = np.zeros((2048, 1), np.uint64)
    ac = np.array([4000], np.int64)
    am = np.array([16 << 30], np.int64)
    rows, best, node, _ = _check(ks, orc, rc, rm, sel, ac, am, ac, am, np.zeros((1, 1), np.uint64),
                                 np.array([1024], np.uint32))
    assert rows["nodes"][0] == 1024 and rows["placed"][0] == 1024 and rows["utilization"][0] == 100
    assert np.array_equal(node[0, :1024], np.arange(1024)) and (node[0, 1024:] == -1).all()


def test_identical_pods_take_ceil_nodes(ks, orc):
    rc = np.full(1000, 700, np.int64)
    rm = np.full(1000, 1 << 30, np.int64)
    ac = np.array([4000, 3000, 64000], np.int64)
    am = np.array([64 << 30, 64 << 30, 4 << 30], np.int64)
    rows = _check(ks, orc, rc, rm, np.zeros((1000, 1), np.uint64), ac, am, ac, am, np.zeros((3, 1), np.uint64),
                  np.full(3, 1024, np.uint32))[0]
    per = np.minimum(ac // 700, am // (1 << 30))
    assert rows["nodes"].tolist() == (-(-1000 // per)).tolist()


def test_tie_heavy_orders(ks, orc):
    """(300, 100) and (100, 300) against A_c = A_m give equal keys; the pod index decides."""
    rng = np.random.default_rng(11)
    base = np.array([[300, 100], [100, 300], [200, 200], [400, 0], [0, 400]], np.int64)
    k = rng.integers(0, len(base), 5000)
    rc, rm = base[k, 0] * 10, base[k, 1] * 10
    ac = np.array([1000, 1000, 3000, 2000], np.int64)
    am = np.array([1000, 3000, 1000, 2000], np.int64)
    mx = np.array([1024, 40, 7, 1024], np.uint32)
    _check(ks, orc, rc, rm, np.zeros((5000, 1), np.uint64), ac, am, ac, am, np.zeros((4, 1), np.uint64), mx)


def test_zero_requests_and_empty_or_negative_capacity(ks, orc):
    rng = np.random.default_rng(12)
    rc, rm, sel = _pods(rng, 800, 1, sel_p=0.0)
    rc[::3] = 0
    rm[::3] = 0
    rm[1::5] = 0
    ac = np.array([4000, 4000, 4000, 4000, 4000], np.int64)
    am = np.array([8 << 30] * 5, np.int64)
    fc = np.array([0, -1, 4000, 0, -LC], np.int64)
    fm = np.array([0, 8 << 30, -1, 8 << 30, -LM], np.int64)
    rows = _check(ks, orc, rc, rm, sel, ac, am, fc, fm, np.zeros((5, 1), np.uint64), np.full(5, 1024, np.uint32))[0]
    assert rows["eligible"][1] == 0 and rows["eligible"][2] == 0 and rows["eligible"][4] == 0
    assert rows["eligible"][0] == ((rc == 0) & (rm == 0)).sum()


def test_values_at_the_template_limits(ks, orc):
    """A and requests at 2^26 m / 2^45 B: keys up to 2^72, the wide compare."""
    rng = np.random.default_rng(13)
    P = 3000
    rc = rng.integers(0, LC + 1, P).astype(np.int64)
    rm = rng.integers(0, LM + 1, P).astype(np.int64)
    rc[:100], rm[:100] = LC, LM
    rc[100:200], rm[100:200] = LC - rng.integers(0, 3, 100), LM - rng.integers(0, 3, 100)
    ac = np.array([LC, LC, 1, LC, LC - 1], np.int64)
    am = np.array([LM, 1, LM, LM - 1, LM], np.int64)
    fc = np.array([LC, 1, 1, LC - 5, LC - 1], np.int64)
    fm = np.array([LM, 1, LM, LM - 7, LM], np.int64)
    mx = np.array([1024, 1024, 1024, 3, 1024], np.uint32)
    rows = _check(ks, orc, rc, rm, np.zeros((P, 1), np.uint64), ac, am, fc, fm, np.zeros((5, 1), np.uint64), mx)[0]
    assert rows["nodes"][0] == 1024 and rows["used_mem"][0] > (1 << 53)


def test_selectors(ks, orc):
    """Pairs only some templates carry, the never-set bit (the last bit of the last word), dense selectors."""
    rng = np.random.default_rng(14)
    for W in (1, 4):
        P, T = 2000, 24
        rc, rm, sel = _pods(rng, P, W, sel_p=0.6, bits=8)
        dense = np.nonzero(rng.random(P) < 0.1)[0]
        sel[dense] = rng.integers(0, 1 << 62, (len(dense), W), dtype=np.int64).astype(np.uint64) & np.uint64(0x0f0f0f0f0f0f0f0f)
        sel[::17, -1] |= np.uint64(1) << np.uint64(63)  # never set on a template
        ac, am, fc, fm, lab, mx = _templates(rng, T, W, dense=0.3)
        lab[:, -1] &= ~(np.uint64(1) << np.uint64(63))
        lab[:3] = np.uint64(0x0f0f0f0f0f0f0f0f)  # carry every dense pair
        rows, _, _, why = _check(ks, orc, rc, rm, sel, ac, am, fc, fm, lab, mx)
        assert why[:, 3].sum() > 0 and (why[::17, 3] + why[::17, 2] == T).all()


def test_no_side_effects(ks, orc):
    ac0, am0, lab0, bn, bc, bm = _setup(ks)
    rng = np.random.default_rng(15)
    rc, rm, sel = _pods(rng, 500, 1)
    ac, am, fc, fm, lab, mx = _templates(rng, 20, 1)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac0, am0, lab0)
        snap.set_bound(bn, bc, bm)
        before = snap.free()
        sel0 = np.zeros((len(rc), lab0.shape[1]), np.uint64)
        r0 = snap.select(rc, rm, sel0)
        _check(ks, orc, rc, rm, sel, ac, am, fc, fm, lab, mx, snap=snap)
        after = snap.free()
        r1 = snap.select(rc, rm, sel0)
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    assert np.array_equal(r0.node_idx, r1.node_idx) and np.array_equal(r0.score, r1.score)


def test_templates_split_over_calls_give_the_same_rows(ks, orc):
    rng = np.random.default_rng(16)
    rc, rm, sel = _pods(rng, 3000, 2)
    ac, am, fc, fm, lab, mx = _templates(rng, 50, 2)
    with ks.Snapshot(0) as snap:
        whole = snap.scaleup_estimate(rc, rm, sel, ac, am, fc, fm, lab, mx)
        a = snap.scaleup_estimate(rc, rm, sel, ac[:17], am[:17], fc[:17], fm[:17], lab[:17], mx[:17])
        b = snap.scaleup_estimate(rc, rm, sel, ac[17:], am[17:], fc[17:], fm[17:], lab[17:], mx[17:])
    assert np.array_equal(np.concatenate([a[0], b[0]]), whole[0])
    assert np.array_equal(np.concatenate([a[2], b[2]]), whole[2])
    assert np.array_equal(a[3] + b[3], whole[3])
    assert best_template(np.concatenate([a[0], b[0]])) == whole[1]


def test_reasons_equal_explain_over_the_templates(ks, orc):
    rng = np.random.default_rng(17)
    rc, rm, sel = _pods(rng, 4000, 2, sel_p=0.5, bits=16)
    ac, am, fc, fm, lab, mx = _templates(rng, 300, 2, dense=0.4)
    _, _, _, why = _check(ks, orc, rc, rm, sel, ac, am, fc, fm, lab, mx)
    assert np.array_equal(why, explain_packed(orc, fc, fm, lab, rc, rm, sel))


def test_optional_outputs_and_empty_calls(ks, orc):
    rng = np.random.default_rng(18)
    rc, rm, sel = _pods(rng, 300, 1)
    ac, am, fc, fm, lab, mx = _templates(rng, 9, 1)
    want = scaleup_packed(orc, ac, am, fc, fm, lab, mx, rc, rm, sel)
    with ks.Snapshot(0) as snap:
        rows, best, node, why = snap.scaleup_estimate(rc, rm, sel, ac, am, fc, fm, lab, mx, want_nodes=False,
                                                      want_reasons=False)
        assert node is None and why is None and np.array_equal(rows, want[0]) and best == want[1]
        rows, best, node, why = snap.scaleup_estimate(rc[:0], rm[:0], sel[:0], ac, am, fc, fm, lab, mx)
        assert best == -1 and (rows["placed"] == 0).all() and (rows["nodes"] == 0).all() and node.shape == (9, 0)
        rows, best, node, why = snap.scaleup_estimate(rc, rm, sel, ac[:0], am[:0], fc[:0], fm[:0], lab[:0], mx[:0])
        assert best == -1 and len(rows) == 0 and (why == 0).all()


def test_argument_and_range_errors(ks):
    E = ks.capi
    rng = np.random.default_rng(19)
    rc, rm, sel = _pods(rng, 10, 1)
    ac, am, fc, fm, lab, mx = _templates(rng, 3, 1)
    with ks.Snapshot(0) as snap:
        def code(**kw):
            a = dict(req_cpu=rc, req_mem=rm, sel=sel, alloc_cpu=ac, alloc_mem=am, free_cpu=fc, free_mem=fm, labels=lab,
                     max_nodes=mx)
            a.update(kw)
            with pytest.raises(ks.KsError) as e:
                snap.scaleup_estimate(**a)
            return e.value.code

        assert code(alloc_cpu=np.array([0, 1, 1])) == E.KS_ERR_RANGE
        assert code(alloc_cpu=np.array([LC + 1, 1, 1]), free_cpu=np.array([0, 0, 0])) == E.KS_ERR_RANGE
        assert code(alloc_mem=np.array([LM + 1, 1, 1]), free_mem=np.array([0, 0, 0])) == E.KS_ERR_RANGE
        assert code(free_cpu=ac + 1) == E.KS_ERR_RANGE
        assert code(free_mem=np.full(3, -LM - 1)) == E.KS_ERR_RANGE
        assert code(max_nodes=np.array([1025, 1, 1])) == E.KS_ERR_RANGE
        assert code(req_cpu=np.r_[rc[:9], -1]) == E.KS_ERR_RANGE
        assert code(req_mem=np.r_[rm[:9], (1 << 55) + 1]) == E.KS_ERR_RANGE
        big = np.zeros(65537, np.int64)
        assert code(req_cpu=big, req_mem=big, sel=np.zeros((65537, 1), np.uint64)) == E.KS_ERR_RANGE
        t = 4097
        assert code(alloc_cpu=np.ones(t), alloc_mem=np.ones(t), free_cpu=np.ones(t), free_mem=np.ones(t),
                    labels=np.zeros((t, 1), np.uint64), max_nodes=np.ones(t)) == E.KS_ERR_RANGE
        assert code(labels=np.zeros((3, 3), np.uint64), sel=np.zeros((10, 3), np.uint64)) == E.KS_ERR_INVALID
        # NULL arrays and device-space pods, through the raw entry point
        out = (E.ks_scaleup_option * 3)()
        best = C.c_int32(0)
        pods = E.ks_pods(10, rc.ctypes.data, rm.ctypes.data, sel.ctypes.data, E.KS_MEM_HOST)
        tm = E.ks_node_templates(3, 1, ac.ctypes.data, am.ctypes.data, fc.ctypes.data, fm.ctypes.data, lab.ctypes.data,
                                 None)
        assert ks.lib.ks_scaleup_estimate(snap._h, C.byref(pods), C.byref(tm), C.addressof(out), C.addressof(best), None,
                                          None) == E.KS_ERR_INVALID
        tm.max_nodes = mx.ctypes.data
        assert ks.lib.ks_scaleup_estimate(snap._h, C.byref(pods), C.byref(tm), None, C.addressof(best), None,
                                          None) == E.KS_ERR_INVALID
        assert ks.lib.ks_scaleup_estimate(snap._h, C.byref(pods), C.byref(tm), C.addressof(out), None, None, None) == E.KS_ERR_INVALID
        dpods = E.ks_pods(10, rc.ctypes.data, rm.ctypes.data, sel.ctypes.data, E.KS_MEM_DEVICE)
        assert ks.lib.ks_scaleup_estimate(snap._h, C.byref(dpods), C.byref(tm), C.addressof(out), C.addressof(best), None,
                                          None) == E.KS_ERR_INVALID
        assert ks.lib.ks_scaleup_estimate(snap._h, C.byref(pods), C.byref(tm), C.addressof(out), C.addressof(best), None, None) == E.KS_OK


def test_host_layer_daemonsets_instance_type_and_no_side_effects(ks, orc):
    """ksh_scaleup_estimate over objects equals the restatement on an independent packing of the same specs: DaemonSet
    pods charged to their template, an instance-type selector only a template carries, a pair no template carries.
    The context's store and ksh_select_nodes are the same before and after."""
    tmpl, mx, ds, pods = _host_case()
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        ctx.set_cluster_pods(arena.pods(g["bound_pods"]), len(g["bound_pods"]))
        probe = arena.pods(g["pods"])
        before = ctx.export_packed(), ctx.select_nodes(probe, len(g["pods"]))
        got = ctx.scaleup_estimate(arena.nodes(tmpl), len(tmpl), mx, arena.pods(pods), len(pods), arena.pods(ds), len(ds))
        after = ctx.export_packed(), ctx.select_nodes(probe, len(g["pods"]))
        e = ctx.scaleup_estimate(None, 0, [], arena.pods(pods), len(pods), None, 0)  # no templates: nothing placed
        assert e[1] == -1 and (e[3] == 0).all()
        E = ks.capi
        for bad_t, bad_o, bad_p in (([tmpl[0], tmpl[0]], [], []),
                                    (tmpl, [{"name": "x", "node_name": "nope", "containers": []}], []),
                                    (tmpl, [], [{"name": "b", "node_name": "n1", "containers": []}])):
            with pytest.raises(ks.KsError) as err:
                ctx.scaleup_estimate(arena.nodes(bad_t), len(bad_t), [1] * len(bad_t), arena.pods(bad_p) if bad_p else None,
                                     len(bad_p), arena.pods(bad_o) if bad_o else None, len(bad_o))
            assert err.value.code == E.KS_ERR_INVALID
    for a, b in zip(before[0] + before[1], after[0] + after[1]):
        assert np.array_equal(a, b)
    want = scaleup_packed(orc, *packed_from_specs(tmpl, mx, ds, pods))
    for f in want[0].dtype.names:
        assert np.array_equal(got[0][f], want[0][f]), f
    assert got[1] == want[1] and np.array_equal(got[2], want[2]) and np.array_equal(got[3], want[3])
    itype = np.arange(len(pods)) % 5 == 1
    assert (got[2][1, itype] >= 0).any() and (got[2][[0, 2]][:, itype] == -1).all()  # only group-1 takes them
    assert (got[2][:, np.arange(len(pods)) % 5 == 3] == -1).all()  # disk=ssd: no template
    assert got[1] >= 0 and (got[0]["placed"] < got[0]["eligible"]).any()
