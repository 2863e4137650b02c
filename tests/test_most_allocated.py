"""KS_SCORE_MOST_ALLOCATED (bin-packing), CPU part: the Python-integer definition against the numpy restatement on
random and edge cells; the restatement's select against the oracle's cell codes and its round loop against one pod at a
time; the prefix-fill replica plan against one copy at a time on thousands of random small clusters; the hand-derived
GV-1 values of tests/golden/gv1_most_allocated.json; the policy constant in the header, ctypes and the Rust shim; and
KS_ERR_NO_DEVICE from every object-level call that takes a policy on a packing-only context."""
import os
import re

import numpy as np
import pytest

from helpers import load_golden
from most_allocated_oracle import MOST_ALLOCATED, Oracle, prefix_fill_packed, score, scores, term, topk_packed
from replicas_oracle import sequential_packed
from test_replicas import random_cluster

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIM_C, LIM_M = 1 << 36, 1 << 55


def test_term_definition_by_hand():
    assert term(4000, 4000, 500) == 12 and term(1500, 2000, 500) == 50 and term(5500, 8000, 500) == 37
    assert term(5, 0, 1) == 0 and term(5, -3, 1) == 0  # allocatable <= 0
    assert term(9, 4, 0) == 0  # free above allocatable: requested clamps to 0
    assert term(-7, 4, 3) == 100  # requested above allocatable clamps to it
    assert term(3, 4, 0) == 25 and term(3, 400, 0) == 99 and term(4, 400, 3) == 99 and term(1, 400, 0) == 99


def _edge_values():
    f = [0, 1, -1, 7, LIM_M, -LIM_M, LIM_M - 1, LIM_C, -LIM_C]
    a = [-5, 0, 1, 3, 100, 400, LIM_C, LIM_M]
    q = [0, 1, 3, LIM_C, LIM_M, -1, -LIM_M]
    return f, a, q


def test_numpy_restatement_equals_integers_on_edges_and_random_cells():
    f, a, q = _edge_values()
    cells = [(x, y, z) for x in f for y in a for z in q]
    rng = np.random.default_rng(0xB1A)
    for _ in range(20000):
        A = int(rng.choice([int(rng.integers(1, 1000)), int(rng.integers(-3, 3)), int(rng.integers(1, LIM_M))]))
        cells.append((int(rng.integers(-LIM_M, LIM_M)), A, int(rng.integers(0, LIM_M))))
        cells.append((int(rng.integers(-1000, 1000)), A, int(rng.integers(0, 1000))))
    fv, av, qv = (np.array(c, np.int64) for c in zip(*cells))
    got = scores(fv, fv[::-1], av, av[::-1], qv, qv[::-1])
    want = [score(x, y, aa, bb, r, s) for x, y, aa, bb, r, s in zip(fv, fv[::-1], av, av[::-1], qv, qv[::-1])]
    assert got.tolist() == want
    assert got.min() >= 0 and got.max() <= 100
    for x, y, z in cells[:2000]:  # exact-percentage boundaries: A - (f - q) = k * A / 100
        if y > 0 and y % 100 == 0:
            k = (y - (x - z)) * 100 // y
            assert term(x, y, z) == min(max(k, 0), 100)


def _cluster(rng, N, P, W=1):
    ac = rng.choice([0, 1000, 2000, 4000, 96000], N).astype(np.int64)
    am = rng.choice([0, 1 << 30, 1 << 33, 3 << 32], N).astype(np.int64)
    fc = (ac * rng.integers(-1, 9, N) // 8).astype(np.int64)
    fm = (am * rng.integers(-1, 9, N) // 8).astype(np.int64)
    lab = rng.integers(0, 8, (N, W)).astype(np.uint64)
    rc = rng.choice([0, 250, 500, 1000], P).astype(np.int64)
    rm = rng.choice([0, 1 << 28, 1 << 30], P).astype(np.int64)
    sel = np.where(rng.random((P, W)) < 0.3, rng.integers(1, 4, (P, W)), 0).astype(np.uint64)
    return fc, fm, ac, am, lab, rc, rm, sel


def test_select_restatement_is_the_argmax_of_the_definition(orc):
    o = Oracle(orc)
    rng = np.random.default_rng(0xA3)
    for it in range(60):
        fc, fm, ac, am, lab, rc, rm, sel = _cluster(rng, int(rng.integers(1, 40)), int(rng.integers(1, 30)))
        idx, sc, cnt, mask, codes = o.run_packed(fc, fm, ac, am, lab, rc, rm, sel, MOST_ALLOCATED, want_codes=True)
        lo = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, 0)
        assert np.array_equal(cnt, lo[2]) and np.array_equal(mask, lo[3])  # the mask and counts do not depend on it
        for p in range(len(rc)):
            cand = [(score(fc[n], fm[n], ac[n], am[n], rc[p], rm[p]), -n) for n in range(len(fc)) if codes[p, n] == 0]
            if not cand:
                assert idx[p] == -1 and sc[p] == 0
            else:
                s, n = max(cand)
                assert (idx[p], sc[p]) == (-n, s), (it, p)
        top = topk_packed(o, fc, fm, ac, am, lab, rc, rm, sel, 5)
        assert np.array_equal(top[0][:, 0], idx) and np.array_equal(top[1][:, 0], sc) and np.array_equal(top[2], cnt)


def test_round_loop_restatement_with_singletons_is_one_pod_at_a_time(orc):
    """Pods that never share a round (one pod per call) bind as the sequential restatement binds them."""
    from gang_oracle import sequential_packed as one_at_a_time
    o = Oracle(orc)
    rng = np.random.default_rng(0xA4)
    for _ in range(20):
        fc, fm, ac, am, lab, rc, rm, sel = _cluster(rng, 12, 10)
        f1, m1, f2, m2 = fc.copy(), fm.copy(), fc.copy(), fm.copy()
        got = [o.stream_bind_packed(f1, m1, ac, am, lab, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], MOST_ALLOCATED)[:2]
               for p in range(len(rc))]
        want = one_at_a_time(o, f2, m2, ac, am, lab, rc, rm, sel, MOST_ALLOCATED)
        assert [int(i[0]) for i, _ in got] == want[0].tolist() and [int(s[0]) for _, s in got] == want[1].tolist()
        assert np.array_equal(f1, f2) and np.array_equal(m1, m2)


def test_prefix_fill_equals_one_copy_at_a_time(orc):
    o = Oracle(orc)
    rng = np.random.default_rng(0x5EED3)
    cases = 0
    for it in range(2500):
        fc, fm, ac, am, labels, rc, rm, sel, R = random_cluster(rng)
        got = prefix_fill_packed(fc, fm, ac, am, labels, rc, rm, sel, R)
        want = sequential_packed(o, fc, fm, ac, am, labels, rc, rm, sel, R, MOST_ALLOCATED)
        for a, b in zip(got, want):
            assert np.array_equal(a, b), (it, got, want)
        cases += len(rc)
    assert cases > 5000


def _gv1(ks, orc):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        ctx.set_cluster_pods(arena.pods(g["bound_pods"]), len(g["bound_pods"]))
        ac, am, lab, bn, bc, bm = ctx.export_packed()
        rc, rm, sel = ctx.pack_pods(arena.pods(g["pods"]), len(g["pods"]))
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    assert fc.tolist() == g["expected_free_cpu_milli"] and fm.tolist() == g["expected_free_mem_bytes"]
    return g, [p["name"] for p in g["pods"]], (fc, fm, ac, am, lab), rc, rm, sel


def test_gv1_golden(ks, orc):
    o = Oracle(orc)
    want = load_golden("gv1_most_allocated.json")
    g, names, cl, rc, rm, sel = _gv1(ks, orc)
    fc, fm, ac, am, lab = cl
    for pod, w in want["select"].items():
        p = names.index(pod)
        idx, sc = o.run_packed(*cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], MOST_ALLOCATED, want_mask=False)[:2]
        assert (int(idx[0]), int(sc[0])) == (w["node"], w["score"])
        for n, s in enumerate(w["scores"]):
            if s is not None:
                assert score(fc[n], fm[n], ac[n], am[n], rc[p], rm[p]) == s
    p = names.index("p1")
    oth = want["other_policies_p1"]
    assert orc.run_packed(*cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], 0, want_mask=False)[0][0] == oth["leftover"]
    la = orc.run_packed(*cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], 1, want_mask=False)[0][0]
    assert la == oth["least_allocated"]
    k = want["topk"]["k"]
    for pod in ("p0", "p1"):
        p = names.index(pod)
        top = topk_packed(o, *cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], k)
        assert top[0][0].tolist() == want["topk"][pod]["node"] and top[1][0].tolist() == want["topk"][pod]["score"]
    w = want["replicas"]
    p = names.index(w["spec"])
    R = np.array([w["replicas"]], np.uint32)
    rows, node, sc, _ = prefix_fill_packed(*cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], R)
    seq = sequential_packed(o, *cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], R, MOST_ALLOCATED)
    assert all(np.array_equal(a, b) for a, b in zip((rows, node, sc), seq))
    assert {f: int(rows[f][0]) for f in w["row"]} == w["row"]
    assert node.tolist() == w["node"] and sc.tolist() == w["score"]


def test_policy_constant_mirrors(ks):
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    assert int(re.search(r"#define KS_SCORE_MOST_ALLOCATED (\d+)", hdr).group(1)) == 3
    assert ks.KS_SCORE_MOST_ALLOCATED == ks.capi.KS_SCORE_MOST_ALLOCATED == 3
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    assert re.search(r"pub const KS_SCORE_MOST_ALLOCATED: c_int = 3;", rs)
    assert not re.search(r"#define KS_SCORE_\w+ 2\b", hdr)  # 2 stays reserved
    assert not hasattr(ks.capi, "KS_SCORE_2")


def test_packing_only_context_is_no_device_under_policy_3(ks):
    """Every object-level call that takes a policy passes 3 through and, without a snapshot, is KS_ERR_NO_DEVICE."""
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    pods = arena.pods(g["pods"][:3])
    on_n2 = arena.pods(g["bound_pods"][1:3])  # b2a and b2b, bound to n2
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        calls = [
            lambda: ctx.select_nodes(pods, 3, policy=3),
            lambda: ctx.rank_nodes(pods, 3, 4, policy=3),
            lambda: ctx.reconcile_batch(pods, 3, policy=3),
            lambda: ctx.reconcile_gangs(pods, 3, [0, 2, 3], [1, 1], policy=3),
            lambda: ctx.drain_nodes(["n2"], on_n2, [0, 2], policy=3),
            lambda: ctx.place_replicas(pods, 3, [3, 1, 2], policy=3),
        ]
        for i, call in enumerate(calls):
            with pytest.raises(ks.KsError) as e:
                call()
            assert e.value.code == ks.capi.KS_ERR_NO_DEVICE, i
