"""The CPU tests of KS_SCORE_MOST_ALLOCATED (3) and KS_SCORE_LEAST_BALANCED (4) that hold for both policies, written
once against the restatement of tests/policy_oracle.py: the restatement's select against the oracle's cell codes and
its round loop against one pod at a time; the hand-derived GV-1 values of tests/golden/gv1_*.json; the policy constant
in the header, ctypes and the Rust shim; KS_ERR_NO_DEVICE from every object-level call that takes a policy on a
packing-only context; and the model of the bit-parallel walk (walk_packed) against the oracle on random clusters, on
clusters that sit exactly at its exits and at its length extremes.  tests/test_most_allocated.py and
tests/test_least_balanced.py collect these tests under their policy (a `policy` fixture) next to the tests of their own
definition."""
import os
import re

import numpy as np
import pytest

from helpers import load_golden
from policy_oracle import (EDGES, FIRST_WINDOW, LB_UNBOUNDED, LEAST_BALANCED, MOST_ALLOCATED, PLAN, SCORE, TILE,
                           WINDOW, Oracle, balanced, exit_tie_cluster, least, most_score, stored_bound, topk_packed,
                           walk_extreme_clusters, walk_packed)
from replicas_oracle import sequential_packed

__all__ = ["check_packing_only_context"]  # + every test_ function, below
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = {MOST_ALLOCATED: "KS_SCORE_MOST_ALLOCATED", LEAST_BALANCED: "KS_SCORE_LEAST_BALANCED"}


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


def test_select_restatement_is_the_argmax_of_the_definition(orc, policy):
    o = Oracle(orc)
    rng = np.random.default_rng({MOST_ALLOCATED: 0xA3, LEAST_BALANCED: 0xA5}[policy])
    for it in range(60):
        fc, fm, ac, am, lab, rc, rm, sel = _cluster(rng, int(rng.integers(1, 40)), int(rng.integers(1, 30)))
        idx, sc, cnt, mask, codes = o.run_packed(fc, fm, ac, am, lab, rc, rm, sel, policy, want_codes=True)
        lo = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, 0)
        assert np.array_equal(cnt, lo[2]) and np.array_equal(mask, lo[3])  # the mask and counts do not depend on it
        for p in range(len(rc)):
            cand = [(SCORE[policy](fc[n], fm[n], ac[n], am[n], rc[p], rm[p]), -n) for n in range(len(fc)) if codes[p, n] == 0]
            if not cand:
                assert idx[p] == -1 and sc[p] == 0
            else:
                s, n = max(cand)
                assert (idx[p], sc[p]) == (-n, s), (it, p)
        top = topk_packed(o, fc, fm, ac, am, lab, rc, rm, sel, 5, policy)
        assert np.array_equal(top[0][:, 0], idx) and np.array_equal(top[1][:, 0], sc) and np.array_equal(top[2], cnt)


def test_round_loop_restatement_with_singletons_is_one_pod_at_a_time(orc, policy):
    """Pods that never share a round (one pod per call) bind as the sequential restatement binds them."""
    from gang_oracle import sequential_packed as one_at_a_time
    o = Oracle(orc)
    rng = np.random.default_rng(0xA4)
    for _ in range(20):
        fc, fm, ac, am, lab, rc, rm, sel = _cluster(rng, 12, 10)
        f1, m1, f2, m2 = fc.copy(), fm.copy(), fc.copy(), fm.copy()
        got = [o.stream_bind_packed(f1, m1, ac, am, lab, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], policy)[:2]
               for p in range(len(rc))]
        want = one_at_a_time(o, f2, m2, ac, am, lab, rc, rm, sel, policy)
        assert [int(i[0]) for i, _ in got] == want[0].tolist() and [int(s[0]) for _, s in got] == want[1].tolist()
        assert np.array_equal(f1, f2) and np.array_equal(m1, m2)


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
    return [p["name"] for p in g["pods"]], (fc, fm, ac, am, lab), rc, rm, sel


def test_gv1_golden(ks, orc, policy):
    o = Oracle(orc)
    want = load_golden({MOST_ALLOCATED: "gv1_most_allocated.json", LEAST_BALANCED: "gv1_least_balanced.json"}[policy])
    names, cl, rc, rm, sel = _gv1(ks, orc)
    fc, fm, ac, am, lab = cl
    for pod, w in want["select"].items():
        p = names.index(pod)
        idx, sc = o.run_packed(*cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], policy, want_mask=False)[:2]
        assert (int(idx[0]), int(sc[0])) == (w["node"], w["score"])
        c = lambda n: (fc[n], fm[n], ac[n], am[n], rc[p], rm[p])  # noqa: E731
        if policy == MOST_ALLOCATED:
            for n, s in enumerate(w["scores"]):
                if s is not None:
                    assert most_score(*c(n)) == s
        else:
            for n, (l, b) in enumerate(zip(w["least"], w["balanced"])):
                if l is not None:
                    assert least(*c(n)) == l and balanced(*c(n)) == b
    if policy == MOST_ALLOCATED:
        p = names.index("p1")
        oth = want["other_policies_p1"]
        assert orc.run_packed(*cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], 0, want_mask=False)[0][0] == oth["leftover"]
        la = orc.run_packed(*cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], 1, want_mask=False)[0][0]
        assert la == oth["least_allocated"]
    k = want["topk"]["k"]
    for pod in ("p0", "p1"):
        p = names.index(pod)
        top = topk_packed(o, *cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], k, policy)
        assert top[0][0].tolist() == want["topk"][pod]["node"] and top[1][0].tolist() == want["topk"][pod]["score"]
    w = want["replicas"]
    p = names.index(w["spec"])
    R = np.array([w["replicas"]], np.uint32)
    rows, node, sc, _ = PLAN[policy](*cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], R)
    seq = sequential_packed(o, *cl, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], R, policy)
    assert all(np.array_equal(a, b) for a, b in zip((rows, node, sc), seq))
    assert {f: int(rows[f][0]) for f in w["row"]} == w["row"]
    assert node.tolist() == w["node"] and sc.tolist() == w["score"]


def _walk_clusters(rng):
    """(name, cluster): random clusters from one to many windows, and test_least_alloc_float_model's value families
    (negative requests, allocatables <= 0 and free above allocatable among them)."""
    from test_least_alloc_float_model import _families
    for N, P in ((37, 30), (1500, 60), (3000, 40), (12000, 25)):
        yield f"random {N}", _cluster(rng, N, P, W=2)
    for name, fc, fm, ac, am, rc, rm in _families(rng, 2600, 40):
        fc, fm, ac, am = (np.asarray(a, np.int64) for a in (fc, fm, ac, am))
        lab = rng.integers(0, 4, (len(fc), 1)).astype(np.uint64)
        sel = np.where(rng.random((len(rc), 1)) < 0.3, 1, 0).astype(np.uint64)
        yield name, (fc, fm, ac, am, lab, np.asarray(rc, np.int64), np.asarray(rm, np.int64), sel)


def test_walk_model_equals_the_oracle(orc, policy):
    """walk_packed, the restatement of the bit-parallel walk, returns the argmax of the definition on every pod, and
    these clusters reach its early exit and its later windows."""
    o = Oracle(orc)
    rng = np.random.default_rng({MOST_ALLOCATED: 0xE3, LEAST_BALANCED: 0xE4}[policy])
    exits = windows = 0
    for name, cl in _walk_clusters(rng):
        idx, sc, scored, ex = walk_packed(o, *cl, policy)
        w = o.run_packed(*cl, policy, want_mask=False)
        assert np.array_equal(idx, w[0]) and np.array_equal(sc, w[1]), name
        exits += int((ex > 0).sum())
        windows += sum(bool(s) and s[-1] >= FIRST_WINDOW for s in scored)
    assert exits > 50 and windows > 10


@pytest.mark.parametrize("edge", list(EDGES))
def test_exit_edge_clusters_reach_their_boundary(orc, policy, edge):
    """exit_tie_cluster puts X and Y on each side of the boundary.  Tie: the walk does not stop in front of Y's tile,
    scores it, and Y - later in bound order, lower in index - wins.  Mirror: the walk stops exactly in front of Y's tile
    and X wins.  An exit one step too early (margin -1) stops in front of Y's tile in the tie case too and loses Y: the
    case catches that off-by-one wherever an exit test lies between X and Y."""
    o = Oracle(orc)
    tx, ty = EDGES[edge][:2]
    for mirror in (False, True):
        cl, x, y = exit_tie_cluster(policy, edge, mirror, seed=ty)
        assert y < x
        idx, sc, scored, ex = walk_packed(o, *cl, policy)
        w = o.run_packed(*cl, policy, want_mask=False)
        assert np.array_equal(idx, w[0]) and np.array_equal(sc, w[1]), (edge, mirror)
        assert (w[0] == (x if mirror else y)).all(), (edge, mirror)
        assert all(s[0] == tx for s in scored)  # nothing in front of X is feasible
        if tx == ty:  # no exit test between them: the tie is the tile merge's
            assert all(ty in s for s in scored) and (ex != ty).all()
        elif mirror:
            assert (ex == ty).all() and all(ty not in s for s in scored), edge
        else:
            assert all(ty in s for s in scored) and ((ex == -1) | (ex > ty)).all(), edge
        early = walk_packed(o, *cl, policy, margin=-1)
        if mirror or tx == ty:
            assert np.array_equal(early[0], w[0]), (edge, mirror)
        else:
            assert (early[3] == ty).all() and (early[0] == x).all() and (early[1] == w[1]).all(), edge


def test_walk_extreme_clusters_reach_their_extremes(orc, policy):
    """The clusters of walk_extreme_clusters do what they are named for, by the walk model, which equals the oracle on
    them: the selector pods of "last tiles only" score nothing before the last window; no walk stops while a node stored
    at 2^62 is left; a saturated D leaves MOST_ALLOCATED no exit for a pod that requests something; equal allocatables
    let most pods stop early."""
    o = Oracle(orc)
    for name, cl in walk_extreme_clusters(policy, seed=policy):
        fc, fm, ac, am, lab, rc, rm, sel = cl
        idx, sc, scored, ex = walk_packed(o, *cl, policy)
        w = o.run_packed(*cl, policy, want_mask=False)
        assert np.array_equal(idx, w[0]) and np.array_equal(sc, w[1]), name
        if name == "last tiles only":
            walked = [s for s, q in zip(scored, sel[:, 0]) if q == 1 << 9 and s]
            assert len(walked) > 40 and all(s[0] >= FIRST_WINDOW + 2 * WINDOW for s in walked)
        elif name == "free above alloc":
            unbounded = sum(stored_bound(policy, *v) == LB_UNBOUNDED for v in zip(fc, fm, ac, am))
            assert 2000 < unbounded < 4000 if policy == LEAST_BALANCED else unbounded == 0
            assert (ex[ex >= 0] * TILE >= unbounded).all() and (ex > 0).any()
        elif name == "one alloc of 1" and policy == MOST_ALLOCATED:  # D = 200 once both requests are positive
            assert (ex[(rc > 0) & (rm > 0)] == -1).all() and (ex[(rc == 0) & (rm == 0)] > 0).any()
        elif name == "equal allocatables":
            assert (ex > 0).mean() > 0.5


def test_policy_constant_mirrors(ks, policy):
    name = NAME[policy]
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    assert int(re.search(rf"#define {name} (\d+)", hdr).group(1)) == policy
    assert getattr(ks, name) == getattr(ks.capi, name) == policy
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    assert re.search(rf"pub const {name}: c_int = {policy};", rs)
    assert name in open(os.path.join(ROOT, "examples", "rust_shim", "ksched.rs")).read()
    assert not re.search(r"#define KS_SCORE_\w+ (2|5)\b", hdr)  # 2 stays reserved, nothing above 4
    assert not hasattr(ks.capi, "KS_SCORE_2")


def check_packing_only_context(ks, policy):
    """Every object-level call that takes a policy passes it through and, without a snapshot, is KS_ERR_NO_DEVICE."""
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    pods = arena.pods(g["pods"][:3])
    on_n2 = arena.pods(g["bound_pods"][1:3])  # b2a and b2b, bound to n2
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        calls = [
            lambda: ctx.select_nodes(pods, 3, policy=policy),
            lambda: ctx.rank_nodes(pods, 3, 4, policy=policy),
            lambda: ctx.reconcile_batch(pods, 3, policy=policy),
            lambda: ctx.reconcile_gangs(pods, 3, [0, 2, 3], [1, 1], policy=policy),
            lambda: ctx.drain_nodes(["n2"], on_n2, [0, 2], policy=policy),
            lambda: ctx.place_replicas(pods, 3, [3, 1, 2], policy=policy),
        ]
        for i, call in enumerate(calls):
            with pytest.raises(ks.KsError) as e:
                call()
            assert e.value.code == ks.capi.KS_ERR_NO_DEVICE, i


__all__ += [n for n in dir() if n.startswith("test_")]
