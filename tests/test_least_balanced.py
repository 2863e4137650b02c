"""KS_SCORE_LEAST_BALANCED (upstream's default resource scoring), CPU part: the numpy restatement against the Python
definition on random and edge cells, near 2^53-2^55 and on cells where (1 - std) * 100 lies within a few ulps of an
integer; the early-exit bound of the bit-parallel walk on a million (pod, node) pairs; the one-copy-at-a-time replica
heap against one full select per copy; and, under policy 4, the tests of tests/policy_suite.py (select, round loop,
GV-1, constant mirrors, packing-only context; policies 2 and 5 are refused on the GPU, test_least_balanced_gpu)."""
from fractions import Fraction

import numpy as np
import pytest

from policy_oracle import (LEAST_BALANCED, Oracle, _chain, balanced, hazard_cells, heap_packed, least, node_bound,
                           pod_slack)
from policy_oracle import balanced_score as score
from policy_oracle import balanced_scores as scores
from policy_suite import *  # noqa: F401,F403 - the shared tests, run under the policy fixture below
from policy_suite import check_packing_only_context
from replicas_oracle import sequential_packed
from test_replicas import random_cluster

LIM_C, LIM_M = 1 << 36, 1 << 55
LB = LEAST_BALANCED
I64_MAX = (1 << 63) - 1


@pytest.fixture(scope="module")
def policy():
    return LEAST_BALANCED


def test_definition_by_hand():
    # equal shares: std 0, balanced 100
    assert balanced(4000, 8, 4000, 8, 500, 1) == 100 and score(4000, 8, 4000, 8, 500, 1) == 87 + 100
    # shares 0.375 and 0.34375: std 0.015625, (1 - std) * 100 = 98.4375
    assert balanced(5500, 23, 8000, 32, 500, 2) == 98
    assert balanced(0, 0, 1000, 1 << 30, 0, 0) == 100  # both full
    assert balanced(1000, 0, 1000, 1 << 30, 0, 0) == 50  # shares 0 and 1: the lowest value
    assert balanced(5, 7, 0, 9, 1, 1) == 100 and balanced(5, 7, 9, -3, 1, 1) == 100  # a skipped resource
    assert balanced(9, 9, 4, 4, 0, 0) == 100  # free above allocatable: u clamps to 0 on both
    assert balanced(-7, 4, 4, 4, 3, 0) == 50  # u above allocatable clamps to it: shares 1 and 0


def test_python_int_division_is_not_the_definition():
    """float(u) / float(A) (the definition) and u / A (one rounding of the exact quotient) differ above 2^53."""
    rng = np.random.default_rng(0x53)
    pairs = [(int(rng.integers(1 << 53, LIM_M)), int(rng.integers(1 << 53, LIM_M))) for _ in range(2000)]
    differ = [(u, a) for u, a in pairs if u <= a and float(u) / float(a) != u / a]
    assert len(differ) > 10
    assert all(balanced(a - u, a - u, a, a, 0, 0) == 100 for u, a in differ)  # equal shares stay equal either way


def _edge_values():
    f = [0, 1, -1, 7, LIM_M, -LIM_M, LIM_M - 1, LIM_C, -LIM_C, (1 << 53) + 1, (1 << 54) + 3]
    a = [-5, 0, 1, 3, 100, 400, LIM_C, LIM_M, (1 << 53) + 1, (1 << 55) - 1, (1 << 54) + 7]
    q = [0, 1, 3, LIM_C, LIM_M, -1, -LIM_M, (1 << 53) - 1]
    return f, a, q


def test_numpy_restatement_equals_python_on_edges_and_random_cells():
    f, a, q = _edge_values()
    cells = [(x, y, z) for x in f for y in a for z in q]
    rng = np.random.default_rng(0xB4A)
    for _ in range(20000):
        A = int(rng.choice([int(rng.integers(1, 1000)), int(rng.integers(-3, 3)), int(rng.integers(1, LIM_M)),
                            int(rng.integers(1 << 53, LIM_M))]))
        cells.append((int(rng.integers(-LIM_M, LIM_M)), A, int(rng.integers(0, LIM_M))))
        cells.append((int(rng.integers(-1000, 1000)), A, int(rng.integers(0, 1000))))
        cells.append((A - int(rng.integers(0, max(A, 1))), A, int(rng.integers(0, 1 << 20))))  # u inside [0, A]
    fv, av, qv = (np.array(c, np.int64) for c in zip(*cells))
    args = (fv, fv[::-1], av, av[::-1], qv, qv[::-1])
    got = scores(*args)
    want = [score(*c) for c in zip(*args)]
    assert got.tolist() == want
    bal = [balanced(*c) for c in zip(*args)]
    assert min(bal) >= 50 and max(bal) <= 100
    # u < 0 and u > A both occur, and both resources skipped, one skipped and both kept
    u = av - (fv - qv)
    assert (u < 0).any() and (u > av).any()
    assert ((av <= 0) & (av[::-1] <= 0)).any() and ((av > 0) ^ (av[::-1] > 0)).any()


def test_float_hazard_family_against_exact_rationals():
    """Cells whose exact (1 - std) * 100 is an integer: the double evaluation lands a few ulps either side of it, so an
    FMA or a reciprocal would change the truncated result on half of them.  The restatements agree with the one-op-at-
    a-time chain on all of them, and the chain is within 2^-43 of the exact value."""
    (fc, fm, ac, am, rc, rm), n_hit = hazard_cells(0x4A2, 2000)
    assert n_hit == 1000
    got = scores(fc, fm, ac, am, rc, rm)
    lst = np.array([least(*c) for c in zip(fc, fm, ac, am, rc, rm)])
    assert (got - lst).tolist() == [balanced(*c) for c in zip(fc, fm, ac, am, rc, rm)]
    below = 0
    for c in zip(fc.tolist(), fm.tolist(), ac.tolist(), am.tolist(), rc.tolist(), rm.tolist()):
        f1, f2, a1, a2, q1, q2 = c
        uc, um = a1 - (f1 - q1), a2 - (f2 - q2)
        exact = (1 - abs(Fraction(uc, a1) - Fraction(um, a2)) / 2) * 100
        assert exact.denominator == 1  # an integer by construction
        b = balanced(*c)
        assert b == _chain(uc, a1, um, a2) and b in (exact, exact - 1)
        below += b == exact - 1
        # the double value before truncation, recomputed exactly from the rounded operands
        xc, xm = float(uc) / float(a1), float(um) / float(a2)
        v = (1.0 - abs(xc - xm) / 2.0) * 100.0
        assert abs(Fraction(v) - exact) < Fraction(1, 1 << 43)
    assert below > 100  # the family does reach below the exact integer


def _bounds_np(fc, fm, ac, am):
    """node_bound on arrays."""
    def most(f, a):
        pos = a > 0
        u = np.clip(a - f, 0, np.maximum(a, 0))
        return np.where(pos, u * 100 // np.where(pos, a, 1), 0)
    lst = np.array([least(x, y, a, b, 0, 0) for x, y, a, b in zip(fc, fm, ac, am)])
    d = np.abs(most(fc, ac) - most(fm, am))
    bal = np.where((ac > 0) & (am > 0), 100 - np.maximum(d - 1, 0) // 2, 100)
    return lst + bal


def _stored(b):
    """The bound the walk stores: LB_UNBOUNDED above 200, 0 below 0."""
    return np.where(b > 200, 1 << 62, np.maximum(b, 0))


@pytest.mark.parametrize("family", ["random", "adversarial"])
def test_walk_bound_holds_on_a_million_pairs(family):
    """score(p, n) <= b(n) - (D(p) - E(p)) on every feasible cell with requests >= 0, rounding included."""
    rng = np.random.default_rng(0xB0 + (family == "adversarial"))
    N, P = 1000, 1000
    if family == "random":
        ac = rng.choice([1000, 4000, 16000, 96000], N).astype(np.int64)
        am = rng.choice([1, 4, 64, 384], N).astype(np.int64) << 30
        fc, fm = ac * rng.integers(0, 17, N) // 16, am * rng.integers(0, 17, N) // 16
        rc = rng.choice([0, 1, 100, 500, 4000], P).astype(np.int64)
        rm = rng.choice([0, 1, 1 << 27, 1 << 32], P).astype(np.int64)
    else:  # tiny and huge allocatables, free above allocatable, a skipped resource, hazard-like exact shares
        ac = rng.choice([1, 2, 50, 4000, LIM_C], N).astype(np.int64)
        am = rng.choice([1, 3, 50 << 20, 1 << 53, LIM_M], N).astype(np.int64)
        ac[rng.random(N) < 0.05] = 0
        am[rng.random(N) < 0.05] = -7
        fc = ac // 50 * rng.integers(0, 51, N) + ac % 50  # no product leaves int64
        fm = am // 50 * rng.integers(0, 51, N) + am % 50
        over = rng.random(N) < 0.05
        fc[over] += 1000
        fm[over] += 1 << 40
        rc = rng.choice([0, 1, 2, 25, 1 << 20, LIM_C], P).astype(np.int64)
        rm = rng.choice([0, 1, 7, 1 << 40, LIM_M], P).astype(np.int64)
    b = _bounds_np(fc, fm, ac, am)
    for n in range(0, N, 97):
        assert b[n] == node_bound(fc[n], fm[n], ac[n], am[n])
    stored = _stored(b)
    amax_c = I64_MAX if (ac <= 0).any() else int(ac.max())
    amax_m = I64_MAX if (am <= 0).any() else int(am.max())
    amin_c = int(ac[ac > 0].min()) if (ac > 0).any() else I64_MAX
    amin_m = int(am[am > 0].min()) if (am > 0).any() else I64_MAX
    S = np.array([pod_slack(int(x), int(y), amax_c, amax_m, amin_c, amin_m) for x, y in zip(rc, rm)], np.int64)
    s = scores(fc[None, :], fm[None, :], ac[None, :], am[None, :], rc[:, None], rm[:, None])
    feas = (rc[:, None] <= fc[None, :]) & (rm[:, None] <= fm[None, :])
    lim = stored[None, :] - S[:, None]
    assert feas.sum() > 100000
    assert (s[feas] <= lim[feas]).all()
    # the bound is not vacuous: most feasible cells are within 60 of it
    assert np.median((lim - s)[feas & (stored[None, :] <= 200)]) <= 60


def test_copy_scores_are_not_monotone():
    """Why ks_place_replicas places these copies one at a time: s_n(j) rises and falls with j."""
    ac, am, fc, fm, rc, rm = 8000, 16 << 30, 8000, 4 << 30, 1000, 0
    s = [score(fc - j * rc, fm - j * rm, ac, am, rc, rm) for j in range(8)]
    assert any(a < b for a, b in zip(s, s[1:])) and any(a > b for a, b in zip(s, s[1:]))


def test_heap_plan_equals_one_copy_at_a_time(orc):
    o = Oracle(orc)
    rng = np.random.default_rng(0x5EED4)
    cases = 0
    for it in range(600):
        fc, fm, ac, am, labels, rc, rm, sel, R = random_cluster(rng)
        got = heap_packed(fc, fm, ac, am, labels, rc, rm, sel, R)
        want = sequential_packed(o, fc, fm, ac, am, labels, rc, rm, sel, R, LB)
        for a, b in zip(got, want):
            assert np.array_equal(a, b), (it, got, want)
        cases += len(rc)
    assert cases > 1000


def test_packing_only_context_is_no_device_under_policy_4(ks, policy):
    """Every object-level call that takes a policy passes 4 through and, without a snapshot, is KS_ERR_NO_DEVICE."""
    check_packing_only_context(ks, policy)
