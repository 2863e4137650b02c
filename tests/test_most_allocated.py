"""KS_SCORE_MOST_ALLOCATED (bin-packing), CPU part: the Python-integer definition against the numpy restatement on
random and edge cells; the early-exit bound of the bit-parallel walk on a million pairs per family; the prefix-fill
replica plan against one copy at a time on thousands of random small clusters; and, under policy 3, the tests of
tests/policy_suite.py (select, round loop, GV-1, constant mirrors, packing-only context, walk model)."""
import numpy as np
import pytest

from policy_oracle import I64_MAX, MOST_ALLOCATED, Oracle, most_bound, most_slack, prefix_fill_packed, term
from policy_oracle import most_score as score
from policy_oracle import most_scores as scores
from policy_suite import *  # noqa: F401,F403 - the shared tests, run under the policy fixture below
from policy_suite import check_packing_only_context
from replicas_oracle import sequential_packed
from test_replicas import random_cluster

LIM_C, LIM_M = 1 << 36, 1 << 55


@pytest.fixture(scope="module")
def policy():
    return MOST_ALLOCATED


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


@pytest.mark.parametrize("family", ["random", "adversarial", "exact percentages"])
def test_walk_bound_holds_on_a_million_pairs(family):
    """score(p, n) <= (b(n) + D(p)) // 2 on every feasible cell with requests >= 0 (k_most_alloc's early exit), and
    with no request the bound is the score itself - which is what lets a tie sit exactly at the exit."""
    rng = np.random.default_rng({"random": 0xB3, "adversarial": 0xB4, "exact percentages": 0xB5}[family])
    N, P = 1000, 1000
    if family == "random":
        ac = rng.choice([1000, 4000, 16000, 96000], N).astype(np.int64)
        am = rng.choice([1, 4, 64, 384], N).astype(np.int64) << 30
        fc, fm = ac * rng.integers(0, 17, N) // 16, am * rng.integers(0, 17, N) // 16
        rc = rng.choice([0, 1, 100, 500, 4000], P).astype(np.int64)
        rm = rng.choice([0, 1, 1 << 27, 1 << 32], P).astype(np.int64)
    elif family == "adversarial":  # tiny and huge allocatables, allocatable <= 0, free above allocatable, limits
        ac = rng.choice([1, 2, 50, 4000, LIM_C], N).astype(np.int64)
        am = rng.choice([1, 3, 50 << 20, 1 << 53, LIM_M], N).astype(np.int64)
        ac[rng.random(N) < 0.05] = 0
        am[rng.random(N) < 0.05] = -7
        fc = ac // 50 * rng.integers(0, 51, N) + ac % 50
        fm = am // 50 * rng.integers(0, 51, N) + am % 50
        over = rng.random(N) < 0.05
        fc[over] += 1000
        fm[over] += 1 << 40
        rc = rng.choice([0, 1, 2, 25, 1 << 20, LIM_C], P).astype(np.int64)
        rm = rng.choice([0, 1, 7, 1 << 40, LIM_M], P).astype(np.int64)
    else:  # A - (f - q) = k * A / 100 on every cell: each A / 100 divides 960 (512 MiB) and the requests are multiples
        unit_c = rng.choice([48, 96, 320, 960], N).astype(np.int64)
        unit_m = rng.choice([64, 128, 256, 512], N).astype(np.int64) << 20
        ac, am = 100 * unit_c, 100 * unit_m
        fc, fm = ac - unit_c * rng.integers(0, 101, N), am - unit_m * rng.integers(0, 101, N)
        rc = 960 * rng.integers(0, 6, P).astype(np.int64)
        rm = (512 << 20) * rng.integers(0, 13, P).astype(np.int64)
        u = ac[None, :] - (fc[None, :] - rc[:, None])
        assert (u % unit_c[None, :] == 0).all()
    b = np.array([most_bound(*v) for v in zip(fc, fm, ac, am)], np.int64)
    assert b.min() >= 0 and b.max() <= 200
    amin_c = int(ac[ac > 0].min()) if (ac > 0).any() else I64_MAX
    amin_m = int(am[am > 0].min()) if (am > 0).any() else I64_MAX
    D = np.array([most_slack(int(x), int(y), amin_c, amin_m) for x, y in zip(rc, rm)], np.int64)
    s = scores(fc[None, :], fm[None, :], ac[None, :], am[None, :], rc[:, None], rm[:, None])
    feas = (rc[:, None] <= fc[None, :]) & (rm[:, None] <= fm[None, :])
    lim = (b[None, :] + D[:, None]) // 2
    assert feas.sum() > 100000
    assert (s[feas] <= lim[feas]).all()
    zero = (rc == 0) & (rm == 0)
    assert zero.any() and (s[zero][feas[zero]] == lim[zero][feas[zero]]).all()  # attained without a request
    assert np.median((lim - s)[feas]) <= 60  # and not vacuous with one
    if family == "exact percentages":
        assert ((lim - s)[feas] == 0).mean() > 0.05  # the limit is reached with requests too


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


def test_packing_only_context_is_no_device_under_policy_3(ks, policy):
    """Every object-level call that takes a policy passes 3 through and, without a snapshot, is KS_ERR_NO_DEVICE."""
    check_packing_only_context(ks, policy)
