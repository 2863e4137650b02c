"""KS_SCORE_MOST_ALLOCATED (bin-packing), CPU part: the Python-integer definition against the numpy restatement on
random and edge cells; the prefix-fill replica plan against one copy at a time on thousands of random small clusters;
and, under policy 3, the tests of tests/policy_suite.py (select, round loop, GV-1, constant mirrors, packing-only
context)."""
import numpy as np
import pytest

from policy_oracle import MOST_ALLOCATED, Oracle, prefix_fill_packed, term
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
