"""KS_SCORE_LEAST_BALANCED (upstream's default resource scoring) on the GPU: the tests of tests/policy_suite_gpu.py under
policy 4, the refusal of policies 2 and 5, and the float-hazard cells, where (1 - std) * 100 lies within a few ulps of
an integer."""
import numpy as np
import pytest

from policy_oracle import LEAST_BALANCED, hazard_cells, topk_packed
from policy_suite_gpu import *  # noqa: F401,F403 - the shared tests, run under the policy fixture below
from policy_suite_gpu import assert_refused, snapshot


@pytest.fixture(scope="module")
def policy():
    return LEAST_BALANCED


@pytest.mark.parametrize("bad", [2, 5])
def test_policies_2_and_5_are_refused(ks, bad):
    assert_refused(ks, bad)


@pytest.mark.parametrize("N", [1, 255, 256, 257, 5000])
def test_float_hazard_cells_on_both_paths(ks, o, N):
    """Cells where (1 - std) * 100 lies within a few ulps of an integer (half of them change under an FMA or a reciprocal):
    every node carries one such cell for a pod that requests nothing, so each pod's argmax and score depend on them."""
    (hc, hm, hac, ham, _, _), _ = hazard_cells(0x600 + N, 2 * N)
    fc, fm, ac, am = hc[:N], hm[:N], hac[:N], ham[:N]
    lab = np.zeros((N, 1), np.uint64)
    P = 64
    rng = np.random.default_rng(N)
    rc = np.where(np.arange(P) < 8, 0, rng.integers(0, 200, P)).astype(np.int64)
    rm = np.zeros(P, np.int64)
    sel = np.zeros((P, 1), np.uint64)
    want = o.run_packed(fc, fm, ac, am, lab, rc, rm, sel, LEAST_BALANCED, want_mask=False)
    with snapshot(ks, fc, fm, ac, am, lab) as s:
        for flags in (ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR):
            r = s.select(rc, rm, sel, policy=LEAST_BALANCED, flags=flags)
            assert np.array_equal(r.node_idx, want[0]) and np.array_equal(r.score, want[1]), flags
        k = min(N, 32)
        top = s.select_topk(rc[:8], rm[:8], sel[:8], k, LEAST_BALANCED)
        wt = topk_packed(o, fc, fm, ac, am, lab, rc[:8], rm[:8], sel[:8], k, LEAST_BALANCED)
        assert all(np.array_equal(a, b) for a, b in zip(top, wt))
