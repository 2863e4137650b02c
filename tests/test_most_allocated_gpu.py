"""KS_SCORE_MOST_ALLOCATED (bin-packing) on the GPU: the tests of tests/policy_suite_gpu.py under policy 3, and the
refusal of the reserved policy 2."""
import pytest

from policy_oracle import MOST_ALLOCATED
from policy_suite_gpu import *  # noqa: F401,F403 - the shared tests, run under the policy fixture below
from policy_suite_gpu import assert_refused


@pytest.fixture(scope="module")
def policy():
    return MOST_ALLOCATED


def test_policy_2_is_refused(ks):
    assert_refused(ks, 2)
