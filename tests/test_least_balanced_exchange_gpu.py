"""KS_SCORE_LEAST_BALANCED with the fused all-gather of the bindings (ks_exchange): two ranks on the bit-parallel path,
where k_least_balanced stores every binding into both ranks' gather buffers.  Every rank must end with every rank's
bindings, and its own counts and mask, bit for bit against the CPU restatement of the unsharded batch
(test_exchange_gpu.run_two_ranks)."""
import os

import pytest

from policy_oracle import LEAST_BALANCED
from test_exchange_gpu import run_two_ranks

pytestmark = pytest.mark.gpu
FORCE_BITPAR = 2  # KS_SELECT_FORCE_BITPAR


@pytest.mark.parametrize("P,N,steps", [(20000, 3000, 3), (1, 5000, 2)])
def test_least_balanced_exchange_two_ranks(P, N, steps):
    """P = 1 leaves rank 1 with an empty shard."""
    run_two_ranks(LEAST_BALANCED, P, N, FORCE_BITPAR, steps, 37000 + (os.getpid() % 2000) + P % 7)
