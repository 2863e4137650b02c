"""Score parts at their edges on the H100 (-m gpu): ks_profile_bind, ks_node_bind, ks_fit_bind and ks_gang_fit_bind bit
for bit against their oracles on the cases of tests/score_edges.py, at policies 1, 3 and 4: node, total, every parts
word, every refusal word, hard and soft counts, free[], free_r and (gangs) placed.

Each group of cases and the mutants of the oracle arithmetic it kills (test_score_edges.py checks every claim whose
shape does not depend on the SM count, and the tie queue at N = 129 on 132 SMs):
  - PodTopologySpread: the 29 exact-half raws through existing soft counts up to 2^24 kill round-half-to-even, and the
    20 whose exact product lies below the half kill the exactly summed raw; the count that crosses 2^24 kills float32
    counts; soft_skew 2^31 and 2^32 - 1 kill soft_skew read as int32; the empty value's +1 (two zones, and a one-domain
    key) kills its omission; an ignored node's domain kills counting it; zone domains on both sides of 2048 (two nodes per
    zone, so size_k goes through both bitmaps) kill a size_k without either bitmap's domains and w read one entry off
    the log table, which the hostname key at N = 150,000 (the table's last entry) kills too.  Queues where every
    candidate, or all but one, is ignored or max is 0 are parity only.
  - InterPodAffinity: the eight truncating pairs (weight-1 preferred terms, and anti-preferred ones with negative
    raws), hard_affinity_weight 100, weight-100 duplicate terms and 20,000 existing pods in one domain kill ipa by
    integer division; the extremes only in the first or only in the last slice are the (29, 50) pair again.
  - TaintToleration: maxima 1 to 64 (64 untolerated PreferNoSchedule taints at the end) kill tt rounded and, wherever
    100 t / max is not an integer, tt as the truncated complement.
  - NodeAffinity: 4,096 weight-100 preferred terms (raw 409,600) in a rule class two groups share kill na rounded.
  - Totals: ties between (pts 100, ipa 0) and (pts 0, ipa 100) on both sides of every slice edge at N of 129, 16,897
    and 33,793 kill ties to the higher index; plugin weights 0 and 100 keep the IPA hazard where the spread lift holds.
  - Gangs: ks_gang_fit_bind on the 2^24 queue and the 20,000-pod IPA queue with a self term, where the rolled-back gang
    changed the soft counts or the IPA counters before its rollback, against its oracle and, by M1 (every min_member 0),
    against ks_fit_bind."""
import numpy as np
import pytest

import score_edges as se
from bind_edges import fit_arrays
from node_bind_oracle import compile_rules
from test_commit_paths_gpu import _free_in_range, _load

pytestmark = pytest.mark.gpu

POLICIES = (1, 3, 4)
FIELDS = ("node_idx", "score", "parts", "refused", "counts", "soft_counts", "free_r", "placed")


@pytest.fixture(scope="module")
def sms(ks):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def device(snap, case, call, policy, gangs=None):
    """The call on the snapshot as the oracle's tuple"""
    rc, rm, sel, group = case.queue()
    kw, (wt, wn) = se.device_args(case)
    args = (rc, rm, sel, group, case.G, case.keys)
    if call == "profile":
        return snap.profile_bind(*args, policy=policy, **kw) + (None,)
    kw["rules"] = compile_rules(*case.rules_cluster(), weight_taint=wt, weight_node_affinity=wn)
    if call == "node":
        return snap.node_bind(*args, policy=policy, **kw) + (None,)
    kw["node_free"], kw["pod_req"] = fit_arrays(case.res())
    if call == "fit":
        return snap.fit_bind(*args, policy=policy, **kw)
    return snap.gang_fit_bind(*args, *(gangs or case.gangs), policy=policy, **kw)


def same(got, want, tag):
    for name, g, w in zip(FIELDS, got, want):
        if w is None:
            continue
        if name in ("counts", "soft_counts"):
            assert len(g) == len(w) and all(np.array_equal(a, b) for a, b in zip(g, w)), f"{name} {tag}"
            continue
        g, w = np.asarray(g), np.asarray(w)
        bad = np.nonzero((g != w).reshape(len(g), -1).any(1))[0] if g.shape == w.shape else []
        assert g.shape == w.shape and not len(bad), f"{name} {tag}: first rows {bad[:8]} got {g[bad[:2]]} want {w[bad[:2]]}"


def check(ks, case, calls=None, policies=POLICIES):
    with ks.Snapshot(0) as snap:
        for call in calls or case.calls:
            for policy in policies:
                tag = f"{case.name} {call} policy={policy}"
                _load(snap, *case.nodes())
                got = device(snap, case, call, policy)
                want, fc, fm = se.oracle(case, call, policy)
                same(got, want, tag)
                gfc, gfm = _free_in_range(snap)
                assert np.array_equal(gfc, fc) and np.array_equal(gfm, fm), f"free {tag}"


# ------------------------------------------------------------------------------------------------ PodTopologySpread
PTS = se.pts_cases()


@pytest.mark.parametrize("case", PTS, ids=[c.name for c in PTS])
def test_pts(ks, case):
    check(ks, case)


def test_pts_hostname_at_large_n(ks):
    """N = 150,000 hosts, every node a candidate: size_k = N reads logw[N]"""
    check(ks, se.hostname_case(150_000))


# ------------------------------------------------------------------------------------------------ InterPodAffinity
IPA = se.ipa_cases()


@pytest.mark.parametrize("case", IPA, ids=[c.name for c in IPA])
def test_ipa(ks, case):
    check(ks, case)


@pytest.mark.parametrize("which", (0, 1), ids=("first-slice", "last-slice"))
def test_ipa_extremes_in_one_slice(ks, sms, which):
    check(ks, se.ipa_slice_cases(16_897, sms)[which])


# ------------------------------------------------------------------------------------ TaintToleration, NodeAffinity
RULES = se.node_rule_cases()


@pytest.mark.parametrize("case", RULES, ids=[c.name for c in RULES])
def test_node_rules(ks, case):
    check(ks, case)


# -------------------------------------------------------------------------------------------------------- totals
@pytest.mark.parametrize("N", (129, 16_897, 33_793))
def test_ties_at_every_slice_edge(ks, sms, N):
    check(ks, se.tie_case(N, sms))


WEIGHTS = se.weight_cases()


@pytest.mark.parametrize("case", WEIGHTS, ids=[c.name for c in WEIGHTS])
def test_plugin_weights(ks, case):
    check(ks, case)


# ---------------------------------------------------------------------------------------------------------- gangs
GANGS = se.gang_cases()


@pytest.mark.parametrize("case", GANGS, ids=[c.name for c in GANGS])
def test_gangs(ks, case):
    """Every output against the oracle (gang 1 rolls back over the soft counts near 2^24 or the 20,000-pod IPA
    counters), then M1: every min_member 0 is ks_fit_bind bit for bit"""
    check(ks, case, calls=("gang",))
    offset, _ = case.gangs
    with ks.Snapshot(0) as snap:
        for policy in POLICIES:
            _load(snap, *case.nodes())
            got = device(snap, case, "gang", policy, gangs=(offset, np.zeros(len(offset) - 1, np.uint32)))
            _load(snap, *case.nodes())
            want = device(snap, case, "fit", policy)
            same(got[:7], want, f"{case.name} M1 policy={policy}")
            assert np.array_equal(got[7], [(want[0][int(offset[j]):int(offset[j + 1])] >= 0).sum()
                                           for j in range(len(offset) - 1)])
