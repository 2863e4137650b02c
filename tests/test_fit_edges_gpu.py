"""Preemption and drain under the full filter at their edges on the H100 (-m gpu): ks_fit_preempt and ks_fit_drain_check
bit for bit against their restatements on the cases of tests/fit_edges.py - every row field, victim slot and
unresolvable count at max_victims 1, 3 and 128 (or the case's own), and placed, node, score and the refusal words at
all four policies with and without KS_DRAIN_EXCLUDE_CANDIDATES - with free[] and ks_select on both paths unchanged
after every call.

The families and the mutants of the restatements each kills (test_fit_edges.py checks every claim on the CPU):
  - Geometry, with the device's SM count: (a) 8 pods over 2 sms + 1 tiles, chunks of 2 tiles and a short last one;
    (b) four chunks over ten tiles, the last of one; (c) one chunk over all ten tiles.  Candidates on both sides of
    every tile boundary and on N - 1, the best one the last node of a chunk, unresolvable sums across every chunk and
    the padding: node ties to the higher index, bound pods at the pod's priority in the lower set.  Q1 (rules and
    resources NULL is ks_preempt) on each shape.
  - Victim key: sums that differ in the low 8 bits only, counts alone, sum against count, one plan on both sides of a
    chunk edge, 128 victims with sums within 2^8 of each other near 2^39.
  - Reprieve walk: a bound pod at the pod's priority, equal priorities in bound order, reprieves that leave exactly 0
    cpu, memory, a scalar resource and pods, max_victims at the victims needed and one below, priorities INT32_MIN and
    INT32_MAX.
  - Scalar edges: zero requests on negative free amounts, requests r2, r5, r7 at R = 8, a drain overlay that takes x
    or the pod count to exactly 0 (the next pod refused with word 1, also where a taint fails too), ties to the lower
    index, and a drain on the chunks of (a) whose picks tie everywhere.  D1 (rules and resources NULL is
    ks_drain_check) on every drain case."""
import numpy as np
import pytest

import fit_edges as fe
import fit_preempt_oracle as fpo
from test_fit_drain_gpu import call as drain_call, load as drain_load, same as drain_same, select_state
from test_fit_preempt_gpu import device as preempt_device, same as preempt_same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sms(ks):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def preempt_runs(ks, d, mvs, with_res=True, with_rules=True):
    """Snapshot.fit_preempt at each max_victims on one snapshot; free[] and ks_select on both paths unchanged after
    every call"""
    probe = slice(0, min(len(d["rc"]), 200))
    with ks.Snapshot(0) as s:
        s.set_nodes(d["ac"], d["am"], d["labels"])
        s.set_bound(d["bn"], d["bc"], d["bm"])
        before = s.free(), select_state(ks, s, d["rc"][probe], d["rm"][probe], d["sel"][probe])
        outs = []
        for mv in mvs:
            outs.append(preempt_device(ks, d, mv, with_rules=with_rules, with_res=with_res, snap=s))
            after = s.free(), select_state(ks, s, d["rc"][probe], d["rm"][probe], d["sel"][probe])
            assert all(np.array_equal(a, b) for a, b in zip(before[0], after[0])), "free[] changed"
            for x, y in zip(before[1], after[1]):
                assert all(np.array_equal(a, b) for a, b in zip(x, y)), "ks_select changed"
        if not with_rules and not with_res:  # Q1
            for mv, got in zip(mvs, outs):
                rows, vic = s.preempt(d["rc"], d["rm"], d["sel"], d["prio"], d["bn"], d["bc"], d["bm"], d["bp"], mv)
                assert all(np.array_equal(got[0][f], rows[f]) for f in rows.dtype.names) and np.array_equal(got[1], vic)
    return outs


def check_preempt(ks, case):
    for mv, got in zip(case.mvs, preempt_runs(ks, case.d, case.mvs)):
        preempt_same(got, fe.run(case, mv))


def check_drain(ks, case, runs=fe.RUNS):
    d = case.d
    with ks.Snapshot(0) as s:
        drain_load(ks, s, d)
        for policy, flags in runs:
            drain_same(drain_call(ks, s, d, policy, flags), fe.run(case, (policy, flags)))
        # without the resources, and D1: rules and resources NULL against ks_drain_check
        drain_same(drain_call(ks, s, d, 0, 0, with_res=False),
                   fe.fdo.fit_drain(d, d["node_idx"], d["offset"], 0, False, with_res=False))
        drain_call(ks, s, d, 4, 1, with_rules=False, with_res=False)


PREEMPT = [c for c in fe.cpu_cases() if c.call == "preempt"]
DRAIN = [c for c in fe.cpu_cases() if c.call == "drain"]


@pytest.mark.parametrize("case", PREEMPT, ids=[c.name for c in PREEMPT])
def test_preempt_cases(ks, case):
    check_preempt(ks, case)


@pytest.mark.parametrize("case", DRAIN, ids=[c.name for c in DRAIN])
def test_drain_cases(ks, case):
    check_drain(ks, case)


@pytest.mark.parametrize("kind", fe.GEOMETRY)
def test_preempt_geometry(ks, sms, kind, capsys):
    """Each family on the device's own grid, which the test states and checks, then Q1 on the same shape"""
    case = fe.geometry_case(kind, sms)
    d = case.d
    g = fe.preempt_grid(len(d["rc"]), len(d["fc"]), sms)
    with capsys.disabled():
        print(f"\n{case.name}: {g}")
    if kind == "a":
        assert g.tiles_per_chunk >= 2 and g.uneven
    elif kind == "b":
        assert g.n_chunks == 4 and g.n_tiles == 10 and g.uneven
    else:
        assert g.n_chunks == 1 and g.n_tiles > 1
    check_preempt(ks, case)
    for mv, got in zip(fe.MVS, preempt_runs(ks, d, fe.MVS, with_res=False, with_rules=False)):
        preempt_same(got, fpo.run(d, mv, with_res=False))


def test_drain_geometry(ks, sms, capsys):
    case = fe.drain_geometry_case(sms)
    g = fe.drain_grid(len(case.d["node_idx"]), len(case.d["fc"]), sms)
    with capsys.disabled():
        print(f"\n{case.name}: {g}")
    assert g.tiles_per_chunk >= 2 and g.uneven
    check_drain(ks, case, runs=((0, 0), (0, 1), (1, 0), (3, 1), (4, 0)))
