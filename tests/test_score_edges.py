"""Score parts at their edges, CPU part: the hazard fixture (tests/golden/score_edges.json) against the searches that
made it, every case of tests/score_edges.py through the real oracle, and every mutant of the oracle arithmetic against
the cases that claim to kill it, so that test_score_edges_gpu.py fails on a kernel that makes that mistake.  The shapes of
the GPU cases that depend on the SM count are checked at 114 and 132 SMs.  Run with -s to see each mutant's killers."""
import math
from fractions import Fraction

import numpy as np
import pytest

import score_edges as se
from bind_edges import bind_slices

SMS = (114, 132)  # H100 PCIe and SXM
CASES = se.cpu_cases()
NEUTRAL_INPUT = {"float32-existing": "existing", "uint32-skew": "soft_skew"}  # the input each neutral patch reads


@pytest.fixture(scope="module")
def results():
    """The oracle's outputs of every case and call at policy 4, memoised (the policy score is one constant over the
    nodes of every case, so the policy does not move a hazard; the GPU file runs policies 1, 3 and 4)"""
    return {}


def real(results, case, call):
    key = (case.name, call)
    if key not in results:
        results[key] = se.oracle(case, call, 4)[0]
    return results[key]


def killed(results, case, name):
    """Whether mutant `name` changes the node, score or parts of some call of the case"""
    for call in case.calls:
        with se.mutant(name):
            got = se.oracle(case, call, 4)[0]
        if se.differs(got, real(results, case, call)):
            return True
    return False


# --------------------------------------------------------------------------------------------------- the fixture
def test_exact_halves_fixture():
    """Each stored (size, sc) gives exactly k + 0.5 in double, below or above the exact product as stored; sizes 15 and
    132 searched again over the whole count range give the same entries; 29 entries, 14 with an even floor, 20 with
    the exact product below the half"""
    fx = se.fixture()["exact_halves"]
    for size, sc, k, below in fx:
        w = math.log(size + 2)
        assert float(sc) * w == k + 0.5 and sc <= se.MAX_EXISTING
        assert (Fraction(sc) * Fraction(w) < Fraction(2 * k + 1, 2)) == below
    assert se.search_exact_halves((15, 132)) == [h for h in fx if h[0] in (15, 132)]
    assert len(fx) == 29 and sum(h[2] % 2 == 0 for h in fx) == 14 and sum(h[3] for h in fx) == 20


def test_truncating_pairs_fixture():
    """The eight (a, b), b <= 200, where the double ipa truncates below the integer quotient, and the pair at b = 20,000"""
    fx = se.fixture()
    assert fx["truncating"] == se.search_truncating() == [[29, 50], [29, 100], [57, 100], [58, 100], [87, 150],
                                                          [58, 200], [114, 200], [116, 200]]
    a, b = fx["truncating_20000"]
    assert b == 20_000 and a == se.truncating_at(b) and int(100.0 * (a / b)) == 100 * a // b - 1


# ---------------------------------------------------------------------------------------------------- the cases
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_case_reproduces_its_hazard(results, case):
    """The oracle gives each case's stated part values on every call it applies to, and binds every pod"""
    for call in case.calls:
        node, score, parts = real(results, case, call)[:3]
        assert (node >= 0).all(), call
        for p, word, value in case.expect:
            assert parts[p, word] == value, (call, p, word, parts[p])


@pytest.mark.parametrize("name", list(se.MUTANTS))
def test_mutant_is_killed(results, capsys, name):
    """Every case that lists the mutant tells it apart: node, score or parts differ.  The killers are written to the
    terminal with the test's result."""
    claimed = [c for c in CASES if name in c.kills]
    assert claimed, f"no case claims {name}"
    with capsys.disabled():
        print(f"\n{name} ({se.MUTANTS[name][0]}): killed by {len(claimed)} cases: {', '.join(c.name for c in claimed)}")
    survives = [c.name for c in claimed if not killed(results, c, name)]
    assert not survives, f"{name} survives {survives}"


@pytest.mark.parametrize("name", list(se.NEUTRAL))
def test_neutral_mutant_is_indistinguishable(results, capsys, name):
    """The mistakes no reachable input can show leave every case unchanged"""
    with capsys.disabled():
        print(f"\n{name}: no reachable input tells it apart: {se.NEUTRAL[name][0]}")
    uses = [c for c in CASES if c.kw.get(NEUTRAL_INPUT[name]) is not None]  # elsewhere the patched line reads nothing
    assert len(uses) > 50
    assert not [c.name for c in uses if killed(results, c, name)]


# --------------------------------------------------------------------------------------- shapes at 114 and 132 SMs
@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("N", (129, 16_897, 33_793))
def test_tie_queue_straddles_every_edge(sms, N):
    """Every slice edge has one 'a' node (pts 100, ipa 0) and one 'b' node (pts 0, ipa 100) on its two sides, the side
    alternating from edge to edge, and the first pod's candidates all tie at 200 over both decompositions"""
    case = se.tie_case(N, sms)
    grid, chunk = bind_slices(N, sms)
    E = set(se.tie_nodes(N, sms).tolist())
    b = set(case.kw["existing_pods"][1].tolist())
    sides = []
    for s in range(1, grid):
        e = s * chunk
        if e < N:
            assert {e - 1, e} <= E and ((e - 1 in b) != (e in b)), (s, e)
            sides.append(e - 1 in b)
    assert all(x != y for x, y in zip(sides, sides[1:]))
    F = sorted(E)
    pts = se.profile_bind_oracle.pts_scores(F, 0, case.kw["soft_skew"], np.ones(2, np.int64), [case.keys[0][0]],
                                            [case.kw["existing"][0]])
    assert {pts[n] for n in F} == {0, 100} and all((pts[n] == 0) == (n in b) for n in F)


@pytest.mark.parametrize("sms", SMS)
def test_ipa_extremes_sit_in_one_slice(sms):
    """The slice cases: min and max both in the first slice and the winner in the last non-empty one, then the other way
    round"""
    N = 16_897
    grid, chunk = bind_slices(N, sms)
    first, last = se.ipa_slice_cases(N, sms)
    for case, (lo, mid, hi) in ((first, (0, N - 1, 1)), (last, (N - 1, 0, N - 2))):
        assert case.kw["existing_pods"][1].min() >= 0
        assert lo // chunk == hi // chunk and lo // chunk != mid // chunk
    assert (N - 1) // chunk == (N - 2) // chunk != 0


@pytest.mark.parametrize("sms", SMS)
def test_bitmap_edge_domains(sms):
    """The zone key has two nodes per domain, so the walk counts size_k through the domain bitmaps rather than by nodes;
    the candidates' 26 zones lie on both sides of 2048 (8 below, 18 at or above, up to 4099) and in several slices; the
    winner's zone is 2048 and the maximum's 2047"""
    case = se.bitmap_edge_case()
    zone = case.keys[0][0]
    assert np.bincount(zone).max() >= 2
    cand = np.flatnonzero(case.lab[:, 0])
    zones = np.unique(zone[cand])
    assert len(zones) == 26 and (zones < se.SHARED_BITMAP).sum() == 8 and zones.max() == 4099
    assert 2047 in zones and 2048 in zones
    assert zone[case.kw["existing_pods"][1][0]] == 2048 and case.kw["existing"][0][0, 2047] > case.kw["existing"][0][0, 2048]
    _, chunk = bind_slices(case.N, sms)
    assert len({int(n) // chunk for n in cand}) >= 2


def test_hostname_at_large_n_reads_the_last_logw_entry(capsys):
    """At N = 150,000 every node is a candidate on the hostname soft key: size = N, the last entry the call reads of its
    log table [N + 2].  The winner sits between the extremes, so its pts turns on w: log(N + 3) changes it."""
    N = 150_000
    case = se.hostname_case(N)
    assert case.keys[0][1] == N and (case.keys[0][0] >= 0).all() and case.lab is None
    want = se.oracle(case, "profile", 4)[0]
    for p, word, value in case.expect:
        assert want[2][p, word] == value
    with se.mutant("logw-shifted"):
        assert se.differs(se.oracle(case, "profile", 4)[0], want)
    with capsys.disabled():
        print(f"\nlogw-shifted: also killed by {case.name}")


@pytest.mark.parametrize("case", se.gang_cases(), ids=lambda c: c.name)
def test_gang_rollback_is_visible(case):
    """The middle gang binds one pod and rolls back.  Had it not rolled back (every min_member 0, which is ks_fit_bind
    on the same queue), the final soft counts (the 2^24 queue) or the last gang's ipa parts (the IPA queue) would
    differ: so a rollback that leaves the soft counts or the IPA counters changed shows in the outputs"""
    offset, mm = case.gangs
    got = se.oracle(case, "gang", 4)[0]
    assert (got[0][int(offset[1]):int(offset[2])] < 0).all() and got[7][1] == 1  # placed 1 of 2, rolled back
    kept = se.oracle(case, "fit", 4)[0]
    last = slice(int(offset[2]), int(offset[3]))
    assert (got[0][last] >= 0).all()
    parts_differ = not np.array_equal(got[2][last], kept[2][last])
    soft_differ = any(not np.array_equal(a, b) for a, b in zip(got[5], kept[5]))
    assert parts_differ or soft_differ
    if "ipa" in case.name:  # the IPA counters: one point of ipa for the last gang
        assert parts_differ
