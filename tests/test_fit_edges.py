"""Preemption and drain under the full filter at their edges, CPU part: the grid model against a brute-force
recomputation and the launcher's source, each case of tests/fit_edges.py on the hazard it claims (at 114 and 132 SMs
where the shape depends on the SM count), and every mutant of the two restatements against the cases that claim to kill
it, so that test_fit_edges_gpu.py fails on a kernel that makes that mistake.  Run with -s to see each mutant's killers."""
import os

import numpy as np
import pytest

import fit_edges as fe
import fit_preempt_oracle as fpo

SMS = (114, 132)  # H100 PCIe and SXM
CASES = fe.cpu_cases()
BY_NAME = {c.name: c for c in CASES}


def geometry(kind, sms, _memo={}):
    if (kind, sms) not in _memo:
        _memo[kind, sms] = fe.geometry_case(kind, sms)
    return _memo[kind, sms]


# ---------------------------------------------------------------------------------------------------- grid model
def _brute_grid(ppw, P, N, sms):
    """The launch by enumeration: the smallest chunk count that gives two CTAs per SM (capped at the tiles), the
    smallest tiles per chunk that covers the tiles with it, and the chunks the tiles then fall in"""
    per_cta = fe.DIRECT_THREADS // 32 * ppw
    n_tiles = next(t for t in range(1, N + 2) if t * fe.TILE_N >= N)
    pod_ctas = next(c for c in range(1, P + 2) if c * per_cta >= P)
    if pod_ctas >= 2 * sms:
        want = 1
    else:
        want = min(n_tiles, next(c for c in range(1, 2 * sms + 1) if c * pod_ctas >= 2 * sms))
    tpc = next(t for t in range(1, n_tiles + 1) if t * want >= n_tiles)
    chunks = sorted({t // tpc for t in range(n_tiles)})
    assert chunks == list(range(len(chunks)))
    return pod_ctas, len(chunks), tpc, n_tiles


@pytest.mark.parametrize("sms", (1, 2, 114, 132))
def test_grid_model_matches_brute_force(sms):
    for P in (1, 7, 8, 9, 64, 455, 456, 528, 912, 1823, 1824, 2111, 2112, 2113, 5000):
        for N in (1, 1023, 1024, 1025, 3072, 9221, 10_000, 2 * sms * 1024 + 1, 270_337):
            for ppw in (fe.FIT_PREEMPT_PODS_PER_WARP, fe.FIT_DRAIN_PODS_PER_WARP, 2, 8):
                g = fe.direct_grid(ppw, P, N, sms)
                assert (g.pod_ctas, g.n_chunks, g.tiles_per_chunk, g.n_tiles) == _brute_grid(ppw, P, N, sms)
                ch = g.chunks()
                assert ch[0][0] == 0 and ch[-1][1] == N - 1
                assert all(a[1] + 1 == b[0] for a, b in zip(ch, ch[1:]))


def test_grid_model_reads_the_launcher():
    """The constants come from the sources, and both launchers size their grid by direct_grid_ppw with them"""
    assert fe.TILE_N == 1024 and fe.DIRECT_THREADS == 256
    with open(os.path.join(fe.CSRC, "ks_direct.cu")) as f:
        src = f.read()
    assert "return direct_grid_ppw(FIT_PREEMPT_PODS_PER_WARP, P, Npad, sms);" in src
    assert "return direct_grid_ppw(FIT_DRAIN_PODS_PER_WARP, P, Npad, sms);" in src
    assert "if (g.pod_ctas < want_ctas) g.n_chunks = std::min<uint32_t>(n_tiles, (want_ctas + g.pod_ctas - 1) / g.pod_ctas);" in src
    assert "g.n_chunks = (n_tiles + g.tiles_per_chunk - 1) / g.tiles_per_chunk;" in src


# ------------------------------------------------------------------------------------------------------ geometry
@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("kind", fe.GEOMETRY)
def test_geometry_reaches_its_shape(kind, sms):
    """(a) chunks of 2 tiles and a short last one, (b) 4 chunks of 3, 3, 3, 1 tiles, (c) one chunk over 10 tiles; the
    candidates lie on both sides of every chunk edge and on N - 1; every other node is unresolvable"""
    case = geometry(kind, sms)
    d = case.d
    P, N = len(d["rc"]), len(d["fc"])
    g = fe.preempt_grid(P, N, sms)
    if kind == "a":
        assert g.tiles_per_chunk == 2 and g.uneven and g.n_chunks == sms + 1
    elif kind == "b":
        assert (g.n_chunks, g.tiles_per_chunk, g.n_tiles) == (4, 3, 10) and g.uneven
    else:
        assert g.n_chunks == 1 and g.n_tiles == 10
    cand = {n for n, lab in enumerate(d["node_labels"]) if lab.get("c")}
    for first, last in g.chunks()[1:]:
        assert {first - 1, first} <= cand
    assert {0, N - 1} <= cand
    assert len(cand) == 2 + 2 * (g.n_tiles - 1) - (N - 1 == (g.n_tiles - 1) * fe.TILE_N)  # (a): N - 1 starts a tile


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("kind", fe.GEOMETRY)
def test_geometry_winners(kind, sms):
    """The all-candidate pods at priority 10 pick the star node, the last node of a chunk with candidates in its earlier
    tiles, and count every candidate; a tied pair on a chunk edge goes to its left node; an even pair at priority 0 has no
    candidate; the unresolvable count is every node without the selector's label"""
    case = geometry(kind, sms)
    d = case.d
    P, N = len(d["rc"]), len(d["fc"])
    g = fe.preempt_grid(P, N, sms)
    rows, _, unres = fe.run(case, 3)
    star = case.notes["star"] * fe.TILE_N - 1
    cand = [n for n, lab in enumerate(d["node_labels"]) if lab.get("c")]
    assert [n for n in cand if g.chunk_of(n) == g.chunk_of(star) and n < star]
    all10 = (np.arange(P) % 4 == 0)
    assert (rows["node_idx"][all10] == star).all() and (rows["candidates"][all10] == len(cand)).all()
    assert (unres[all10] == N - len(cand)).all()
    edge_ties = 0
    for p in np.flatnonzero(np.arange(P) % 4 == 1):
        t = int(d["node_labels"][int(rows["node_idx"][p])]["e"])
        left, right = t * fe.TILE_N - 1, t * fe.TILE_N
        assert int(rows["node_idx"][p]) == (right if t % 2 and t != case.notes["star"] else left)
        edge_ties += t % 2 == 0 and g.chunk_of(left) != g.chunk_of(right)
    assert edge_ties or kind == "c"
    assert (rows["node_idx"][np.arange(P) % 4 == 2] >= -1).all()


@pytest.mark.parametrize("sms", SMS)
def test_drain_geometry_shape(sms):
    """The drain case's rounds and refusal pass run on chunks of 2 tiles with a short last one; x sits on both sides of
    every chunk edge; candidate 0 stops with every destination refused on x"""
    case = fe.drain_geometry_case(sms)
    d = case.d
    N, D = len(d["fc"]), len(d["node_idx"])
    g = fe.drain_grid(D, N, sms)
    assert g.tiles_per_chunk == 2 and g.uneven
    xs = set(case.notes["xs"])
    assert all({first - 1, first} <= xs for first, _ in g.chunks()[1:])
    if sms == 132:
        placed, _, _, refused = fe.run(case, (0, 0))
        size = np.diff(d["offset"].astype(np.int64))
        assert placed[0] < size[0] and refused[0].tolist() == [0, N - 1, 0, 0]
        assert (placed[1:] == size[1:]).all()


# ---------------------------------------------------------------------------------------------------- the cases
def _only(d, n):
    """d with one more label word that only node n carries and every pod selects: the plans on node n alone"""
    e = dict(d)
    col = np.zeros((len(d["fc"]), 1), np.uint64)
    col[n] = 1
    e["labels"] = np.concatenate([d["labels"], col], axis=1)
    e["sel"] = np.concatenate([d["sel"], np.ones((len(d["rc"]), 1), np.uint64)], axis=1)
    return e


def plan(case, n, mv=128, p=0):
    """(vmax, vsum, vcnt) of pod p's plan on node n alone"""
    rows, vic, _ = fpo.run(_only(case.d, n), mv)
    assert rows["node_idx"][p] == n
    return int(rows["max_victim_priority"][p]), int(rows["victim_priority_sum"][p]), int(rows["n_victims"][p])


def test_key_cases_tie_in_all_but_one_field():
    a, b = (plan(BY_NAME["key: sum's low 8 bits"], n) for n in (0, 1))
    assert a[0] == b[0] and a[2] == b[2] and a[1] != b[1] and a[1] >> 8 == b[1] >> 8
    a, b = (plan(BY_NAME["key: count only"], n) for n in (0, 1))
    assert a[:2] == b[:2] and a[2] > b[2]
    a, b = (plan(BY_NAME["key: sum before count"], n) for n in (0, 1))
    assert a[0] == b[0] and a[1] > b[1] and a[2] < b[2]
    case = BY_NAME["key: node ties across a chunk edge"]
    assert plan(case, 1023) == plan(case, 1024)
    for sms in SMS:
        g = fe.preempt_grid(len(case.d["rc"]), len(case.d["fc"]), sms)
        assert g.chunk_of(1023) != g.chunk_of(1024)
    a, b = (plan(BY_NAME["key: sum near 2^39"], n) for n in (0, 1))
    assert a[2] == b[2] == 128 and a[0] == b[0] and 0 < a[1] - b[1] < 256
    assert (1 << 39) - 512 < b[1] < a[1] < 1 << 39


def test_walk_cases_sit_on_their_boundary():
    for case in CASES:
        what = case.notes.get("zero")
        if what is None:
            continue
        d = case.d
        rows, vic, _ = fe.run(case, 128)
        v = [int(x) for x in vic[0] if x >= 0]
        assert rows["node_idx"][0] == 0 and len(v) == 1 and len(d["bound"]) == 2
        freed = [d["bound"][b] for b in v]
        if what == "cpu":
            left = int(d["fc"][0]) + sum(b[1] for b in freed) - int(d["rc"][0])
        elif what == "memory":
            left = int(d["fm"][0]) + sum(b[2] for b in freed) - int(d["rm"][0])
        elif what == "pods":
            left = int(d["node_free"][0, 0]) + len(freed) - 1
        else:
            left = int(d["node_free"][1, 0]) + sum(b[4][d["names"][1]] for b in freed) - int(d["pod_req"][0, 1])
        assert left == 0, what
    case = BY_NAME["walk: max_victims = needed, needed - 1"]
    assert fe.run(case, 3)[0]["n_victims"][0] == 3 and fe.run(case, 2)[0]["node_idx"][0] == -1
    case = BY_NAME["walk: bound pod at the pod's priority"]
    assert {b[3] for b in case.d["bound"]} >= {int(case.d["prio"][0])}
    case = BY_NAME["walk: priorities INT32_MIN and INT32_MAX"]
    assert {int(x) for x in case.d["prio"]} == {fe.INT32_MIN, fe.INT32_MIN + 1, fe.INT32_MAX}
    rows = fe.run(case, 3)[0]
    assert rows["victim_priority_sum"][2] == 0 and rows["max_victim_priority"][2] == fe.INT32_MIN


def test_scalar_cases_sit_on_their_edge():
    for name in ("scalar: R = 8, requests r2, r5, r7", "drain: R = 8, requests r2, r5, r7"):
        d = BY_NAME[name].d
        assert len(d["names"]) == 8
        assert [r for r in range(8) if d["pod_req"][0, r]] == [0, 2, 5, 7]
        assert (d["node_free"][[1, 3, 4, 6]] < 0).all()
    d = BY_NAME["scalar: zero request, negative free"].d
    assert (d["pod_req"][:, 1] == 0).all() and (d["node_free"][1] < 0).all()
    d = BY_NAME["drain: zero request, negative free"].d
    assert (d["pod_req"][:, 1] == 0).all() and d["node_free"][1, 1] < 0
    case = BY_NAME["drain: x to 0, then refusal word 1"]
    for policy, flags in fe.RUNS:
        placed, idx, _, refused = fe.run(case, (policy, flags))
        assert placed.tolist() == [1, 1] and idx[0] == 1
        assert refused[0].tolist() == case.notes["want_refused"] if not flags else refused[0].tolist() == [0, 2, 1, 1]
    placed, idx, _, refused = fe.run(BY_NAME["drain: pods to 0, then refusal word 1"], (0, 0))
    assert placed.tolist() == [2] and idx.tolist() == [1, 1, -1] and refused[0].tolist() == [2, 1, 0, 0]


# --------------------------------------------------------------------------------------------------- the mutants
@pytest.mark.parametrize("name", list(fe.MUTANTS))
def test_mutant_is_killed(capsys, name):
    """Every case that lists the mutant tells it apart.  The killers are written to the terminal with the result."""
    claimed = [c for c in CASES if name in c.kills]
    claimed += [geometry(k, 132) for k in fe.GEOMETRY if name in geometry(k, 132).kills]
    assert claimed, f"no case claims {name}"
    with capsys.disabled():
        print(f"\n{name} ({fe.MUTANTS[name][0]}): killed by {len(claimed)} cases: {', '.join(c.name for c in claimed)}")
    survives = [c.name for c in claimed if not fe.kills(c, name)]
    assert not survives, f"{name} survives {survives}"


def test_drain_geometry_kills():
    case = fe.drain_geometry_case(132)
    assert [m for m in case.kills if not fe.kills(case, m)] == []


@pytest.mark.parametrize("name", list(fe.NEUTRAL))
def test_neutral_mutant_is_indistinguishable(capsys, name):
    with capsys.disabled():
        print(f"\n{name}: no reachable input tells it apart: {fe.NEUTRAL[name][0]}")
    uses = [c for c in CASES if c.call == "preempt"]
    assert not [c.name for c in uses if fe.kills(c, name)]
