"""Soft constraints when binding (ks_profile_bind), CPU part: hand-derived queues against the restatement of
tests/profile_bind_oracle.py; identities J1 (no soft term is ks_affinity_bind), J2 (soft terms on a one-domain key add
100 * weight_spread and move nothing) and J3 (preferred terms are symmetric in their owner) on the restatements; Go's
rounding and both normalisations at their edges; the C / ctypes mirrors; and the errors caught without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from affinity_bind_oracle import AFFINITY, ANTI, affinity_bind_packed
from helpers import load_golden
from profile_bind_oracle import ANTI_PREFERRED, PREFERRED, go_round, pts_scores, profile_bind_packed
from test_replicas import random_cluster
from test_spread_bind import _queue, _random_keys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = (1, 3, 4)


def golden_runs():
    """Every run of tests/golden/gv1_profile_bind.json: (id, args, scoring, expected), args and scoring as
    profile_bind_packed and Snapshot.profile_bind take them after the cluster arrays."""
    for case in load_golden("gv1_profile_bind.json")["cases"]:
        n = case["nodes"]
        N, P, G = len(n["alloc_cpu"]), len(case["pods"]), case["G"]
        keys = [(np.array(d, np.int32), D) for d, D in case["keys"]]
        pods = np.array(case["pods"], np.int64).reshape(P, 3)
        ex = case.get("existing")
        args = dict(fc=np.array(n["free_cpu"], np.int64), fm=np.array(n["free_mem"], np.int64),
                    ac=np.array(n["alloc_cpu"], np.int64), am=np.array(n["alloc_mem"], np.int64),
                    lab=np.zeros((N, 1), np.uint64), rc=pods[:, 0].copy(), rm=pods[:, 1].copy(),
                    sel=np.zeros((P, 1), np.uint64), group=pods[:, 2].astype(np.int32), G=G, keys=keys,
                    terms=[tuple(t) for t in case.get("terms", [])],
                    ex_pods=None if "existing_pods" not in case else tuple(np.array(e) for e in case["existing_pods"]),
                    skew=None if "max_skew" not in case else np.array(case["max_skew"], np.uint32),
                    ex=None if ex is None else [np.array(e, np.uint32) for e in ex], policy=case["policy"])
        for i, run in enumerate(case["runs"]):
            scoring = dict(soft_skew=case.get("soft_skew"), soft_all_keys=case.get("soft_all_keys"),
                           term_weight=case.get("term_weight"))
            scoring.update(run["scoring"])
            yield f"{case['name']} / {i}", args, scoring, run


def run_oracle(args, scoring):
    a = args
    fc, fm = a["fc"].copy(), a["fm"].copy()
    got = profile_bind_packed(fc, fm, a["ac"], a["am"], a["lab"], a["rc"], a["rm"], a["sel"], a["group"], a["G"],
                              a["keys"], a["terms"], a["ex_pods"], a["skew"], None, a["ex"], a["policy"], **scoring)
    return got, (fc, fm)


def assert_golden(got, want, name):
    assert got[0].tolist() == want["node"], name
    assert got[1].tolist() == want["score"], name
    assert got[2].tolist() == want["parts"], name
    for i, k in ((4, "counts"), (5, "soft_counts")):
        if k in want:
            assert [c.tolist() for c in got[i]] == want[k], (name, k)


@pytest.mark.parametrize("run", list(golden_runs()), ids=lambda r: r[0])
def test_golden_against_the_oracle(run):
    name, args, scoring, want = run
    got, _ = run_oracle(args, scoring)
    assert_golden(got, want, name)


def _uniform(n, cpu=4000, mem=16 << 30):
    fc, fm = np.full(n, cpu, np.int64), np.full(n, mem, np.int64)
    return fc, fm, fc.copy(), fm.copy(), np.zeros((n, 1), np.uint64)


def test_system_default_spread_moves_replicas():
    """Three identical replicas on four equal nodes in two zones (nodes 0, 1 in zone 0; 2, 3 in zone 1), request
    1000m / 4 GiB of 4000m / 16 GiB, LEAST_BALANCED.  Resources alone take nodes 0, 1, 2: after replica 1, node 0
    scores lower and node 1 is the next equal node by index, in the same zone.  With the system default constraints
    (zone 5, hostname 3, soft_all_keys 0), size_zone = 2 and size_host = 4, so w = log 4 and log 6:
      replica 2: raw(0) = round(1 * log 4 + 4 + 1 * log 6 + 2) = round(9.18) = 9, raw(1) = round(log 4 + 4 + 2) = 7,
      raw(2) = raw(3) = 6; max 9, min 6: pts = 100 * (15 - raw) / 9 = 66, 88, 100, 100, and node 2 wins;
      replica 3: raw = 9, 7, 9, 7 and pts = 77, 100, 77, 100; nodes 1 and 3 tie and node 1 wins by index."""
    fc, fm, ac, am, lab = _uniform(4)
    zone, host = np.array([0, 0, 1, 1]), np.arange(4)
    keys = [(zone, 2), (host, 4)]
    rc, rm = np.full(3, 1000, np.int64), np.full(3, 4 << 30, np.int64)
    sel = np.zeros((3, 1), np.uint64)
    plain = profile_bind_packed(fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, [0, 0, 0], 1, keys)
    got = profile_bind_packed(fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, [0, 0, 0], 1, keys,
                              soft_skew=[[5, 3]], soft_all_keys=[0])
    assert plain[0].tolist() == [0, 1, 2]  # resources alone: the next equal node by index
    assert got[0].tolist() == [0, 2, 1]
    assert got[2][1].tolist() == [int(got[2][1][0]), 100, 0]
    assert [c.tolist() for c in got[5]] == [[[2, 1]], [[1, 1, 1, 0]]]


def test_ignored_node_loses_by_two_hundred():
    """Explicit constraints (soft_all_keys 1) on zone: node 1 has no zone and is ignored (pts 0); node 0 gets 100.
    Both score the same under the policy, so node 0 wins by exactly weight_spread * 100 = 200."""
    fc, fm, ac, am, lab = _uniform(2)
    keys = [(np.array([0, -1]), 1)]
    got = profile_bind_packed(fc.copy(), fm.copy(), ac, am, lab, [1000], [4 << 30], np.zeros((1, 1), np.uint64), [0], 1,
                              keys, soft_skew=[[1]], soft_all_keys=[1])
    assert got[0][0] == 0 and got[2][0][1] == 100
    # the margin: both nodes score the same under the policy, and the ignored one loses exactly 2 * 100
    alone = profile_bind_packed(fc.copy(), fm.copy(), ac, am, lab, [1000], [4 << 30], np.zeros((1, 1), np.uint64),
                                [0], 1, keys, soft_skew=[[1]], soft_all_keys=[1], weight_spread=0)
    assert alone[0][0] == 0 and got[1][0] - alone[1][0] == 200 and got[2][0][0] == alone[1][0]
    # node 0 made unfit: the ignored node still binds, with pts 0
    got = profile_bind_packed(np.array([0, 4000]), fm.copy(), ac, am, lab, [1000], [4 << 30],
                              np.zeros((1, 1), np.uint64), [0], 1, keys, soft_skew=[[1]], soft_all_keys=[1])
    assert got[0][0] == 1 and got[2][0][1] == 0 and got[5][0].tolist() == [[0]]  # nor does the soft count rise


def test_self_preferred_anti_affinity_counts_twice():
    """Group 0 prefers (weight 10) not to share a hostname with itself.  One existing pod of group 0 on node 0: the
    bound pod's term and the incoming pod's term each add -10, so node 0's raw is -20 and the others 0."""
    from profile_bind_oracle import ipa_raw
    dom = [np.arange(3)]
    raw = ipa_raw(0, [(0, 0)], [(0, ANTI_PREFERRED, 0, {0})], [10], 1, dom)
    assert raw.tolist() == [-20, 0, 0]
    # an existing pod's required affinity to the incoming group adds hard_affinity_weight
    raw = ipa_raw(1, [(0, 2)], [(0, AFFINITY, 0, {1})], [0], 7, dom)
    assert raw.tolist() == [0, 0, 7]


def test_go_round_and_normalisation_edges():
    assert [go_round(x) for x in (0.5, 1.5, 2.5, -0.5, -2.5, 0.49999999999999994, 2.4999999999999996)] == \
        [1, 2, 3, -1, -3, 0, 2]
    dom = [np.array([0, 0, 0])]
    sc = [np.zeros((1, 1), np.int64)]
    # max = 0 (every raw 0 with max_skew 1): every node 100
    assert pts_scores([0, 1, 2], 0, np.array([[1]]), np.array([1]), dom, sc) == {0: 100, 1: 100, 2: 100}
    # max = min > 0: 100 * (max + min - raw) / max = 100
    assert pts_scores([0, 1], 0, np.array([[3]]), np.array([1]), dom, sc) == {0: 100, 1: 100}


def _random_scoring_case(rng, n_max=12):
    fc, fm, ac, am, labels, rc, rm, sel, _ = random_cluster(rng, n_max=n_max)
    N = len(fc)
    K = int(rng.integers(1, 4))
    keys = _random_keys(rng, N, K)
    G = int(rng.integers(1, 4))
    P = int(rng.integers(1, 20))
    qc, qm, qs, group = _queue(rng, rc, rm, sel, G, P)
    return fc, fm, ac, am, labels, qc, qm, qs, group, G, keys


@pytest.mark.parametrize("policy", POLICIES)
def test_j1_no_soft_terms_is_affinity_bind(policy):
    """J1 on the restatements, which share only affinity_mask: nodes, scores, both refusals, hard counts and free[]."""
    rng = np.random.default_rng(0x5C1 + policy)
    for it in range(60):
        fc, fm, ac, am, labels, qc, qm, qs, group, G, keys = _random_scoring_case(rng)
        K = len(keys)
        skew = rng.integers(0, 3, (G, K))
        terms = [(int(rng.integers(0, G)), int(rng.integers(0, 2)), int(rng.integers(0, K)),
                  sorted(set(rng.integers(0, G, 2).tolist()))) for _ in range(int(rng.integers(0, 3)))]
        afc, afm = fc.copy(), fm.copy()
        want = affinity_bind_packed(afc, afm, ac, am, labels, qc, qm, qs, group, G, keys, terms, None, skew,
                                    policy=policy)
        pfc, pfm = fc.copy(), fm.copy()
        got = profile_bind_packed(pfc, pfm, ac, am, labels, qc, qm, qs, group, G, keys, terms, None, skew,
                                  policy=policy, hard_affinity_weight=0)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), it
        assert np.array_equal(got[3], want[2]), it
        assert all(np.array_equal(a, b) for a, b in zip(got[4], want[3])), it
        assert np.array_equal(got[2][:, 0], np.where(got[0] >= 0, got[1], 0)) and not got[2][:, 1:].any(), it
        assert np.array_equal(pfc, afc) and np.array_equal(pfm, afm), it


@pytest.mark.parametrize("policy", POLICIES)
def test_j2_one_domain_key(policy):
    """J2: soft spread and preferred terms only on a key every node carries with one domain: the nodes are
    ks_affinity_bind's and each bound pod of a group with soft keys scores 100 * weight_spread more."""
    rng = np.random.default_rng(0x5C2 + policy)
    for it in range(60):
        fc, fm, ac, am, labels, qc, qm, qs, group, G, keys = _random_scoring_case(rng)
        N = len(fc)
        keys = keys + [(np.zeros(N, np.int64), 1)]
        K = len(keys)
        soft = np.zeros((G, K), np.int64)
        soft[:, K - 1] = rng.integers(0, 3, G)
        terms = [(int(rng.integers(0, G)), int(rng.integers(2, 4)), K - 1, [int(rng.integers(0, G))])]
        want = affinity_bind_packed(fc.copy(), fm.copy(), ac, am, labels, qc, qm, qs, group, G, keys, policy=policy)
        got = profile_bind_packed(fc.copy(), fm.copy(), ac, am, labels, qc, qm, qs, group, G, keys, terms,
                                  policy=policy, soft_skew=soft, term_weight=[50])
        assert np.array_equal(got[0], want[0]), it
        has = np.array([g >= 0 and soft[g].any() for g in group]) & (got[0] >= 0)
        assert np.array_equal(got[1], want[1] + 200 * has), it
        assert not got[2][:, 2].any(), it


@pytest.mark.parametrize("policy", POLICIES)
def test_j3_preferred_terms_are_symmetric(policy):
    rng = np.random.default_rng(0x5C3 + policy)
    for it in range(60):
        fc, fm, ac, am, labels, qc, qm, qs, group, G, keys = _random_scoring_case(rng)
        if G < 2:
            continue
        N, K = len(fc), len(keys)
        g, h, k = 0, 1, int(rng.integers(0, K))
        kind, w = int(rng.integers(2, 4)), int(rng.integers(1, 101))
        ex = (rng.integers(0, G, 3), rng.integers(0, N, 3)) if it % 2 else None
        runs = [profile_bind_packed(fc.copy(), fm.copy(), ac, am, labels, qc, qm, qs, group, G, keys, [t], ex,
                                    policy=policy, term_weight=[w])
                for t in ((g, kind, k, [h]), (h, kind, k, [g]))]
        for a, b in zip(*runs):
            if isinstance(a, list):
                assert all(np.array_equal(x, y) for x, y in zip(a, b)), it
            else:
                assert np.array_equal(a, b), it


def test_struct_and_constant_mirrors(ks):
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    assert re.search(r"#define KS_POD_AFFINITY_PREFERRED 2\b", hdr)
    assert re.search(r"#define KS_POD_ANTI_AFFINITY_PREFERRED 3\b", hdr)
    assert (ks.capi.KS_POD_AFFINITY_PREFERRED, ks.capi.KS_POD_ANTI_AFFINITY_PREFERRED) == (PREFERRED, ANTI_PREFERRED)
    fields = ["soft_skew", "soft_all_keys", "term_weight", "hard_affinity_weight", "weight_spread", "weight_affinity"]
    body = re.search(r"typedef struct ks_bind_scoring \{(.*?)\} ks_bind_scoring;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body)
    assert re.findall(r"(\w+);", body) == fields
    assert [f[0] for f in ks.capi.ks_bind_scoring._fields_] == fields
    assert C.sizeof(ks.capi.ks_bind_scoring) == 40  # three pointers, three u32 (+ pad)
    for fn, n_args in (("ks_profile_bind", 14), ("ksh_reconcile_profile", 19)):
        assert fn in ks.declared_symbols() and hasattr(ks.lib, fn), fn
        assert len(getattr(ks.lib, fn).argtypes) == n_args, fn
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    assert re.search(r"pub const KS_POD_AFFINITY_PREFERRED: u8 = 2;", rs)
    assert re.search(r"pub const KS_POD_ANTI_AFFINITY_PREFERRED: u8 = 3;", rs)
    rs_body = re.search(r"pub struct ks_bind_scoring \{(.*?)\}", rs, re.S).group(1)
    assert re.findall(r"pub (\w+):", rs_body) == fields
    for fn in ("ks_profile_bind", "ksh_reconcile_profile"):
        assert re.search(r"pub fn %s\(" % fn, rs), fn


def test_errors_without_a_device(ks):
    """A NULL scoring is refused before the snapshot is looked at (a valid snapshot is not needed to see it); a NULL
    snapshot with a valid scoring is refused too.  ksh_reconcile_profile refuses a NULL scoring the same way, and is
    KS_ERR_NO_DEVICE on a packing-only context."""
    rc_, sel = np.zeros(1, np.int64), np.zeros(1, np.uint64)
    pods = ks.capi.ks_pods(1, rc_.ctypes.data, rc_.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
    grp, dom = np.zeros(1, np.int32), np.zeros(4, np.int32)
    idx = np.empty(1, np.int32)
    sp = ks.capi.ks_spread_multi(1, (C.c_uint32 * 4)(1), (C.c_void_p * 4)(dom.ctypes.data), None, None, None)
    aff = ks.capi.ks_pod_affinity()
    sc = ks.capi.ks_bind_scoring(None, None, None, 1, 2, 2)
    assert ks.lib.ks_profile_bind(None, C.byref(pods), grp.ctypes.data, 1, C.byref(sp), C.byref(aff), None, 4,
                                  idx.ctypes.data, None, None, None, None, None) == ks.capi.KS_ERR_INVALID
    assert "NULL scoring" in ks.lib.ks_last_error().decode()
    assert ks.lib.ks_profile_bind(None, C.byref(pods), grp.ctypes.data, 1, C.byref(sp), C.byref(aff), C.byref(sc), 4,
                                  idx.ctypes.data, None, None, None, None, None) == ks.capi.KS_ERR_INVALID
    assert "NULL scoring" not in ks.lib.ks_last_error().decode()
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        p = arena.pods(g["pods"][:2])
        with pytest.raises(ks.KsError) as e:
            ctx.reconcile_profile(p, 2, [0, -1], 1, ["zone"], [(0, PREFERRED, 0, [0])], [(0, "n0")], term_weight=[5],
                                  soft_skew=[[1]])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
        keys = (C.c_char_p * 1)(b"zone")
        st, nd = np.empty(2, np.int32), np.empty(2, np.int32)
        grp2 = np.zeros(2, np.int32)
        assert ks.lib.ksh_reconcile_profile(ctx._h, C.addressof(p), 2, grp2.ctypes.data, 1, C.cast(keys, C.c_void_p), 1,
                                            None, None, None, None, None, None, 4, st.ctypes.data, nd.ctypes.data,
                                            None, 0, None) == ks.capi.KS_ERR_INVALID
