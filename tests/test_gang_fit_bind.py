"""Gangs when binding (ks_gang_fit_bind), without a device: the restatement in tests/gang_fit_bind_oracle.py against
identities M1-M3 (restated between oracles) on random small clusters, the hand-derived queues of
tests/golden/gv1_gang_fit_bind.json, the C / ctypes / Rust mirrors, and the errors caught without a device."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from fit_bind_oracle import compile_resources, final_free, fit_bind_packed
from gang_fit_bind_oracle import gang_fit_bind_packed, gangs_of, golden_inputs
from test_fit_bind import GPU, _case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = (1, 3, 4)
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "gv1_gang_fit_bind.json")))["cases"]


def random_case(rng):
    """_case's cluster with GPUs on a third of the nodes and GPU requests on some pods, so that gangs come up short."""
    fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, skew, taints, rules = _case(rng)
    N, P = len(fc), len(rc)
    alloc = [{"pods": int(rng.integers(1, 4)), GPU: int(rng.integers(0, 5)) if n % 3 == 0 else 0} for n in range(N)]
    pods = [{GPU: int(rng.integers(1, 3))} if rng.random() < 0.3 else {} for _ in range(P)]
    soft = rng.integers(0, 3, (G, 2))
    return (fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, [{}] * N, taints, rules, alloc, [], pods), \
        dict(max_skew=skew, soft_skew=soft)


def random_cut(rng, P, most=6):
    sizes = []
    while sum(sizes) < P:
        sizes.append(int(min(rng.integers(1, most + 1), P - sum(sizes))))
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)


def fit(args, kw, pods=None):
    """fit_bind_packed over the queue's pods `pods` (all by default) from the initial state; also the charged free[]."""
    fc, fm, ac, am, lab, rc, rm, sel, group = args[:9]
    pods = np.arange(len(rc)) if pods is None else np.asarray(pods, np.int64)
    ofc, ofm = fc.copy(), fm.copy()
    out = fit_bind_packed(ofc, ofm, ac, am, lab, rc[pods], rm[pods], sel[pods], group[pods], *args[9:16],
                          [args[16][p] for p in pods], **kw)
    return out, ofc, ofm


def gang(args, kw, offset, min_member):
    fc, fm = args[0].copy(), args[1].copy()
    out = gang_fit_bind_packed(fc, fm, *args[2:], offset, min_member, **kw)
    return out, fc, fm


def same_walk(a, b):
    (an, asc, ap, ar, acnt, asoft, ause), afc, afm = a
    (bn, bsc, bp, br, bcnt, bsoft, buse), bfc, bfm = b
    for x, y in ((an, bn), (asc, bsc), (ap, bp), (ar, br), (afc, bfc), (afm, bfm)):
        assert np.array_equal(x, y)
    assert all(np.array_equal(x, y) for x, y in zip(acnt + asoft, bcnt + bsoft))
    assert ause.req == buse.req and ause.pods == buse.pods


@pytest.mark.parametrize("policy", POLICIES)
def test_m1_m2_are_fit_bind(policy):
    """M1: every min_member 0 is ks_fit_bind, placed = the gang's bound pods.  M2: singleton gangs with min_member 1."""
    rng = np.random.default_rng(0x6A9F + policy)
    for it in range(8):
        args, kw = random_case(rng)
        kw["policy"] = policy
        P = len(args[5])
        want = fit(args, kw)
        for offset, mm in ((random_cut(rng, P), None), (np.arange(P + 1, dtype=np.uint64), 1)):
            mm = np.zeros(len(offset) - 1, np.uint32) if mm is None else np.ones(len(offset) - 1, np.uint32)
            (*got, placed), fc, fm = gang(args, kw, offset, mm)
            same_walk((tuple(got), fc, fm), want)
            assert placed.tolist() == [int((want[0][0][g] >= 0).sum()) for g in gangs_of(offset)], it


@pytest.mark.parametrize("policy", POLICIES)
def test_m3_committed_subsequence(policy):
    """M3: the committed gangs' pods bind, score and are refused as ks_fit_bind over those pods alone, and the final
    state is that call's; the other pods are unbound with their own turn's refusals."""
    rng = np.random.default_rng(0x6A30 + policy)
    both = [0, 0]
    for it in range(8):
        args, kw = random_case(rng)
        kw["policy"] = policy
        P = len(args[5])
        offset = random_cut(rng, P)
        sizes = np.diff(offset).astype(np.uint32)
        mm = np.minimum(sizes, rng.integers(0, 4, len(sizes))).astype(np.uint32)
        (node, score, parts, refused, cnt, soft, use, placed), fc, fm = gang(args, kw, offset, mm)
        gangs = gangs_of(offset)
        C_ = [p for j, g in enumerate(gangs) if placed[j] >= mm[j] for p in g]
        R_ = [p for j, g in enumerate(gangs) if placed[j] < mm[j] for p in g]
        both[0] += len(C_) > 0
        both[1] += len(R_) > 0
        (wn, ws, wp, wr, wc, wsoft, wuse), wfc, wfm = fit(args, kw, C_)
        assert np.array_equal(node[C_], wn) and np.array_equal(score[C_], ws) and np.array_equal(parts[C_], wp)
        assert np.array_equal(refused[C_], wr), it
        assert all(np.array_equal(x, y) for x, y in zip(cnt + soft, wc + wsoft))
        assert np.array_equal(fc, wfc) and np.array_equal(fm, wfm) and use.req == wuse.req and use.pods == wuse.pods
        assert (node[R_] == -1).all() and not score[R_].any() and not parts[R_].any()
    assert all(both)


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_golden(case):
    args, kw = golden_inputs(case)
    exp = case["expect"]
    (node, score, parts, refused, cnt, soft, use, placed), fc, fm = gang(args, kw, case["gangs"]["offset"],
                                                                        case["gangs"]["min_member"])
    assert node.tolist() == exp["node"] and placed.tolist() == exp["placed"]
    assert refused.tolist() == exp["refused"]
    assert fc.tolist() == exp["free_cpu"]
    names = compile_resources(case["alloc"], [], case["pods"]["res"])[0]
    assert names == ["pods", GPU] and final_free(case["alloc"], use, names).tolist() == exp["free_r"]
    assert [c.tolist() for c in cnt] == exp["counts"]


def test_golden_gpu_gang_is_not_gang_bind():
    """The GPU gang of the first golden case: by cpu and memory alone (ks_gang_bind's view) both workers would take the
    emptier CPU nodes 0 and 1."""
    case = GOLDEN[0]
    args, kw = golden_inputs(case)
    blind = list(args)
    blind[12] = [[]] * len(blind[12])            # no taint
    blind[14] = [{"pods": 110}] * len(blind[14])  # no GPU on any node
    blind[16] = [{}] * len(blind[16])            # no GPU request
    assert fit(tuple(blind), kw)[0][0].tolist() == [0, 1] and case["expect"]["node"] == [2, 3]


def test_struct_and_constant_mirrors(ks):
    assert "ks_gang_fit_bind" in ks.declared_symbols() and hasattr(ks.lib, "ks_gang_fit_bind")
    assert len(ks.lib.ks_gang_fit_bind.argtypes) == 19
    assert ks.lib.ks_gang_fit_bind.argtypes[9]._type_ is ks.capi.ks_gangs
    assert "ksh_reconcile_fit_gangs" in ks.declared_symbols() and hasattr(ks.lib, "ksh_reconcile_fit_gangs")
    assert len(ks.lib.ksh_reconcile_fit_gangs.argtypes) == 24
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    decl = re.search(r"int ks_gang_fit_bind\((.*?)\);", hdr, re.S).group(1)
    assert len(re.sub(r"/\*.*?\*/", "", decl).split(",")) == 19
    hh = open(os.path.join(ROOT, "include", "ksched_host.h")).read()
    decl = re.search(r"int ksh_reconcile_fit_gangs\((.*?)\);", hh, re.S).group(1)
    assert len(re.sub(r"/\*.*?\*/", "", decl).split(",")) == 24


def test_rust_shim_mirror():
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    for fn, n in (("ks_gang_fit_bind", 19), ("ksh_reconcile_fit_gangs", 24)):
        m = re.search(r"pub fn %s\((.*?)\) -> c_int;" % fn, rs, re.S)
        assert m and len([a for a in m.group(1).split(",") if a.strip()]) == n, fn


def test_errors_without_a_device(ks):
    """NULL scoring and NULL gangs are refused before the snapshot is read; a NULL snapshot with both given is
    KS_ERR_INVALID (the gang checks need the queue and run in tests/test_gang_fit_bind_gpu.py)."""
    rc_, sel = np.zeros(1, np.int64), np.zeros(1, np.uint64)
    pods = ks.capi.ks_pods(1, rc_.ctypes.data, rc_.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
    grp, dom = np.zeros(1, np.int32), np.zeros(4, np.int32)
    idx = np.empty(1, np.int32)
    sp = ks.capi.ks_spread_multi(1, (C.c_uint32 * 4)(1), (C.c_void_p * 4)(dom.ctypes.data), None, None, None)
    aff = ks.capi.ks_pod_affinity()
    sc = ks.capi.ks_bind_scoring(None, None, None, 1, 2, 2)
    off, mm = np.array([0, 1], np.uint64), np.ones(1, np.uint32)
    gangs = ks.capi.ks_gangs(1, off.ctypes.data, mm.ctypes.data)
    nulls = (None,) * 8
    assert ks.lib.ks_gang_fit_bind(None, C.byref(pods), grp.ctypes.data, 1, C.byref(sp), C.byref(aff), None, None,
                                   None, C.byref(gangs), 4, idx.ctypes.data, *nulls[:7]) == ks.capi.KS_ERR_INVALID
    assert "NULL scoring" in ks.lib.ks_last_error().decode()
    assert ks.lib.ks_gang_fit_bind(None, C.byref(pods), grp.ctypes.data, 1, C.byref(sp), C.byref(aff), C.byref(sc),
                                   None, None, None, 4, idx.ctypes.data, *nulls[:7]) == ks.capi.KS_ERR_INVALID
    assert "NULL gangs" in ks.lib.ks_last_error().decode()
    assert ks.lib.ks_gang_fit_bind(None, C.byref(pods), grp.ctypes.data, 1, C.byref(sp), C.byref(aff), C.byref(sc),
                                   None, None, C.byref(gangs), 4, idx.ctypes.data, *nulls[:7]) == ks.capi.KS_ERR_INVALID


def test_shapes_are_checked_before_the_call(ks):
    """Snapshot.gang_fit_bind refuses offset and min_member of mismatched lengths with ValueError before any call."""
    snap = ks.Snapshot.__new__(ks.Snapshot)
    snap._h = None
    rc, sel = np.zeros(2, np.int64), np.zeros((2, 0), np.uint64)
    keys = [(np.zeros(0, np.int32), 1)]
    for off, mm in (([0, 2], [1, 1]), ([], []), ([0, 1, 2], [1])):
        with pytest.raises(ValueError):
            snap.gang_fit_bind(rc, rc, sel, np.zeros(2, np.int32), 1, keys, off, mm)
    with pytest.raises(ks.KsError) as e:
        snap.gang_fit_bind(rc, rc, sel, np.zeros(2, np.int32), 1, keys, [0, 2], [1])
    assert e.value.code == ks.capi.KS_ERR_INVALID
