"""Pod groups (ks_gang_bind / ksh_reconcile_gangs), CPU part: the restatement of tests/gang_oracle.py against its two
special cases (singleton groups = one pod at a time, one group without a minimum = the stream loop) and the hand-derived
GV-1 cases of tests/golden/gv1_gang.json; the no-device status, argument errors caught before any device work, and the
C / ctypes / Rust mirrors of ks_gangs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from gang_oracle import gang_bind_packed, groups, sequential_packed
from helpers import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gv1_packed(ks, orc):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(g["nodes"]), arena.pods(g["bound_pods"]), arena.pods(g["pods"])
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        ctx.set_cluster_pods(bound, len(g["bound_pods"]))
        rc, rm, sel = ctx.pack_pods(pods, len(g["pods"]))
        ac, am, lab, bn, bc, bm = ctx.export_packed()
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    return [p["name"] for p in g["pods"]], ac, am, lab, rc, rm, sel, fc, fm


def gv1_case(names, case):
    """(pod indices into GV-1's pods, offsets, min_member) of a golden case"""
    order = [names.index(p) for grp in case["groups"] for p in grp["pods"]]
    off = np.cumsum([0] + [len(grp["pods"]) for grp in case["groups"]]).astype(np.uint64)
    return np.array(order), off, np.array([grp["min_member"] for grp in case["groups"]], np.uint32)


def _cluster(ks, P, N, seed, scale=1):
    cl = ks.synth.make(P, N, seed=seed, bound_per_node=2)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    fc, fm = cl.free()
    return ac, am, lab, rc * scale, rm * scale, sel, fc, fm


def test_gv1_gang_golden(ks, orc):
    names, ac, am, lab, rc, rm, sel, fc0, fm0 = _gv1_packed(ks, orc)
    assert fc0.tolist() == [4000, 1500, 5500, 0, -100]
    for case in load_golden("gv1_gang.json")["cases"]:
        order, off, mm = gv1_case(names, case)
        fc, fm = fc0.copy(), fm0.copy()
        idx, score, placed, rounds = gang_bind_packed(orc, fc, fm, ac, am, lab, rc[order], rm[order], sel[order], off, mm)
        assert idx.tolist() == case["node_idx"], case["name"]
        assert score.tolist() == case["score"], case["name"]
        assert placed.tolist() == case["placed"] and rounds.tolist() == case["rounds"], case["name"]
        assert fc.tolist() == case["free_cpu"] and fm.tolist() == case["free_mem"], case["name"]


@pytest.mark.parametrize("policy", [0, 1])
def test_singleton_groups_are_one_pod_at_a_time(ks, orc, policy):
    ac, am, lab, rc, rm, sel, fc, fm = _cluster(ks, 400, 60, 9300, scale=4)
    off = np.arange(len(rc) + 1, dtype=np.uint64)
    f1, m1, f2, m2 = fc.copy(), fm.copy(), fc.copy(), fm.copy()
    idx, score, placed, rounds = gang_bind_packed(orc, f1, m1, ac, am, lab, rc, rm, sel, off, np.zeros(len(rc), np.uint32),
                                                  policy)
    s_idx, s_score = sequential_packed(orc, f2, m2, ac, am, lab, rc, rm, sel, policy)
    assert (idx >= 0).sum() > 50 and (idx < 0).sum() > 50  # both outcomes occur
    assert np.array_equal(idx, s_idx) and np.array_equal(score, s_score)
    assert np.array_equal(f1, f2) and np.array_equal(m1, m2)
    assert np.array_equal(placed, (idx >= 0).astype(np.uint32)) and (rounds == 1).all()


@pytest.mark.parametrize("policy", [0, 1])
def test_one_group_without_minimum_is_the_stream_loop(ks, orc, policy):
    ac, am, lab, rc, rm, sel, fc, fm = _cluster(ks, 1024, 80, 9400, scale=3)
    f1, m1, f2, m2 = fc.copy(), fm.copy(), fc.copy(), fm.copy()
    idx, score, placed, rounds = gang_bind_packed(orc, f1, m1, ac, am, lab, rc, rm, sel, np.array([0, 1024], np.uint64),
                                                  np.zeros(1, np.uint32), policy)
    s_idx, s_score, s_rounds = orc.stream_bind_packed(f2, m2, ac, am, lab, rc, rm, sel, policy)
    assert np.array_equal(idx, s_idx) and np.array_equal(score, s_score) and rounds[0] == s_rounds > 1
    assert np.array_equal(f1, f2) and np.array_equal(m1, m2) and placed[0] == (s_idx >= 0).sum()


def test_rolled_back_groups_leave_free_unchanged(ks, orc):
    ac, am, lab, rc, rm, sel, fc, fm = _cluster(ks, 600, 50, 9500, scale=6)
    off = groups(np.random.default_rng(1), len(rc), 5, 40)
    size = np.diff(off).astype(np.uint32)
    f1, m1 = fc.copy(), fm.copy()
    idx, score, placed, rounds = gang_bind_packed(orc, f1, m1, ac, am, lab, rc, rm, sel, off, size)
    committed = placed == size
    assert committed.any() and (~committed).any()
    for g in range(len(size)):
        a, b = int(off[g]), int(off[g + 1])
        assert ((idx[a:b] >= 0).all() if committed[g] else ((idx[a:b] == -1).all() and (score[a:b] == 0).all()))
    # only the committed pods are charged
    ok = idx >= 0
    f2, m2 = fc.copy(), fm.copy()
    np.subtract.at(f2, idx[ok], rc[ok])
    np.subtract.at(m2, idx[ok], rm[ok])
    assert np.array_equal(f1, f2) and np.array_equal(m1, m2)


def test_gang_entry_points_need_a_device(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    nodes, pods = arena.nodes(g["nodes"]), arena.pods(g["pods"])
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        with pytest.raises(ks.KsError) as e:
            ctx.reconcile_gangs(pods, 4, [0, 2, 4], [2, 1])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
    if ks.device_count() == 0:
        with pytest.raises(ks.KsError) as e:
            ks.Snapshot(0)
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
    rc = np.zeros(1, np.int64)
    off = np.array([0, 1], np.uint64)
    mm = np.zeros(1, np.uint32)
    idx = np.zeros(1, np.int32)
    pods1 = ks.capi.ks_pods(1, rc.ctypes.data, rc.ctypes.data, rc.ctypes.data, ks.KS_MEM_HOST)
    gangs = ks.capi.ks_gangs(1, off.ctypes.data, mm.ctypes.data)
    assert ks.lib.ks_gang_bind(None, C.byref(pods1), C.byref(gangs), 0, idx.ctypes.data, None, None,
                               None) == ks.capi.KS_ERR_INVALID


def test_argument_errors_before_device_work(ks):
    lib = ks.lib
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    pods = arena.pods(g["pods"] * 103)  # 1030 pods
    n = len(g["pods"]) * 103
    st = np.zeros(n, np.int32)
    nd = np.zeros(n, np.int32)
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        h, P = ctx._h, C.addressof(pods)

        def call(off, mm, n_pods=4, c=h, p=P):
            off = np.asarray(off, np.uint64)
            mm = np.asarray(mm, np.uint32)
            return lib.ksh_reconcile_gangs(c, p, n_pods, off.ctypes.data, len(off) - 1, mm.ctypes.data, 0,
                                           st.ctypes.data, nd.ctypes.data, None, None, 0, None)

        E = ks.capi
        assert call([0, 2, 4], [2, 2]) == E.KS_ERR_NO_DEVICE  # valid: reaches the device check
        assert call([0, 2, 2, 4], [1, 0, 1]) == E.KS_ERR_RANGE  # an empty group
        assert call([0, 1025], [1], n_pods=1025) == E.KS_ERR_RANGE  # 1025 pods in one group
        assert call([0, 1024, 1025], [1, 1], n_pods=1025) == E.KS_ERR_NO_DEVICE  # 1024 is allowed
        assert call([0, 2, 4], [3, 0]) == E.KS_ERR_RANGE  # min_member above the size
        assert call([1, 2, 4], [1, 1]) == E.KS_ERR_INVALID  # offset[0] != 0
        assert call([0, 3, 2, 4], [0, 0, 0]) == E.KS_ERR_INVALID  # decreasing
        assert call([0, 2, 3], [1, 1]) == E.KS_ERR_INVALID  # does not end at n_pods
        assert call([0, 2, 4], [1, 1], c=None) == E.KS_ERR_INVALID
        assert call([0, 2, 4], [1, 1], p=None) == E.KS_ERR_INVALID
        assert call([0], [], n_pods=0, p=None) == E.KS_ERR_NO_DEVICE


def test_struct_mirrors_c_ctypes_rust(ks):
    cap = ks.capi
    assert C.sizeof(cap.ks_gangs) == 24
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    assert re.search(r"#define KS_GANG_MAX_SIZE (\d+)u", hdr).group(1) == str(cap.KS_GANG_MAX_SIZE) == "1024"
    body = re.search(r"typedef struct ks_gangs \{(.*?)\} ks_gangs;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert re.findall(r"\**([a-z_]+);", body) == [f[0] for f in cap.ks_gangs._fields_]
    hh = open(os.path.join(ROOT, "include", "ksched_host.h")).read()
    assert re.search(r"#define KSH_RECONCILE_GANG_UNSATISFIED (\d+)", hh).group(1) == str(ks.host.KSH_RECONCILE_GANG_UNSATISFIED)
    src = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    body = re.search(r"pub struct ks_gangs \{(.*?)\n\}", src, re.S).group(1)
    assert re.findall(r"pub ([a-z_]+): ([^,]+),", body) == [("n", "u64"), ("offset", "*const u64"),
                                                           ("min_member", "*const u32")]
    assert re.search(r"pub const KS_GANG_MAX_SIZE: u32 = (\d+);", src).group(1) == str(cap.KS_GANG_MAX_SIZE)
    assert re.search(r"pub const KSH_RECONCILE_GANG_UNSATISFIED: c_int = (\d+);", src).group(1) == "4"
    fns = set(re.findall(r"pub fn (ksh?_[a-z0-9_]+)\(", src))
    assert {"ks_gang_bind", "ksh_reconcile_gangs"} <= fns and hasattr(ks.lib, "ks_gang_bind")
    wrapper = open(os.path.join(ROOT, "examples", "rust_shim", "ksched.rs")).read()
    assert "pub fn reconcile_gangs(" in wrapper


def test_group_arrays_must_agree_before_the_call(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    pods = arena.pods(g["pods"])
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        for off, mm in (([0, 2, 4], [1]), ([0, 4], [1, 1]), ([], [])):
            with pytest.raises(ValueError):
                ctx.reconcile_gangs(pods, 4, off, mm)
