"""Drain simulation (ks_drain_check / ksh_drain_nodes), CPU part: the restatement of tests/drain_oracle.py against the
hand-derived GV-1 cases of tests/golden/gv1_drain.json and against its two special cases (a one-pod candidate is one
select with the node removed; a fully placed candidate is one pod at a time on the cluster without the node); argument
errors caught before any device work, the no-device status, and the C / ctypes / Rust mirrors of ks_drain_candidates."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from drain_oracle import SENTINEL, bound_candidates, drain_packed
from gang_oracle import sequential_packed
from helpers import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gv1_packed(ks, orc):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    specs = g["bound_pods"] + g["pods"]
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        ctx.set_cluster_pods(arena.pods(g["bound_pods"]), len(g["bound_pods"]))
        rc, rm, sel = ctx.pack_pods(arena.pods(specs), len(specs))
        ac, am, lab, bn, bc, bm = ctx.export_packed()
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    return [p["name"] for p in specs], ac, am, lab, rc, rm, sel, fc, fm


def _cluster(ks, P, N, seed):
    cl = ks.synth.make(P, N, seed=seed, bound_per_node=3)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    fc, fm = cl.free()
    return ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm


def test_gv1_drain_golden(ks, orc):
    names, ac, am, lab, rc, rm, sel, fc, fm = _gv1_packed(ks, orc)
    assert fc.tolist() == [4000, 1500, 5500, 0, -100]
    for case in load_golden("gv1_drain.json")["cases"]:
        pick = [names.index(p) for c in case["candidates"] for p in c["pods"]]
        node = [c["node"] for c in case["candidates"]]
        off = np.cumsum([0] + [len(c["pods"]) for c in case["candidates"]]).astype(np.uint64)
        for policy, key in ((0, "leftover"), (1, "least_allocated")):
            f1, m1 = fc.copy(), fm.copy()
            placed, idx, score = drain_packed(orc, f1, m1, ac, am, lab, rc[pick], rm[pick], sel[pick], node, off, policy,
                                              case["exclude_candidates"])
            want = case[key]
            assert placed.tolist() == want["placed"], (case["name"], key)
            assert idx.tolist() == want["node_idx"] and score.tolist() == want["score"], (case["name"], key)
            assert np.array_equal(f1, fc) and np.array_equal(m1, fm)  # nothing is charged


@pytest.mark.parametrize("policy", [0, 1])
def test_one_pod_candidate_is_select_without_the_node(ks, orc, policy):
    ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm = _cluster(ks, 300, 50, 24000 + policy)
    rc, rm = rc * 4, rm * 4
    P = len(rc)
    node = np.arange(P, dtype=np.int32) % 50
    off = np.arange(P + 1, dtype=np.uint64)
    placed, idx, score = drain_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, node, off, policy)
    for p in range(P):
        f1, m1 = fc.copy(), fm.copy()
        f1[node[p]] = m1[node[p]] = SENTINEL
        i, s, _, _, _ = orc.run_packed(f1, m1, ac, am, lab, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1], policy, want_mask=False)
        assert (idx[p], score[p], placed[p]) == (i[0], s[0], int(i[0] >= 0))
    assert (placed == 1).sum() > 50 and (placed == 0).sum() > 50


@pytest.mark.parametrize("policy", [0, 1])
def test_placed_candidate_is_one_pod_at_a_time_without_the_node(ks, orc, policy):
    """On the cluster with the candidate's node taken out (its columns deleted), gang_oracle.sequential_packed gives the
    same nodes (renumbered) and scores."""
    ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm = _cluster(ks, 200, 60, 24100 + policy)
    order, node, off = bound_candidates(bn, 60)
    prc, prm, psel = bc[order], bm[order], sel[np.arange(len(order)) % len(sel)]
    placed, idx, score = drain_packed(orc, fc, fm, ac, am, lab, prc, prm, psel, node, off, policy)
    size = np.diff(off)
    full = np.nonzero((placed == size) & (size > 0))[0]
    assert len(full) > 10
    for d in full:
        keep = np.arange(60) != d
        a, b = int(off[d]), int(off[d + 1])
        i, s = sequential_packed(orc, fc[keep].copy(), fm[keep].copy(), ac[keep], am[keep], lab[keep], prc[a:b], prm[a:b],
                                 psel[a:b], policy)
        assert np.array_equal(np.nonzero(keep)[0][i], idx[a:b]) and np.array_equal(s, score[a:b])


def test_exclude_candidates_removes_every_listed_node(ks, orc):
    ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm = _cluster(ks, 400, 40, 24200)
    order, node, off = bound_candidates(bn, 40)
    prc, prm, psel = bc[order], bm[order], np.zeros((len(order), lab.shape[1]), np.uint64)
    pick = np.sort(np.argsort(-(fc * (1 << 22) + fm), kind="stable")[:4])  # the nodes with the most left over
    sub_off = np.concatenate([[0], np.cumsum(np.diff(off)[pick])]).astype(np.uint64)
    pods = np.concatenate([np.arange(int(off[d]), int(off[d + 1])) for d in pick])
    _, idx, _ = drain_packed(orc, fc, fm, ac, am, lab, prc[pods], prm[pods], psel[pods], node[pick], sub_off, 0, True)
    assert not set(idx.tolist()) & set(pick.tolist())
    _, idx0, _ = drain_packed(orc, fc, fm, ac, am, lab, prc[pods], prm[pods], psel[pods], node[pick], sub_off, 0, False)
    assert set(idx0.tolist()) & set(pick.tolist())  # without the flag the others are destinations


def test_drain_entry_points_need_a_device(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        with pytest.raises(ks.KsError) as e:
            ctx.drain_nodes(["n2"], arena.pods(g["bound_pods"][1:3]), [0, 2])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
    rc = np.zeros(1, np.int64)
    node = np.zeros(1, np.int32)
    off = np.array([0, 1], np.uint64)
    out = np.zeros(1, np.int32)
    placed = np.zeros(1, np.uint32)
    pods1 = ks.capi.ks_pods(1, rc.ctypes.data, rc.ctypes.data, rc.ctypes.data, ks.KS_MEM_HOST)
    cand = ks.capi.ks_drain_candidates(1, node.ctypes.data, off.ctypes.data)
    assert ks.lib.ks_drain_check(None, C.byref(pods1), C.byref(cand), 0, 0, placed.ctypes.data, out.ctypes.data,
                                 None) == ks.capi.KS_ERR_INVALID


def test_host_layer_argument_errors_before_device_work(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    bound = arena.pods(g["bound_pods"])  # b1@n1, b2a@n2, b2b@n2, b3@n3, b4@n4, stray@not-a-node
    E = ks.capi
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))

        def code(names, off, pods=bound, flags=0):
            with pytest.raises(ks.KsError) as e:
                ctx.drain_nodes(names, pods, off, 0, flags)
            return e.value.code, str(e.value)

        assert code(["n1", "n2"], [0, 1, 3])[0] == E.KS_ERR_NO_DEVICE  # well grouped: reaches the device check
        assert code(["n1", "n0"], [0, 1, 3], flags=1)[0] == E.KS_ERR_INVALID  # b2a is on n2, not n0
        c, msg = code(["n1", "n0"], [0, 1, 3])
        assert "spec.nodeName" in msg and "n2" in msg
        c, msg = code(["n1", "nx"], [0, 1, 1])
        assert c == E.KS_ERR_INVALID and "nx" in msg  # unknown name, even without pods
        assert code(["not-a-node"], [5, 6])[0] == E.KS_ERR_INVALID  # offset[0] != 0
        assert code(["n1", "n2"], [0, 3, 1])[0] == E.KS_ERR_INVALID  # decreasing
        unbound = arena.pods(g["pods"][:1])
        c, msg = code(["n1"], [0, 1], pods=unbound)
        assert c == E.KS_ERR_INVALID and "p0" in msg  # a pending pod is bound nowhere
        assert code([], [0], pods=None)[0] == E.KS_ERR_NO_DEVICE
        with pytest.raises(ValueError):
            ctx.drain_nodes(["n1"], bound, [0, 1, 2])


def test_struct_mirrors_c_ctypes_rust(ks):
    cap = ks.capi
    assert C.sizeof(cap.ks_drain_candidates) == 24
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    assert re.search(r"#define KS_DRAIN_MAX_PODS (\d+)u", hdr).group(1) == str(cap.KS_DRAIN_MAX_PODS) == "1024"
    assert re.search(r"#define KS_DRAIN_EXCLUDE_CANDIDATES (\d+)u", hdr).group(1) == str(cap.KS_DRAIN_EXCLUDE_CANDIDATES)
    body = re.search(r"typedef struct ks_drain_candidates \{(.*?)\} ks_drain_candidates;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert re.findall(r"\**([a-z_]+);", body) == [f[0] for f in cap.ks_drain_candidates._fields_]
    src = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    body = re.search(r"pub struct ks_drain_candidates \{(.*?)\n\}", src, re.S).group(1)
    assert re.findall(r"pub ([a-z_]+): ([^,]+),", body) == [("n", "u64"), ("node_idx", "*const i32"),
                                                           ("offset", "*const u64")]
    assert re.search(r"pub const KS_DRAIN_MAX_PODS: u32 = (\d+);", src).group(1) == str(cap.KS_DRAIN_MAX_PODS)
    assert re.search(r"pub const KS_DRAIN_EXCLUDE_CANDIDATES: u32 = (\d+);", src).group(1) == "1"
    fns = set(re.findall(r"pub fn (ksh?_[a-z0-9_]+)\(", src))
    assert {"ks_drain_check", "ksh_drain_nodes"} <= fns and hasattr(ks.lib, "ks_drain_check")
    wrapper = open(os.path.join(ROOT, "examples", "rust_shim", "ksched.rs")).read()
    assert "pub fn drain_nodes(" in wrapper
