"""Priority preemption (ks_preempt / ksh_preempt_pods), CPU part: the restatement of tests/preempt_oracle.py against the
hand-derived plans of tests/golden/gv1_preempt.json and against consistency checks of its own, the no-device status,
argument errors caught before any device work, and the C / ctypes / Rust mirrors of the two structs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from helpers import load_golden
from preempt_oracle import ROW_DTYPE, crowded, preempt_packed

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
    return ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm


def _check_row(row, vic, want, max_victims):
    assert int(row["node_idx"]) == want["node_idx"]
    assert int(row["n_victims"]) == len(want["victims"])
    assert vic.tolist() == want["victims"] + [-1] * (max_victims - len(want["victims"]))
    for f in ("candidates", "max_victim_priority", "victim_priority_sum"):
        assert int(row[f]) == want[f], f
    assert int(row["reserved"]) == 0


def test_gv1_preempt_golden(ks, orc):
    gold = load_golden("gv1_preempt.json")["gv1"]
    ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm = _gv1_packed(ks, orc)
    assert bn.tolist() == [1, 2, 2, 3, 4]  # b1, b2a, b2b, b3, b4: the stray pod names no node
    p, mv = gold["pod"], gold["max_victims"]
    assert (rc[p], rm[p], fc[2]) == (5501, 0, 5500)
    for case in gold["cases"]:
        rows, vic = preempt_packed(orc, fc, fm, ac, am, lab, rc[p:p + 1], rm[p:p + 1], sel[p:p + 1],
                                   [case["priority"]], bn, bc, bm, gold["bound_priority"], mv)
        _check_row(rows[0], vic[0], case, mv)
        assert int(rows[0]["feasible_cnt"]) == case["feasible_cnt"]
    # every other GV-1 pod fits somewhere: no plan and no candidates whatever its priority
    rows, vic = preempt_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, np.full(len(rc), 10**6), bn, bc, bm,
                               gold["bound_priority"], mv)
    fits = rows["feasible_cnt"] > 0
    assert fits.sum() == len(rc) - 1 and np.all(rows["node_idx"][fits] == -1) and np.all(rows["candidates"][fits] == 0)


def _rules(gold):
    r = gold["rules"]
    n = len(r["alloc_cpu"])
    ac, am = np.array(r["alloc_cpu"], np.int64), np.array(r["alloc_mem"], np.int64)
    lab = np.array(r["labels"], np.uint64).reshape(n, 1)
    bn = np.array(r["bound_node"], np.int32)
    bc = np.array(r["bound_cpu"], np.int64)
    bm = np.zeros(len(bn), np.int64)
    bp = np.array(r["bound_priority"], np.int32)
    pods = r["pods"]
    rc = np.array([q["req_cpu"] for q in pods], np.int64)
    rm = np.zeros(len(pods), np.int64)
    sel = np.array([q["sel"] for q in pods], np.uint64).reshape(-1, 1)
    pp = np.array([q["priority"] for q in pods], np.int32)
    return ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp, pods, r["max_victims"]


def test_node_choice_rules_golden(ks, orc):
    ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp, pods, mv = _rules(load_golden("gv1_preempt.json"))
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    rows, vic = preempt_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, pp, bn, bc, bm, bp, mv)
    for i, want in enumerate(pods):
        _check_row(rows[i], vic[i], want, mv)
    rows, vic = preempt_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, pp, bn, bc, bm, bp, 1)
    assert rows["node_idx"].tolist() == [1, -1, 4, 6, -1]  # two victims are over a cap of one


def test_restatement_consistency(ks, orc):
    """Without the restatement's own walk: evicting a plan's victims makes the cell fit, putting any one back (requests
    are non-negative here) makes it fail again, victims have lower priority and sit on the chosen node."""
    ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp = crowded(ks, 400, 300, 9100)
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    rows, vic = preempt_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, pp, bn, bc, bm, bp, 16)
    planned = np.nonzero(rows["node_idx"] >= 0)[0]
    assert len(planned) > 20 and (rows["candidates"][planned] >= 1).all()
    for p in planned:
        n, v = rows["node_idx"][p], vic[p][: rows["n_victims"][p]]
        assert (bn[v] == n).all() and (bp[v] < pp[p]).all() and (vic[p][len(v):] == -1).all()
        assert rows["max_victim_priority"][p] == bp[v].max()
        assert rows["victim_priority_sum"][p] == int((bp[v].astype(np.int64) + (1 << 31)).sum())
        c, m = fc[n] + bc[v].sum(), fm[n] + bm[v].sum()
        assert rc[p] <= c and rm[p] <= m
        for b in v:
            assert rc[p] > c - bc[b] or rm[p] > m - bm[b]


def test_preempt_entry_points_need_a_device(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(g["nodes"]), arena.pods(g["bound_pods"]), arena.pods(g["pods"])
    prio = np.zeros(len(g["pods"]), np.int32)
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        ctx.set_cluster_pods(bound, len(g["bound_pods"]))
        ctx.set_pod_priorities(bound, np.arange(len(g["bound_pods"])), len(g["bound_pods"]))  # host-only: works
        with pytest.raises(ks.KsError) as e:
            ctx.preempt_pods(pods, len(g["pods"]), prio, 4)
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
    if ks.device_count() == 0:
        with pytest.raises(ks.KsError) as e:
            ks.Snapshot(0)
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
    rc = np.zeros(1, np.int64)
    out = np.zeros(1, ks.capi.PREEMPTION_DTYPE)
    pods1 = ks.capi.ks_pods(1, rc.ctypes.data, rc.ctypes.data, rc.ctypes.data, ks.KS_MEM_HOST)
    bound0 = ks.capi.ks_bound_pods(0, None, None, None, None)
    assert ks.lib.ks_preempt(None, C.byref(pods1), rc.ctypes.data, C.byref(bound0), 4, out.ctypes.data, None,
                             ks.KS_MEM_HOST, None) == ks.capi.KS_ERR_INVALID


def test_argument_errors_before_device_work(ks):
    lib = ks.lib
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    pods = arena.pods(g["pods"])
    prio = np.zeros(4, np.int32)
    out = np.zeros(4, ks.capi.PREEMPTION_DTYPE)
    off = np.zeros(4, np.int64)
    buf = C.create_string_buffer(64)
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        h, P = ctx._h, C.addressof(pods)

        def call(c=h, p=P, n=4, pr=prio.ctypes.data, mv=4, o=out.ctypes.data):
            return lib.ksh_preempt_pods(c, p, n, pr, mv, o, C.addressof(buf), 64, off.ctypes.data)

        assert call(mv=0) == ks.capi.KS_ERR_RANGE and call(mv=129) == ks.capi.KS_ERR_RANGE
        assert call(c=None) == -1 and call(p=None) == -1 and call(pr=None) == -1 and call(o=None) == -1
        assert call(n=0, p=None, pr=None, o=None, mv=0) == ks.capi.KS_ERR_RANGE
        assert call(mv=128) == ks.capi.KS_ERR_NO_DEVICE and call(mv=1) == ks.capi.KS_ERR_NO_DEVICE
        assert lib.ksh_context_set_pod_priorities(None, P, prio.ctypes.data, 1) == -1
        assert lib.ksh_context_set_pod_priorities(h, None, prio.ctypes.data, 1) == -1
        assert lib.ksh_context_set_pod_priorities(h, P, None, 1) == -1
        assert lib.ksh_context_set_pod_priorities(h, P, prio.ctypes.data, 4) == 0  # unknown pods: ignored
        assert lib.ksh_context_set_pod_priorities(h, None, None, 0) == 0


def test_struct_mirrors_c_ctypes_numpy_rust(ks):
    cap = ks.capi
    assert C.sizeof(cap.ks_preemption) == 32 and cap.PREEMPTION_DTYPE.itemsize == 32
    assert [f[0] for f in cap.ks_preemption._fields_] == list(cap.PREEMPTION_DTYPE.names) == list(ROW_DTYPE.names)
    for name in cap.PREEMPTION_DTYPE.names:
        assert getattr(cap.ks_preemption, name).offset == cap.PREEMPTION_DTYPE.fields[name][1]
        assert cap.PREEMPTION_DTYPE.fields[name][0] == ROW_DTYPE.fields[name][0]
    assert C.sizeof(cap.ks_bound_pods) == 40
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    assert re.search(r"#define KS_PREEMPT_MAX_VICTIMS (\d+)u", hdr).group(1) == str(cap.KS_PREEMPT_MAX_VICTIMS)
    for struct, fields in (("ks_preemption", cap.ks_preemption._fields_), ("ks_bound_pods", cap.ks_bound_pods._fields_)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), hdr, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        assert re.findall(r"\**([a-z_]+);", body) == [f[0] for f in fields], struct
    src = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    rust_ty = {C.c_int32: "i32", C.c_uint32: "u32", C.c_int64: "i64", C.c_uint64: "u64"}
    body = re.search(r"pub struct ks_preemption \{(.*?)\n\}", src, re.S).group(1)
    assert re.findall(r"pub ([a-z_]+): ([a-z0-9]+),", body) == [(n, rust_ty[t]) for n, t in cap.ks_preemption._fields_]
    body = re.search(r"pub struct ks_bound_pods \{(.*?)\n\}", src, re.S).group(1)
    assert [n for n, _ in re.findall(r"pub ([a-z_]+): ([^,]+),", body)] == [f[0] for f in cap.ks_bound_pods._fields_]
    assert re.search(r"pub const KS_PREEMPT_MAX_VICTIMS: u32 = (\d+);", src).group(1) == str(cap.KS_PREEMPT_MAX_VICTIMS)
    fns = set(re.findall(r"pub fn (ksh?_[a-z0-9_]+)\(", src))
    names = {"ks_preempt", "ksh_preempt_pods", "ksh_context_set_pod_priorities"}
    assert names <= fns and all(hasattr(ks.lib, n) for n in names)
    wrapper = open(os.path.join(ROOT, "examples", "rust_shim", "ksched.rs")).read()
    assert "pub fn preempt(&self, pod: &corev1::Pod, priority: i32, max_victims: u32)" in wrapper
