"""Scale-up estimate under the full filter (ks_fit_scaleup_estimate), CPU part: the restatement of
tests/fit_scaleup_oracle.py against the hand-derived cases of tests/golden/gv1_fit_scaleup.json, identity E1 against
scaleup_oracle.scaleup_packed, E2-E6 between restatements, the C / ctypes / Rust mirrors, and the argument errors caught
before any device work."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import fit_scaleup_oracle as fso
from helpers import load_golden
from scaleup_oracle import scaleup_packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = load_golden("gv1_fit_scaleup.json")["cases"]


def e1_want(orc, a, which=None):
    return scaleup_packed(orc, a["alloc_cpu"], a["alloc_mem"], a["free_cpu"], a["free_mem"], a["labels"],
                          a["max_nodes"], a["req_cpu"], a["req_mem"], a["sel"], which)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_cases(case, orc):
    d = fso.golden_problem(case)
    rows, best, node, refused, used = fso.fit_scaleup(d)
    w = case["want"]
    assert [list(r) for r in rows.tolist()] == w["rows"] and best == w["best"]
    assert node.tolist() == w["node"] and refused.tolist() == w["refused"] and used.tolist() == w["used"]
    # what ks_scaleup_estimate, blind to the new filters, makes of the same pods
    srows, sbest = e1_want(orc, fso.to_arrays(d))[:2]
    assert [list(r) for r in srows.tolist()] == case["scaleup_want"]["rows"] and sbest == case["scaleup_want"]["best"]


def test_e1_without_rules_and_resources_is_ks_scaleup_estimate(orc):
    for seed in range(4):
        d = fso.random_problem(np.random.default_rng(seed), 14, 60)
        rows, best, node, refused, _ = fso.fit_scaleup(d, with_rules=False, with_res=False)
        wrows, wbest, wnode, why = e1_want(orc, fso.to_arrays(d))
        assert np.array_equal(rows, wrows) and best == wbest and np.array_equal(node, wnode)
        assert np.array_equal(refused[:, 0], why[:, 2] + why[:, 3]) and not refused[:, 1:].any()


def test_e2_a_copy_of_cpu_changes_nothing():
    for seed in range(4):
        d = fso.random_problem(np.random.default_rng(10 + seed), 14, 60)
        a = fso.fit_scaleup(d)
        e = fso.problem([dict(t, alloc=dict(t["alloc"], **{"cpu-copy": t["fc"]})) for t in d["templates"]],
                        [dict(q, res=dict(q["res"], **{"cpu-copy": q["cpu"]})) for q in d["pods"]], d["group_rules"])
        assert min(q["cpu"] for q in d["pods"]) > 0 and "cpu-copy" in e["names"]
        b = fso.fit_scaleup(e)
        assert all(np.array_equal(x, y) for x, y in zip(a[:4], b[:4]))


def test_e3_no_rule_and_ample_resources_is_e1():
    for seed in range(4):
        d = fso.random_problem(np.random.default_rng(20 + seed), 14, 60)
        total = {n: sum(1 if n == "pods" else q["res"].get(n, 0) for q in d["pods"]) for n in d["names"]}
        e = fso.problem([dict(t, taints=[], alloc={n: total[n] + len(t["ds"]) + sum(r.get(n, 0) for r in t["ds"])
                                                   for n in d["names"]}) for t in d["templates"]],
                        d["pods"], [{} for _ in d["group_rules"]])
        got = fso.fit_scaleup(e)
        want = fso.fit_scaleup(e, with_rules=False, with_res=False)
        assert all(np.array_equal(x, y) for x, y in zip(got[:3], want[:3]))


def replay_ok(d, node):
    """E4: each template's opened nodes hold their pods' summed requests within F and every node_free (zero skip), and
    every placed pod is eligible."""
    a = fso.to_arrays(d)
    for t, tp in enumerate(d["templates"]):
        for o in set(node[t].tolist()) - {-1}:
            ps = np.flatnonzero(node[t] == o)
            if a["req_cpu"][ps].sum() > tp["fc"] or a["req_mem"][ps].sum() > tp["fm"]:
                return False
            s = a["pod_req"][ps].sum(axis=0)
            if ((s > 0) & (s > a["node_free"][:, t])).any():
                return False
            if any(fso.stage(d["pods"][p], tp, d["group_rules"]) != fso.ELIGIBLE for p in ps):
                return False
    return True


def test_e4_replay_e5_words_and_e6_split():
    for seed in range(4):
        d = fso.random_problem(np.random.default_rng(30 + seed), 14, 80, max_nodes=(1, 6))
        rows, best, node, refused, used = fso.fit_scaleup(d)
        assert replay_ok(d, node)
        elig = np.array([[fso.stage(q, tp, d["group_rules"]) == fso.ELIGIBLE for tp in d["templates"]]
                         for q in d["pods"]])
        assert np.array_equal(refused.sum(axis=1) + elig.sum(axis=1), np.full(len(d["pods"]), len(d["templates"])))
        assert np.array_equal(rows["eligible"], elig.sum(axis=0))
        for part in (list(range(0, 14, 2)), list(range(1, 14, 2))):
            got = fso.fit_scaleup(d, which=part)
            assert np.array_equal(got[0][part], rows[part]) and np.array_equal(got[2][part], node[part])


def test_struct_and_prototype_mirrors(ks):
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    decl = re.search(r"int ks_fit_scaleup_estimate\((.*?)\);", hdr, re.S).group(1)
    assert len(re.sub(r"/\*.*?\*/", "", decl, flags=re.S).split(",")) == 12
    assert "ks_fit_scaleup_estimate" in ks.declared_symbols() and hasattr(ks.lib, "ks_fit_scaleup_estimate")
    assert len(ks.lib.ks_fit_scaleup_estimate.argtypes) == 12
    hh = open(os.path.join(ROOT, "include", "ksched_host.h")).read()
    decl = re.search(r"int ksh_scaleup_fit_estimate\((.*?)\);", hh, re.S).group(1)
    assert len(re.sub(r"/\*.*?\*/", "", decl, flags=re.S).split(",")) == 17
    assert len(ks.lib.ksh_scaleup_fit_estimate.argtypes) == 17
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    for name, n in (("ks_fit_scaleup_estimate", 12), ("ksh_scaleup_fit_estimate", 17)):
        m = re.search(rf"pub fn {name}\((.*?)\) -> c_int;", rs, re.S)
        assert m and len(m.group(1).split(",")) == n, name


def test_errors_without_a_device(ks):
    """A NULL snapshot is KS_ERR_INVALID before anything is read (the checks that need a snapshot run in
    tests/test_fit_scaleup_gpu.py); Snapshot.fit_scaleup_estimate refuses misshaped arrays with ValueError first."""
    rc_, sel = np.zeros(1, np.int64), np.zeros(1, np.uint64)
    pods = ks.capi.ks_pods(1, rc_.ctypes.data, rc_.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
    one, mn = np.ones(1, np.int64), np.ones(1, np.uint32)
    tmpl = ks.capi.ks_node_templates(1, 1, one.ctypes.data, one.ctypes.data, one.ctypes.data, one.ctypes.data,
                                     sel.ctypes.data, mn.ctypes.data)
    grp, rows, best = np.zeros(1, np.int32), np.zeros(1, ks.capi.SCALEUP_OPTION_DTYPE), C.c_int32()
    assert ks.lib.ks_fit_scaleup_estimate(None, C.byref(pods), grp.ctypes.data, 1, None, None, C.byref(tmpl),
                                          rows.ctypes.data, C.addressof(best), None, None, None) == ks.capi.KS_ERR_INVALID
    assert "snapshot is NULL" in ks.lib.ks_last_error().decode()
    snap = ks.Snapshot.__new__(ks.Snapshot)
    snap._h = None
    P, T = 3, 2
    rc, sel = np.ones(P, np.int64), np.zeros((P, 1), np.uint64)
    a, lab, m, g = np.ones(T, np.int64), np.zeros((T, 1), np.uint64), np.ones(T, np.uint32), np.zeros(P, np.int32)
    bad = [
        dict(node_free=np.zeros(T, np.int64), pod_req=np.ones((P, 1), np.int64)),  # 1-D node_free
        dict(node_free=np.zeros((1, T + 1), np.int64), pod_req=np.ones((P, 1), np.int64)),  # one template too many
        dict(node_free=np.zeros((2, T), np.int64), pod_req=np.ones((P, 1), np.int64)),  # pod_req short of a column
        dict(node_free=np.zeros((1, T), np.int64), pod_req=np.ones((P - 1, 1), np.int64)),  # one pod short
        dict(node_free=np.zeros((1, T), np.int64), pod_req=None),  # pod_req missing
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            snap.fit_scaleup_estimate(rc, rc, sel, a, a, a, a, lab, m, g, 1, **kw)
    with pytest.raises(ValueError):
        snap.fit_scaleup_estimate(rc, rc, sel, a, a, a, a, lab, m, g[:2], 1)  # group short
    with pytest.raises(ValueError):
        snap.fit_scaleup_estimate(rc, rc, sel, a, a, a[:1], a, lab, m, g, 1)  # free_cpu short
    with pytest.raises(ks.KsError) as e:
        snap.fit_scaleup_estimate(rc, rc, sel, a, a, a, a, lab, m, g, 1)
    assert e.value.code == ks.capi.KS_ERR_INVALID


def test_host_layer_errors_on_a_packing_only_context(ks):
    """ksh_scaleup_fit_estimate: NULL arguments, groups, template taints and rule shapes are refused before the device
    check; a well-formed call on a packing-only context is KS_ERR_NO_DEVICE, and the context is unchanged."""
    lib = ks.lib
    arena = ks.objects.ObjectArena()
    tpl = arena.nodes([{"name": "gpu", "labels": {"node.kubernetes.io/instance-type": "p4d"},
                        "allocatable": {"cpu": "96", "memory": "1024", "pods": "110", "nvidia.com/gpu": "8"}}])
    pods = arena.pods([{"name": f"q{i}", "ns": "w", "containers": [{"cpu": "1", "nvidia.com/gpu": "8"}]}
                       for i in range(2)])
    grp, mn = np.zeros(2, np.int32), np.ones(1, np.uint32)
    rows, best, ref = np.zeros(1, ks.capi.SCALEUP_OPTION_DTYPE), C.c_int32(), np.zeros(8, np.uint32)
    taint = [[{"key": "nvidia.com/gpu", "value": "present", "effect": "NoSchedule"}]]
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        h, T, P = ctx._h, C.addressof(tpl), C.addressof(pods)

        def call(c=h, t=T, m=mn.ctypes.data, p=P, g=grp.ctypes.data, G=1, o=rows.ctypes.data, b=C.addressof(best)):
            return lib.ksh_scaleup_fit_estimate(c, t, 1, m, None, None, None, 0, p, 2, g, G, None, o, b, None,
                                                ref.ctypes.data)

        for bad in (dict(c=None), dict(t=None), dict(m=None), dict(p=None), dict(g=None), dict(o=None), dict(b=None)):
            assert call(**bad) == ks.capi.KS_ERR_INVALID, bad
        assert call(G=0) == ks.capi.KS_ERR_INVALID  # group 0 outside [-1, 0)
        assert call() == ks.capi.KS_ERR_NO_DEVICE
        with pytest.raises(ValueError):
            ctx.scaleup_fit_estimate(tpl, 1, [1], pods, 2, grp, 1, group_rules=[{}, {}])
        with pytest.raises(ValueError):
            ctx.scaleup_fit_estimate(tpl, 1, [1], pods, 2, grp[:1], 1)
        with pytest.raises(ValueError):
            ctx.scaleup_fit_estimate(tpl, 1, [1], pods, 2, grp, 1, template_taints=taint * 2)
        with pytest.raises(ks.KsError) as e:  # a taint without an effect
            ctx.scaleup_fit_estimate(tpl, 1, [1], pods, 2, grp, 1, template_taints=[[{"key": "k", "effect": ""}]])
        assert e.value.code == ks.capi.KS_ERR_INVALID
        with pytest.raises(ks.KsError) as e:  # an unknown requirement operator
            ctx.scaleup_fit_estimate(tpl, 1, [1], pods, 2, grp, 1,
                                     group_rules=[{"required": [[{"key": "k", "operator": "Near", "values": ["a"]}]]}])
        assert e.value.code == ks.capi.KS_ERR_INVALID
        with pytest.raises(ks.KsError) as e:
            ctx.scaleup_fit_estimate(tpl, 1, [1], pods, 2, grp, 1, template_taints=taint,
                                     group_rules=[{"tolerations": [fso.TOL_GPU]}])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
        assert ks.lib.ksh_context_num_nodes(h) == 0
