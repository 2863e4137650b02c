"""Preemption under the full filter (ks_fit_preempt), CPU part: the restatement of tests/fit_preempt_oracle.py against
the hand-derived plans of tests/golden/gv1_fit_preempt.json, identities Q1, Q2, Q4 and Q5 between restatements, the C /
ctypes / Rust mirrors, and the argument errors caught before any device work."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import fit_preempt_oracle as fpo
from helpers import load_golden
from preempt_oracle import crowded, preempt_packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = load_golden("gv1_fit_preempt.json")["cases"]


def _row(rows, vic, unres, p):
    return dict(node_idx=int(rows["node_idx"][p]), victims=[int(v) for v in vic[p] if v >= 0],
                candidates=int(rows["candidates"][p]), feasible_cnt=int(rows["feasible_cnt"][p]),
                max_victim_priority=int(rows["max_victim_priority"][p]),
                victim_priority_sum=int(rows["victim_priority_sum"][p]), unresolvable=int(unres[p]))


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_plans(case, orc):
    d = fpo.golden_case(case)
    rows, vic, unres = fpo.run(d, case["max_victims"])
    assert _row(rows, vic, unres, 0) == case["want"]
    assert int(rows["n_victims"][0]) == len(case["want"]["victims"]) and int(rows["reserved"][0]) == 0
    # what ks_preempt, blind to the new filters, makes of the same pod
    prow, _ = preempt_packed(orc, d["fc"], d["fm"], d["ac"], d["am"], d["labels"], d["rc"], d["rm"], d["sel"], d["prio"],
                             d["bn"], d["bc"], d["bm"], d["bp"], case["max_victims"])
    assert {k: int(prow[k][0]) for k in case["preempt_want"]} == case["preempt_want"]


def _q1_inputs(ks, seed, full_range):
    levels = (None, None) if full_range else ((0, 100, 1000), (0, 100, 1000, 5000))
    ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp = crowded(ks, 60, 40, seed, prio_levels=levels[0], pod_levels=levels[1])
    fc, fm = ac.copy(), am.copy()
    np.subtract.at(fc, bn, bc)
    np.subtract.at(fm, bn, bm)
    bound = [(int(n), int(c), int(m), int(p), {}) for n, c, m, p in zip(bn, bc, bm, bp)]
    return ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp, fc, fm, bound


@pytest.mark.parametrize("full_range", [False, True])
def test_q1_without_rules_and_resources_is_ks_preempt(ks, orc, full_range):
    for seed in range(3):
        ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp, fc, fm, bound = _q1_inputs(ks, seed, full_range)
        N, P = len(ac), len(rc)
        for mv in (1, 3, 128):
            want, wv = preempt_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, pp, bn, bc, bm, bp, mv)
            rows, vic, unres = fpo.fit_preempt_packed(fc, fm, lab, rc, rm, sel, pp, np.full(P, -1), [{}] * N, [[]] * N,
                                                      [], None, bound, [{}] * P, mv)
            assert all(np.array_equal(rows[f], want[f]) for f in want.dtype.names) and np.array_equal(vic, wv)
            miss = ((sel[:, None, :] & ~lab[None, :, :]) != 0).any(axis=2).sum(axis=1)
            assert np.array_equal(unres, miss)
        assert (want["node_idx"] >= 0).sum() > 0


def test_q2_a_copy_of_cpu_changes_nothing():
    for seed in range(4):
        d = fpo.random_cluster(np.random.default_rng(seed), 40, 30, 3)
        a = fpo.run(d, 3)
        e = dict(d)
        e["alloc"] = [dict(m, **{"cpu-copy": int(c)}) for m, c in zip(d["alloc"], d["ac"])]
        e["bound"] = [(n, c, m, p, dict(r, **{"cpu-copy": c})) for n, c, m, p, r in d["bound"]]
        e["pod_res"] = [dict(r, **{"cpu-copy": int(c)}) for r, c in zip(d["pod_res"], d["rc"])]
        assert (d["rc"] > 0).all()
        b = fpo.run(e, 3)
        assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_q4_q5_evict_then_bind_and_put_back():
    """Q4: with a plan's victims evicted the pod fits the planned node (which is resolvable); Q5: with any one of them
    put back it does not."""
    plans = 0
    for seed in range(6):
        d = fpo.random_cluster(np.random.default_rng(100 + seed), 30, 25, 4, full_range=seed % 2 == 1)
        rows, vic, unres = fpo.run(d, 128)
        for p in np.nonzero(rows["node_idx"] >= 0)[0]:
            n, v = int(rows["node_idx"][p]), [int(x) for x in vic[p] if x >= 0]
            assert all(d["bound"][b][0] == n for b in v)
            assert fpo.fits_after(d, p, n, v) and not fpo.fits_after(d, p, n, [])
            for b in v:
                assert not fpo.fits_after(d, p, n, [x for x in v if x != b])
            plans += 1
    assert plans > 20


def test_max_victims_caps_the_plan():
    d = fpo.random_cluster(np.random.default_rng(7), 40, 40, 3, per_node=8)
    wide, wv, _ = fpo.run(d, 128)
    for mv in (1, 3):
        rows, vic, _ = fpo.run(d, mv)
        assert (rows["n_victims"] <= mv).all()
        same = (wide["node_idx"] >= 0) & (wide["candidates"] == rows["candidates"]) & (rows["node_idx"] >= 0)
        assert np.array_equal(rows["node_idx"][same], wide["node_idx"][same])
        assert np.array_equal(vic[same], wv[same][:, :mv])
    assert (wide["n_victims"] > 3).any()


def test_struct_and_prototype_mirrors(ks):
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    decl = re.search(r"int ks_fit_preempt\((.*?)\);", hdr, re.S).group(1)
    assert len(re.sub(r"/\*.*?\*/", "", decl, flags=re.S).split(",")) == 13
    assert "ks_fit_preempt" in ks.declared_symbols() and hasattr(ks.lib, "ks_fit_preempt")
    assert len(ks.lib.ks_fit_preempt.argtypes) == 13
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    m = re.search(r"pub fn ks_fit_preempt\((.*?)\) -> c_int;", rs, re.S)
    assert m and len(m.group(1).split(",")) == 13


def test_errors_without_a_device(ks):
    """A NULL snapshot is KS_ERR_INVALID before anything is read (the other checks need a snapshot and run in
    tests/test_fit_preempt_gpu.py); Snapshot.fit_preempt refuses wrongly shaped arrays with ValueError first."""
    rc_, sel = np.zeros(1, np.int64), np.zeros(1, np.uint64)
    pods = ks.capi.ks_pods(1, rc_.ctypes.data, rc_.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
    grp, prio = np.zeros(1, np.int32), np.zeros(1, np.int32)
    out = np.zeros(1, ks.capi.PREEMPTION_DTYPE)
    b = ks.capi.ks_bound_pods(0, None, None, None, None)
    assert ks.lib.ks_fit_preempt(None, C.byref(pods), grp.ctypes.data, 1, None, None, prio.ctypes.data, C.byref(b), None,
                                 4, out.ctypes.data, None, None) == ks.capi.KS_ERR_INVALID
    assert "snapshot is NULL" in ks.lib.ks_last_error().decode()
    snap = ks.Snapshot.__new__(ks.Snapshot)
    snap._h = None  # N = 0
    P, B = 3, 2
    rc, sel = np.zeros(P, np.int64), np.zeros((P, 0), np.uint64)
    args = (rc, rc, sel, np.zeros(P, np.int32), np.zeros(P, np.int32), 1, np.zeros(B, np.int32), np.zeros(B, np.int64),
            np.zeros(B, np.int64), np.zeros(B, np.int32), 4)
    bad = [
        (np.zeros(0, np.int64), np.ones((P, 1), np.int64), np.ones((B, 1), np.int64)),  # 1-D node_free
        (np.zeros((1, 5), np.int64), np.ones((P, 1), np.int64), np.ones((B, 1), np.int64)),  # 5 columns, 0 nodes
        (np.zeros((2, 0), np.int64), np.ones((P, 1), np.int64), np.ones((B, 2), np.int64)),  # pod_req short
        (np.zeros((1, 0), np.int64), np.ones((P - 1, 1), np.int64), np.ones((B, 1), np.int64)),  # one pod short
        (np.zeros((1, 0), np.int64), np.ones((P, 1), np.int64), np.ones((B + 1, 1), np.int64)),  # bound_req long
        (np.zeros((1, 0), np.int64), np.ones((P, 1), np.int64), np.ones(B, np.int64)),  # 1-D bound_req
        (np.zeros((1, 0), np.int64), np.ones((P, 1), np.int64), None),  # bound_req missing
    ]
    for nf, pr, br in bad:
        with pytest.raises(ValueError):
            snap.fit_preempt(*args, node_free=nf, pod_req=pr, bound_req=br)
    with pytest.raises(ValueError):
        snap.fit_preempt(rc, rc, sel, np.zeros(P - 1, np.int32), *args[4:])  # priority short
    with pytest.raises(ks.KsError) as e:
        snap.fit_preempt(*args, node_free=np.zeros((1, 0), np.int64), pod_req=np.ones((P, 1), np.int64),
                         bound_req=np.ones((B, 1), np.int64))
    assert e.value.code == ks.capi.KS_ERR_INVALID


def test_host_layer_errors_on_a_packing_only_context(ks):
    """ksh_preempt_fit_pods: NULL arguments, max_victims, groups and group_rules shapes are refused before the device
    check; a well-formed call on a packing-only context is KS_ERR_NO_DEVICE."""
    lib = ks.lib
    arena = ks.objects.ObjectArena()
    pods = arena.pods([{"name": f"q{i}", "ns": "w", "containers": [{"cpu": "1", "nvidia.com/gpu": "8"}]}
                       for i in range(3)])
    prio, grp = np.full(3, 1000, np.int32), np.zeros(3, np.int32)
    out = np.zeros(3, ks.capi.PREEMPTION_DTYPE)
    off = np.zeros(3, np.int64)
    buf = C.create_string_buffer(64)
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes([{"name": "a", "allocatable": {"cpu": "4", "memory": "1024", "pods": "4"}}]), 1)
        h, P = ctx._h, C.addressof(pods)

        def call(c=h, p=P, n=3, g=grp.ctypes.data, G=1, pr=prio.ctypes.data, mv=4, o=out.ctypes.data):
            return lib.ksh_preempt_fit_pods(c, p, n, g, G, None, pr, mv, o, C.addressof(buf), 64, off.ctypes.data)

        assert call(mv=0) == ks.capi.KS_ERR_RANGE and call(mv=129) == ks.capi.KS_ERR_RANGE
        for bad in (dict(c=None), dict(p=None), dict(g=None), dict(pr=None), dict(o=None)):
            assert call(**bad) == ks.capi.KS_ERR_INVALID, bad
        assert call(G=0) == ks.capi.KS_ERR_INVALID  # group 0 outside [-1, 0)
        assert call() == ks.capi.KS_ERR_NO_DEVICE and call(mv=128) == ks.capi.KS_ERR_NO_DEVICE
        with pytest.raises(ValueError):
            ctx.preempt_fit_pods(pods, 3, grp, 1, prio, 4, group_rules=[{}, {}])
        with pytest.raises(ValueError):
            ctx.preempt_fit_pods(pods, 3, grp[:2], 1, prio, 4)
        with pytest.raises(ks.KsError) as e:
            ctx.preempt_fit_pods(pods, 3, grp, 1, prio, 4, group_rules=[{}])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
