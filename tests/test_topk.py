"""Ranked candidates (ks_select_topk / ksh_rank_nodes), CPU part: the packed restatement against the faithful one, entry 0
against the oracle's argmax, the hand-derived GV-1 rankings, the no-device status, and the Rust shim's bindings."""
import ctypes as C

import numpy as np
import pytest

from helpers import load_golden
from topk_oracle import topk_faithful, topk_packed

POLICIES = {0: "leftover", 1: "least_allocated"}


def _gv1(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    return g, arena, arena.nodes(g["nodes"]), arena.pods(g["bound_pods"]), arena.pods(g["pods"])


def _check_entry0(orc, got, fc, fm, ac, am, lab, rc, rm, sel, policy):
    idx, score, cnt = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, policy=policy, want_mask=False)[:3]
    assert np.array_equal(got[0][:, 0], idx) and np.array_equal(got[1][:, 0], score) and np.array_equal(got[2], cnt)


@pytest.mark.parametrize("policy", [0, 1])
def test_gv1_topk_golden_packed_and_faithful(ks, orc, policy):
    g, arena, nodes, bound, pods = _gv1(ks)
    gold = load_golden("gv1_topk.json")
    want_idx = np.array(gold[POLICIES[policy]]["node_idx"], np.int32)
    want_score = np.array(gold[POLICIES[policy]]["score"], np.int64)
    k = gold["k"]
    if policy == 0:
        assert want_idx[0].tolist() == [2, 0, 1, 3, -1]  # p0 (feasible 11110): n2 > n0 > n1 > n3
    oc = orc.Cluster(nodes, len(g["nodes"]), bound, len(g["bound_pods"]))
    f_idx, f_score, f_cnt = topk_faithful(orc, oc, pods, len(g["pods"]), k, policy)
    assert np.array_equal(f_idx, want_idx) and np.array_equal(f_score, want_score)
    assert f_cnt.tolist() == [r.count("1") for r in g["expected_feasible_rows"]]
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        ctx.set_cluster_pods(bound, len(g["bound_pods"]))
        rc, rm, sel = ctx.pack_pods(pods, len(g["pods"]))
        ac, am, lab, bn, bc, bm = ctx.export_packed()
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    got = topk_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, k, policy)
    assert np.array_equal(got[0], want_idx) and np.array_equal(got[1], want_score)
    _check_entry0(orc, got, fc, fm, ac, am, lab, rc, rm, sel, policy)


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("n_keys", [8, 16, 32, 64])  # W = 1, 2, 4, 8
def test_packed_topk_equals_faithful_topk(ks, orc, n_keys, policy):
    cl = ks.synth.make(60, 150, seed=4300 + n_keys, n_keys=n_keys, bound_per_node=3)
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    arena = ks.objects.ObjectArena()
    oc = orc.Cluster(arena.nodes(nodes_s), cl.N, arena.pods(bound_s), cl.B)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    assert lab.shape[1] == {8: 1, 16: 2, 32: 4, 64: 8}[n_keys]
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    for k in (1, 5, 32):
        want = topk_faithful(orc, oc, arena.pods(pods_s), cl.P, k, policy)
        got = topk_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, k, policy)
        for a, b in zip(got, want):
            assert np.array_equal(a, b), (k, policy)
        _check_entry0(orc, got, fc, fm, ac, am, lab, rc, rm, sel, policy)
        filled = (got[0] >= 0).sum(axis=1)  # every row fills min(k, feasible_cnt) slots
        assert np.array_equal(filled, np.minimum(got[2], k))
    assert (got[2] > 5).any() and (got[2] < 32).any()


def test_topk_entry_points_need_a_device(ks):
    g, arena, nodes, bound, pods = _gv1(ks)
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        with pytest.raises(ks.KsError) as e:
            ctx.rank_nodes(pods, len(g["pods"]), 3)
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
    if ks.device_count() == 0:  # no snapshot can exist without a GPU, so the core entry only sees a NULL handle
        with pytest.raises(ks.KsError) as e:
            ks.Snapshot(0)
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
    rc = np.zeros(1, np.int64)
    out = np.zeros(4, np.int32)
    pods1 = ks.capi.ks_pods(1, rc.ctypes.data, rc.ctypes.data, rc.ctypes.data, ks.KS_MEM_HOST)
    assert ks.lib.ks_select_topk(None, C.byref(pods1), 0, 4, out.ctypes.data, None, None, ks.KS_MEM_HOST, None) == -1


def test_rust_shim_binds_topk(ks):
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "examples", "rust_shim", "ksched_sys.rs")).read()
    fns = set(re.findall(r"pub fn (ksh?_[a-z0-9_]+)\(", src))
    assert {"ks_select_topk", "ksh_rank_nodes"} <= fns
    assert all(hasattr(ks.lib, n) for n in ("ks_select_topk", "ksh_rank_nodes"))
    assert re.search(r"pub const KS_TOPK_MAX: u32 = (\d+);", src).group(1) == str(ks.capi.KS_TOPK_MAX)
    wrapper = open(os.path.join(root, "examples", "rust_shim", "ksched.rs")).read()
    assert "pub fn rank_nodes(&self, pod: &corev1::Pod, k: u32) -> Result<Vec<(String, i64)>, i32>" in wrapper
