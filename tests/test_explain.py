"""Per-pod rejection counts (ks_explain / ksh_explain_pods), CPU part: the packed oracle against the faithful oracle
and the hand-derived GV-1 counts, the FailedScheduling message format, and the Rust shim's struct mirror."""
import numpy as np
import pytest

from explain_oracle import explain_faithful, explain_packed
from helpers import load_golden


def _gv1(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    return g, arena, arena.nodes(g["nodes"]), arena.pods(g["bound_pods"]), arena.pods(g["pods"])


def _invariants(r, n_nodes):
    cpu, mem, res, sel = (r[:, k].astype(np.int64) for k in range(4))
    assert np.all(np.maximum(cpu, mem) <= res) and np.all(res <= cpu + mem)
    assert np.all(res + sel <= n_nodes)


def test_gv1_reasons_golden_packed_and_faithful(ks, orc):
    g, arena, nodes, bound, pods = _gv1(ks)
    want = np.array(load_golden("gv1_reasons.json")["reasons"], np.uint32)
    oc = orc.Cluster(nodes, len(g["nodes"]), bound, len(g["bound_pods"]))
    assert np.array_equal(explain_faithful(orc, oc, pods, len(g["pods"])), want)
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        ctx.set_cluster_pods(bound, len(g["bound_pods"]))
        rc, rm, sel = ctx.pack_pods(pods, len(g["pods"]))
        ac, am, lab, bn, bc, bm = ctx.export_packed()
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    got = explain_packed(orc, fc, fm, lab, rc, rm, sel)
    assert np.array_equal(got, want)
    # feasible_cnt of the argmax path closes the sum to N
    cnt = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, want_mask=False)[2]
    assert np.array_equal(got[:, 2] + got[:, 3] + cnt, np.full(len(g["pods"]), len(g["nodes"])))


@pytest.mark.parametrize("n_keys", [8, 16, 32, 64])  # W = 1, 2, 4, 8
def test_packed_oracle_equals_faithful_oracle(ks, orc, n_keys):
    cl = ks.synth.make(60, 150, seed=4100 + n_keys, n_keys=n_keys, bound_per_node=3)
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    arena = ks.objects.ObjectArena()
    oc = orc.Cluster(arena.nodes(nodes_s), cl.N, arena.pods(bound_s), cl.B)
    want = explain_faithful(orc, oc, arena.pods(pods_s), cl.P)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    assert lab.shape[1] == {8: 1, 16: 2, 32: 4, 64: 8}[n_keys]
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    got = explain_packed(orc, fc, fm, lab, rc, rm, sel)
    assert np.array_equal(got, want)
    _invariants(got, cl.N)
    assert got[:, 3].any() and got[:, 2].any()  # both kinds of rejection occur
    cnt = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, want_mask=False)[2]
    assert np.array_equal(got[:, 2] + got[:, 3] + cnt, np.full(cl.P, cl.N))


def test_format_unschedulable(ks):
    f = ks.host.format_unschedulable
    assert f(5, [5, 1, 5, 0]) == (67, "0/5 nodes are available: 5 Insufficient cpu, 1 Insufficient memory.")
    assert f(3, [0, 0, 0, 3])[1] == "0/3 nodes are available: 3 node(s) didn't match Pod's node affinity/selector."
    assert f(7, [2, 0, 2, 0])[1] == "0/7 nodes are available: 2 Insufficient cpu."
    assert f(9, [4, 3, 5, 4])[1] == ("0/9 nodes are available: 4 Insufficient cpu, 3 Insufficient memory, "
                                     "4 node(s) didn't match Pod's node affinity/selector.")
    assert f(0, [0, 0, 0, 0]) == (24, "0/0 nodes are available.")
    full = "0/5 nodes are available: 5 Insufficient cpu, 1 Insufficient memory."
    n, text = f(5, [5, 1, 5, 0], cap=10)  # too small: truncated and NUL-terminated, full length returned
    assert n == len(full) and text == full[:9]
    assert f(5, [5, 1, 5, 0], cap=0) == (len(full), "")  # size query
    assert ks.lib.ksh_format_unschedulable(5, None, None, 0) == -1  # KS_ERR_INVALID: no counts


def test_explain_entry_points_need_a_device(ks):
    g, arena, nodes, bound, pods = _gv1(ks)
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        with pytest.raises(ks.KsError) as e:
            ctx.explain_pods(pods, len(g["pods"]))
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE


def test_rust_shim_pod_reasons_mirror(ks):
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "examples", "rust_shim", "ksched_sys.rs")).read()
    body = re.search(r"pub struct ks_pod_reasons \{(.*?)\n\}", src, re.S).group(1)
    assert re.findall(r"pub ([a-z_0-9]+): u32", body) == [f[0] for f in ks.capi.ks_pod_reasons._fields_]
    fns = set(re.findall(r"pub fn (ksh?_[a-z0-9_]+)\(", src))
    assert {"ks_explain", "ksh_explain_pods", "ksh_format_unschedulable"} <= fns
