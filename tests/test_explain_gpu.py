"""Per-pod rejection counts on the GPU (-m gpu): k_explain_counts through ks_explain / Snapshot.explain and the host
layer's ksh_explain_pods, bit-exact against the CPU oracle (integer counts: no tolerance)."""
import ctypes as C
import functools

import numpy as np
import pytest

from explain_oracle import explain_faithful, explain_packed
from helpers import load_golden

pytestmark = pytest.mark.gpu

W_KEYS = {1: 8, 2: 16, 4: 32, 8: 64}  # label words -> synth n_keys
P_MAX = 100_000


def _sample(P, k=1500):
    """Pods the oracle checks: all of them for small batches, else an even spread incl. both ends."""
    return np.arange(P) if P <= k else np.unique(np.linspace(0, P - 1, k).astype(np.int64))


def _check_invariants(r, n_nodes, cnt=None):
    cpu, mem, res, sel = (r[:, k].astype(np.int64) for k in range(4))
    assert np.all(np.maximum(cpu, mem) <= res) and np.all(res <= cpu + mem)
    if cnt is not None:
        assert np.array_equal(res + sel + np.asarray(cnt, np.int64), np.full(len(r), n_nodes))


@functools.lru_cache(maxsize=4)
def _cluster(ks, W, N):
    cl = ks.synth.make(P_MAX, N, seed=7000 + 13 * W + N, n_keys=W_KEYS[W], bound_per_node=3)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    fc, fm = cl.free()
    return ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm


@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("N", [1, 1023, 1025, 10_007])
def test_explain_matches_packed_oracle(ks, orc, W, N):
    ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm = _cluster(ks, W, N)
    assert lab.shape[1] == W
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        for P in (1, 7, 4096, P_MAX):  # small P splits the node dimension across gridDim.y
            got = snap.explain(rc[:P], rm[:P], sel[:P])
            assert got.shape == (P, 4) and got.dtype == np.uint32
            s = _sample(P)
            want = explain_packed(orc, fc, fm, lab, rc[s], rm[s], sel[s])
            assert np.array_equal(got[s], want), f"W={W} N={N} P={P}"
            cnt = snap.select(rc[:P], rm[:P], sel[:P], flags=ks.KS_SELECT_FORCE_DIRECT).feasible_cnt
            _check_invariants(got, N, cnt)


def test_explain_edge_values(ks, orc):
    LC, LM = 1 << 36, 1 << 55
    ac = np.array([LC, 1000, 1000, 0, LC], np.int64)
    am = np.array([LM, 100, 100, 0, LM], np.int64)
    lab = np.array([[1], [1], [0], [3], [2]], np.uint64)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound([1, 4, 4], [1500, 0, 0], [0, LM, LM])  # node 1: negative cpu, node 4: memory -2^55
        fc, fm = snap.free()
        assert fc[1] == -500 and fm[4] == -LM
        rc = np.array([0, -5, LC, -LC, 1001, 0, 0, LC, 1], np.int64)
        rm = np.array([0, -7, LM, -LM, 0, 101, 0, LM, 1], np.int64)
        never = np.uint64(1) << np.uint64(63)  # a pair no node carries: fails the selector everywhere it fits
        sel = np.array([0, 1, 1, 2, 0, 0, never, 0, never], np.uint64).reshape(-1, 1)
        got = snap.explain(rc, rm, sel)
        assert np.array_equal(got, explain_packed(orc, fc, fm, lab, rc, rm, sel))
        _check_invariants(got, 5, snap.select(rc, rm, sel, flags=ks.KS_SELECT_FORCE_DIRECT).feasible_cnt)
        assert got[6, 3] == 5 - got[6, 2] and got[8, 3] == 5 - got[8, 2]  # never-set pair: every fitting node
        assert snap.explain(rc[:0], rm[:0], sel[:0]).shape == (0, 4)  # P = 0
        # N = 0: nothing counts
        snap.set_nodes(np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 1), np.uint64))
        assert not snap.explain(rc, rm, sel).any()


@pytest.mark.parametrize("path", ["direct", "bitpar"])
def test_invariant_against_select_full_c2(ks, orc, path):
    cl = ks.synth.config("c2")
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    fc, fm = cl.free()
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        flag = ks.KS_SELECT_FORCE_DIRECT if path == "direct" else ks.KS_SELECT_FORCE_BITPAR
        r = snap.select(rc, rm, sel, flags=flag)
        assert snap.last_path() == path
        got = snap.explain(rc, rm, sel)
    _check_invariants(got, cl.N, r.feasible_cnt)
    s = _sample(cl.P, 2000)
    assert np.array_equal(got[s], explain_packed(orc, fc, fm, lab, rc[s], rm[s], sel[s]))


def test_explain_no_node_found_pods_c3(ks, orc):
    cl = ks.synth.config("c3")
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    fc, fm = cl.free()
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        r = snap.select(rc, rm, sel)
        miss = np.nonzero(r.node_idx < 0)[0]
        assert len(miss) >= 1000
        got = snap.explain(rc[miss], rm[miss], sel[miss])
    _check_invariants(got, cl.N, np.zeros(len(miss)))
    s = miss[:1200]
    assert np.array_equal(got[:1200], explain_packed(orc, fc, fm, lab, rc[s], rm[s], sel[s]))


def test_device_pods_and_outputs_on_a_torch_stream(ks, orc):
    import torch
    ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm = _cluster(ks, 2, 1025)
    P = 20_000
    rc, rm, sel = rc[:P], rm[:P], np.ascontiguousarray(sel[:P])
    dev = torch.device("cuda:0")
    t = [torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(dev) for x in (rc, rm, sel)]
    out = torch.full((P, 4), -1, dtype=torch.int32, device=dev)
    h_out = np.full((P, 4), 7, np.uint32)
    st = torch.cuda.Stream()
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        want = snap.explain(rc, rm, sel)
        torch.cuda.synchronize()
        snap.explain_raw(P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, out, ks.KS_MEM_DEVICE, stream=st.cuda_stream)
        st.synchronize()
        assert np.array_equal(out.cpu().numpy().view(np.uint32), want)
        snap.explain_raw(P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, h_out, ks.KS_MEM_HOST, stream=st.cuda_stream)
        assert np.array_equal(h_out, want)  # host output: complete on return
        out.fill_(-1)
        torch.cuda.synchronize()
        snap.explain_raw(P, rc, rm, sel, ks.KS_MEM_HOST, out, ks.KS_MEM_DEVICE)
        assert np.array_equal(out.cpu().numpy().view(np.uint32), want)
    s = _sample(P)
    assert np.array_equal(want[s], explain_packed(orc, fc, fm, lab, rc[s], rm[s], sel[s]))


def test_explain_between_cached_graph_selects(ks, orc):
    """ks_explain (re)allocates staging buffers; a cached CUDA graph of an all-device ks_select must never replay into a
    freed buffer.  Every select is compared with the oracle."""
    import torch
    ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm = _cluster(ks, 1, 1025)
    dev = torch.device("cuda:0")
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        for P in (300, 3000, 30_000, P_MAX):
            o_idx, o_score, o_cnt = orc.run_packed(fc, fm, ac, am, lab, rc[:P], rm[:P], sel[:P], want_mask=False)[:3]
            t = [torch.from_numpy(np.ascontiguousarray(x[:P]).view(np.int64)).to(dev) for x in (rc, rm, sel)]
            idx = torch.empty(P, dtype=torch.int32, device=dev)
            score = torch.empty(P, dtype=torch.int64, device=dev)
            cnt = torch.empty(P, dtype=torch.int32, device=dev)
            for rep in range(3):
                idx.fill_(-7)
                cnt.fill_(-7)
                torch.cuda.synchronize()
                snap.select_raw(P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, idx, score, cnt, ks.KS_MEM_DEVICE)
                torch.cuda.synchronize()
                assert np.array_equal(idx.cpu().numpy(), o_idx), (P, rep)
                assert np.array_equal(score.cpu().numpy(), o_score), (P, rep)
                assert np.array_equal(cnt.cpu().numpy().view(np.uint32), o_cnt), (P, rep)
                n_ex = max(1, P * (rep + 1) // 3)  # grows within and across batch sizes
                why = snap.explain(rc[:n_ex], rm[:n_ex], sel[:n_ex])
                _check_invariants(why, len(ac), o_cnt[:n_ex])


def _gv1_context(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(g["nodes"]), arena.pods(g["bound_pods"]), arena.pods(g["pods"])
    return g, arena, nodes, bound, pods


def test_host_layer_gv1_objects(ks, orc):
    g, arena, nodes, bound, pods = _gv1_context(ks)
    gold = load_golden("gv1_reasons.json")
    oc = orc.Cluster(nodes, len(g["nodes"]), bound, len(g["bound_pods"]))
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        ctx.set_cluster_pods(bound, len(g["bound_pods"]))
        why, msgs = ctx.explain_pods(pods, len(g["pods"]))
    assert np.array_equal(why, np.array(gold["reasons"], np.uint32))
    assert np.array_equal(why, explain_faithful(orc, oc, pods, len(g["pods"])))
    assert msgs[8] == gold["messages"]["p8"]
    assert msgs[:8] == [None] * 8 and msgs[9] is None  # every other GV-1 pod has a feasible node


def test_host_layer_random_objects_and_events(ks, orc):
    cl = ks.synth.make(150, 300, seed=77, n_keys=16, bound_per_node=3)
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    # a pair no node carries, a pod too big for any node, one that fits only where a selector misses
    pods_s += [{"name": "nowhere", "ns": "w", "selector": {"zone": "nowhere"}, "containers": [{"cpu": "1"}]},
               {"name": "huge", "ns": "w", "containers": [{"cpu": "100000", "memory": str(1 << 50)}]}]
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(nodes_s), arena.pods(bound_s), arena.pods(pods_s)
    P = len(pods_s)

    def check(ctx, nodes_now, bound_now):
        oc = orc.Cluster(arena.nodes(nodes_now), len(nodes_now), arena.pods(bound_now), len(bound_now))
        want = explain_faithful(orc, oc, pods, P)
        why, msgs = ctx.explain_pods(pods, P)
        assert np.array_equal(why, want)
        cnt = oc.run(pods, P, want_mask=False)[2]
        _check_invariants(why, len(nodes_now), cnt)
        for i in range(P):
            assert msgs[i] == (ks.host.format_unschedulable(len(nodes_now), why[i])[1] if cnt[i] == 0 else None), i
        return why, msgs

    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, cl.N)
        ctx.set_cluster_pods(bound, cl.B)
        why, msgs = check(ctx, nodes_s, bound_s)
        assert why[P - 2, 3] == cl.N - why[P - 2, 2] and msgs[P - 2] is not None
        assert msgs[P - 1] == f"0/{cl.N} nodes are available: {cl.N} Insufficient cpu, {cl.N} Insufficient memory."
        # events: a pod lands on node 0 (capacity charged), node 1's allocatable changes
        extra = {"name": "late", "ns": "load", "node_name": "node-0", "containers": [{"cpu": "64", "memory": str(1 << 38)}]}
        ctx.pod_bound(arena.pods([extra]))
        bound_s = bound_s + [extra]
        check(ctx, nodes_s, bound_s)
        changed = dict(nodes_s[1], allocatable={"cpu": "1", "memory": "1024"})
        ctx.upsert_node(arena.nodes([changed]))
        nodes_s = [nodes_s[0], changed] + nodes_s[2:]
        check(ctx, nodes_s, bound_s)


def test_bad_arguments_are_status_codes(ks):
    lib = ks.lib
    rc = np.zeros(4, np.int64)
    sel = np.zeros(4, np.uint64)
    out = np.zeros((4, 4), np.uint32)
    with ks.Snapshot(0) as snap:
        snap.set_nodes([1000], [1000], np.zeros((1, 1), np.uint64))
        pods = ks.capi.ks_pods(4, rc.ctypes.data, rc.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
        assert lib.ks_explain(None, C.byref(pods), out.ctypes.data, ks.KS_MEM_HOST, None) == -1
        assert lib.ks_explain(snap._h, None, out.ctypes.data, ks.KS_MEM_HOST, None) == -1
        assert lib.ks_explain(snap._h, C.byref(pods), None, ks.KS_MEM_HOST, None) == -1
        assert lib.ks_explain(snap._h, C.byref(pods), out.ctypes.data, 7, None) == -1
        bad_space = ks.capi.ks_pods(4, rc.ctypes.data, rc.ctypes.data, sel.ctypes.data, 5)
        assert lib.ks_explain(snap._h, C.byref(bad_space), out.ctypes.data, ks.KS_MEM_HOST, None) == -1
        too_many = ks.capi.ks_pods(1 << 32, rc.ctypes.data, rc.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
        assert lib.ks_explain(snap._h, C.byref(too_many), out.ctypes.data, ks.KS_MEM_HOST, None) == -5
        empty = ks.capi.ks_pods(0, None, None, None, ks.KS_MEM_HOST)
        assert lib.ks_explain(snap._h, C.byref(empty), None, ks.KS_MEM_HOST, None) == 0
        assert lib.ks_explain(snap._h, C.byref(pods), out.ctypes.data, ks.KS_MEM_HOST, None) == 0
        assert out[:, 2].tolist() == [0, 0, 0, 0] and out[:, 3].tolist() == [0, 0, 0, 0]
    with ks.host.Context(0) as ctx:
        assert lib.ksh_explain_pods(ctx._h, None, 3, out.ctypes.data, None, 0, None) == -1
        assert lib.ksh_explain_pods(None, None, 0, None, None, 0, None) == -1
