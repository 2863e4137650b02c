"""Ranked candidates on the GPU (-m gpu): k_select_topk / k_topk_combine through ks_select_topk / Snapshot.select_topk and
the host layer's ksh_rank_nodes, bit-exact against the CPU restatement of tests/topk_oracle.py and against ks_select."""
import ctypes as C
import functools

import numpy as np
import pytest

from helpers import load_golden
from topk_oracle import topk_faithful, topk_packed

pytestmark = pytest.mark.gpu

W_KEYS = {1: 8, 2: 16, 4: 32, 8: 64}  # label words -> synth n_keys
P_MAX = 100_000
KS = (1, 2, 5, 32)


def _sample(P, k=300):
    """Pods the oracle checks: all of them for small batches, else an even spread incl. both ends."""
    return np.arange(P) if P <= k else np.unique(np.linspace(0, P - 1, k).astype(np.int64))


@functools.lru_cache(maxsize=4)
def _cluster(ks, W, N):
    cl = ks.synth.make(P_MAX, N, seed=8100 + 13 * W + N, n_keys=W_KEYS[W], bound_per_node=3)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    fc, fm = cl.free()
    return ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm


def _check(got, want, k, rows=None, what=""):
    """got = (idx, score, cnt) of the GPU, want = the oracle at k >= this k (a ranking's prefix is the smaller ranking)."""
    g_idx, g_score, g_cnt = got if rows is None else (got[0][rows], got[1][rows], got[2][rows])
    assert g_idx.shape[1] == k and g_idx.dtype == np.int32 and g_score.dtype == np.int64
    assert np.array_equal(g_idx, want[0][:, :k]), what
    assert np.array_equal(g_score, want[1][:, :k]), what
    assert np.array_equal(g_cnt, want[2]), what


@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("N", [1, 1023, 1025, 10_007])
def test_topk_matches_packed_oracle(ks, orc, W, N):
    ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm = _cluster(ks, W, N)
    assert lab.shape[1] == W
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        for policy in (ks.KS_SCORE_LEFTOVER, ks.KS_SCORE_LEAST_ALLOCATED):
            s_all = _sample(P_MAX)
            want_all = topk_packed(orc, fc, fm, ac, am, lab, rc[s_all], rm[s_all], sel[s_all], 32, policy)
            for P in (1, 7, 4096, P_MAX):  # small P splits the node dimension across gridDim.y
                s = _sample(P)
                want = topk_packed(orc, fc, fm, ac, am, lab, rc[s], rm[s], sel[s], 32, policy) if P < P_MAX else want_all
                for k in KS:
                    got = snap.select_topk(rc[:P], rm[:P], sel[:P], k, policy)
                    _check(got, want, k, s, f"W={W} N={N} P={P} k={k} policy={policy}")


def _select_agrees(ks, snap, rc, rm, sel, got, policy, flags):
    r = snap.select(rc, rm, sel, policy=policy, flags=flags)
    assert np.array_equal(got[0][:, 0], r.node_idx) and np.array_equal(got[1][:, 0], r.score)
    assert np.array_equal(got[2], r.feasible_cnt)
    return r


@pytest.mark.parametrize("policy", [0, 1])
def test_ties_and_rising_scores(ks, orc, policy):
    """Tie-heavy: no bound load, so the free values take only the 36 allocatable shapes and equal scores are decided by
    the node index, inside a chunk and across chunks.  Rising: scores grow with the node index, so every feasible node
    is a candidate when it is scanned (the worst case of the insertion)."""
    N = 5000
    cl = ks.synth.make(4096, N, seed=8800, bound_per_node=0, selectors=False)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    rising_c = (1000 + np.arange(N, dtype=np.int64) * 7)
    rising_m = (1 << 30) + np.arange(N, dtype=np.int64) * 4096
    for name, (a_c, a_m) in {"ties": (ac, am), "rising": (rising_c, rising_m)}.items():
        with ks.Snapshot(0) as snap:
            snap.set_nodes(a_c, a_m, lab)
            fc, fm = snap.free()
            req_c, req_m = (rc, rm) if name == "ties" else (rc % 5000, rm % (1 << 29))
            for P in (3, 4096):
                want = topk_packed(orc, fc, fm, a_c, a_m, lab, req_c[:P], req_m[:P], sel[:P], 32, policy)
                if name == "ties":
                    assert (want[1][:, :-1] == want[1][:, 1:]).any()  # ties inside the lists
                for k in KS:
                    got = snap.select_topk(req_c[:P], req_m[:P], sel[:P], k, policy)
                    _check(got, want, k, None, f"{name} P={P} k={k}")
                    _select_agrees(ks, snap, req_c[:P], req_m[:P], sel[:P], got, policy, ks.KS_SELECT_FORCE_DIRECT)
            if name == "rising" and policy == 0:
                assert np.all(np.diff(want[0][want[0][:, 1] >= 0][:, :2], axis=1) < 0)  # best is the highest index


def test_topk_edge_values(ks, orc):
    LC, LM = 1 << 36, 1 << 55
    ac = np.array([LC, 1000, 1000, 0, LC], np.int64)
    am = np.array([LM, 100, 100, 0, LM], np.int64)
    lab = np.array([[1], [1], [0], [3], [2]], np.uint64)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound([1, 4, 4], [1500, 0, 0], [0, LM, LM])  # node 1: negative cpu, node 4: memory -2^55
        fc, fm = snap.free()
        rc = np.array([0, -5, LC, -LC, 1001, 0, 0, LC, 1], np.int64)
        rm = np.array([0, -7, LM, -LM, 0, 101, 0, LM, 1], np.int64)
        never = np.uint64(1) << np.uint64(63)  # a pair no node carries
        sel = np.array([0, 1, 1, 2, 0, 0, never, 0, never], np.uint64).reshape(-1, 1)
        for policy in (0, 1):
            want = topk_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, 32, policy)
            for k in (1, 3, 5, 32):  # k > feasible count everywhere from 5 on
                _check(snap.select_topk(rc, rm, sel, k, policy), want, k, None, f"k={k} policy={policy}")
            assert np.all(want[0][6] == -1) and np.all(want[0][8] == -1)  # never-set bit: nothing is feasible
        idx, score, cnt = snap.select_topk(rc[:0], rm[:0], sel[:0], 4)  # P = 0
        assert idx.shape == (0, 4) and cnt.shape == (0,)
        # N = 0: every slot empty
        snap.set_nodes(np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 1), np.uint64))
        idx, score, cnt = snap.select_topk(rc, rm, sel, 7)
        assert np.all(idx == -1) and not score.any() and not cnt.any()


@pytest.mark.parametrize("policy", [0, 1])
def test_entry0_equals_select_full_c2(ks, orc, policy):
    cl = ks.synth.config("c2")
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    fc, fm = cl.free()
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        got = snap.select_topk(rc, rm, sel, 8, policy)
        paths = (ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR) if policy == 0 else (ks.KS_SELECT_AUTO,)
        for flags in paths:
            _select_agrees(ks, snap, rc, rm, sel, got, policy, flags)
            if flags == ks.KS_SELECT_FORCE_BITPAR:
                assert snap.last_path() == "bitpar"
    s = _sample(cl.P, 400)
    _check(got, topk_packed(orc, fc, fm, ac, am, lab, rc[s], rm[s], sel[s], 8, policy), 8, s)


def test_device_pods_and_outputs_on_a_torch_stream(ks, orc):
    import torch
    ac, am, lab, bn, bc, bm, rc, rm, sel, fc, fm = _cluster(ks, 2, 1025)
    P, k = 20_000, 5
    rc, rm, sel = rc[:P], rm[:P], np.ascontiguousarray(sel[:P])
    dev = torch.device("cuda:0")
    t = [torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(dev) for x in (rc, rm, sel)]
    idx = torch.full((P, k), -7, dtype=torch.int32, device=dev)
    score = torch.full((P, k), -7, dtype=torch.int64, device=dev)
    cnt = torch.full((P,), -7, dtype=torch.int32, device=dev)
    st = torch.cuda.Stream()
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        want = snap.select_topk(rc, rm, sel, k, 1)
        torch.cuda.synchronize()
        snap.select_topk_raw(P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, k, idx, score, cnt, ks.KS_MEM_DEVICE, policy=1,
                             stream=st.cuda_stream)
        st.synchronize()
        assert np.array_equal(idx.cpu().numpy(), want[0]) and np.array_equal(score.cpu().numpy(), want[1])
        assert np.array_equal(cnt.cpu().numpy().view(np.uint32), want[2])
        h_idx = np.full((P, k), 9, np.int32)
        snap.select_topk_raw(P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, k, h_idx, None, None, ks.KS_MEM_HOST, policy=1,
                             stream=st.cuda_stream)
        assert np.array_equal(h_idx, want[0])  # host output: complete on return; score and count skipped
        idx.fill_(-7)
        torch.cuda.synchronize()
        snap.select_topk_raw(P, rc, rm, sel, ks.KS_MEM_HOST, k, idx, None, None, ks.KS_MEM_DEVICE, policy=1)
        assert np.array_equal(idx.cpu().numpy(), want[0])
    s = _sample(P)
    _check(want, topk_packed(orc, fc, fm, ac, am, lab, rc[s], rm[s], sel[s], k, 1), k, s)


def test_topk_between_cached_graph_selects(ks, orc):
    """ks_select_topk (re)allocates staging and partial buffers; a cached CUDA graph of an all-device ks_select must
    never replay into a freed buffer.  Every select is compared with the oracle."""
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
                n_tk = max(1, P * (rep + 1) // 3)  # grows within and across batch sizes
                k = (1, 8, 32)[rep]
                t_idx, t_score, t_cnt = snap.select_topk(rc[:n_tk], rm[:n_tk], sel[:n_tk], k)
                assert np.array_equal(t_idx[:, 0], o_idx[:n_tk]) and np.array_equal(t_score[:, 0], o_score[:n_tk])
                assert np.array_equal(t_cnt, o_cnt[:n_tk])


def test_host_layer_gv1_objects(ks, orc):
    g = load_golden("gv1.json")
    gold = load_golden("gv1_topk.json")
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(g["nodes"]), arena.pods(g["bound_pods"]), arena.pods(g["pods"])
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        ctx.set_cluster_pods(bound, len(g["bound_pods"]))
        n_bound = ctx.num_bound
        for rep in range(2):  # ranking charges nothing: the second pass sees the same capacity
            for policy, name in ((0, "leftover"), (1, "least_allocated")):
                idx, score, cnt = ctx.rank_nodes(pods, len(g["pods"]), gold["k"], policy)
                assert idx.tolist() == gold[name]["node_idx"] and score.tolist() == gold[name]["score"], (rep, name)
                assert cnt.tolist() == [r.count("1") for r in g["expected_feasible_rows"]]
        assert [ctx.node_name(i) for i in idx[0] if i >= 0] == ["n0", "n1", "n2", "n3"]  # least_allocated row of p0
        assert ctx.num_bound == n_bound


def test_host_layer_random_objects_and_events(ks, orc):
    cl = ks.synth.make(150, 300, seed=78, n_keys=16, bound_per_node=3)
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    pods_s += [{"name": "nowhere", "ns": "w", "selector": {"zone": "nowhere"}, "containers": [{"cpu": "1"}]}]
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(nodes_s), arena.pods(bound_s), arena.pods(pods_s)
    P = len(pods_s)

    def check(ctx, nodes_now, bound_now):
        oc = orc.Cluster(arena.nodes(nodes_now), len(nodes_now), arena.pods(bound_now), len(bound_now))
        for policy in (0, 1):
            want = topk_faithful(orc, oc, pods, P, 32, policy)
            for k in (1, 6, 32):
                _check(ctx.rank_nodes(pods, P, k, policy), want, k, None, f"k={k} policy={policy}")
            sel_idx, sel_score, _ = ctx.select_nodes(pods, P, policy)
            assert np.array_equal(sel_idx, want[0][:, 0]) and np.array_equal(sel_score, want[1][:, 0])
        assert np.all(want[0][P - 1] == -1)

    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, cl.N)
        ctx.set_cluster_pods(bound, cl.B)
        check(ctx, nodes_s, bound_s)
        # events: a pod lands on node 0 (capacity charged), node 1's allocatable changes, node 2 goes away
        extra = {"name": "late", "ns": "load", "node_name": "node-0", "containers": [{"cpu": "64", "memory": str(1 << 38)}]}
        ctx.pod_bound(arena.pods([extra]))
        bound_s = bound_s + [extra]
        check(ctx, nodes_s, bound_s)
        changed = dict(nodes_s[1], allocatable={"cpu": "1", "memory": "1024"})
        ctx.upsert_node(arena.nodes([changed]))
        nodes_s = [nodes_s[0], changed] + nodes_s[2:]
        check(ctx, nodes_s, bound_s)
        ctx.remove_node(nodes_s[2]["name"])
        gone = nodes_s[2]["name"]
        nodes_s = nodes_s[:2] + nodes_s[3:]
        check(ctx, nodes_s, [b for b in bound_s if b.get("node_name") != gone])


def test_bad_arguments_are_status_codes(ks):
    lib = ks.lib
    rc = np.zeros(4, np.int64)
    sel = np.zeros(4, np.uint64)
    idx = np.zeros(4 * 32, np.int32)
    with ks.Snapshot(0) as snap:
        snap.set_nodes([1000], [1000], np.zeros((1, 1), np.uint64))
        h = snap._h
        pods = ks.capi.ks_pods(4, rc.ctypes.data, rc.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
        H = ks.KS_MEM_HOST

        def call(k=3, policy=0, out=idx.ctypes.data, space=H, p=pods, s=h):
            return lib.ks_select_topk(s, C.byref(p) if p is not None else None, policy, k, out, None, None, space, None)

        assert call(k=0) == -5 and call(k=33) == -5  # KS_ERR_RANGE
        assert call(k=32) == 0 and call(k=1) == 0
        assert call(out=None) == -1 and call(policy=2) == -1 and call(policy=-1) == -1 and call(space=7) == -1
        assert call(s=None) == -1 and call(p=None) == -1
        bad_space = ks.capi.ks_pods(4, rc.ctypes.data, rc.ctypes.data, sel.ctypes.data, 5)
        assert call(p=bad_space) == -1
        empty = ks.capi.ks_pods(0, None, None, None, H)
        assert call(p=empty, out=None) == 0  # P = 0 does nothing
        assert call(p=empty, k=0) == -5
        assert call() == 0 and idx[:12].reshape(4, 3).tolist() == [[0, -1, -1]] * 4
    with ks.host.Context(0) as ctx:
        assert lib.ksh_rank_nodes(ctx._h, None, 3, 0, 4, idx.ctypes.data, None, None) == -1
        assert lib.ksh_rank_nodes(None, None, 0, 0, 4, None, None, None) == -1
        assert lib.ksh_rank_nodes(ctx._h, None, 0, 0, 0, None, None, None) == -5
        assert lib.ksh_rank_nodes(ctx._h, None, 0, 0, 33, None, None, None) == -5
        assert lib.ksh_rank_nodes(ctx._h, None, 0, 0, 4, None, None, None) == 0
