"""Priority preemption on the GPU (-m gpu): the victim index, k_preempt_scan and k_preempt_emit through ks_preempt /
Snapshot.preempt and the host layer's ksh_preempt_pods, bit-exact against the CPU restatement of tests/preempt_oracle.py,
plus consistency checks that do not rely on it."""
import functools

import numpy as np
import pytest

from helpers import load_golden
from preempt_oracle import INT32_MAX, INT32_MIN, crowded, preempt_packed

pytestmark = pytest.mark.gpu

W_KEYS = {1: 8, 2: 16, 4: 32, 8: 64}  # label words -> synth n_keys
P_MAX = 100_000
FIELDS = ("node_idx", "n_victims", "candidates", "feasible_cnt", "max_victim_priority", "reserved", "victim_priority_sum")


def _sample(P, k=200):
    return np.arange(P) if P <= k else np.unique(np.linspace(0, P - 1, k).astype(np.int64))


def _check(got, want, rows=None, what=""):
    """got / want = (rows, victims); rows = indices of got that want describes (None = all)."""
    g_rows, g_vic = got if rows is None else (got[0][rows], got[1][rows])
    for f in FIELDS:
        assert np.array_equal(g_rows[f], want[0][f]), (f, what)
    assert np.array_equal(g_vic, want[1]), ("victims", what)


@functools.lru_cache(maxsize=2)
def _cluster(ks, W, N, full_range):
    levels = None if full_range else (0, 100, 1000)
    return crowded(ks, P_MAX, N, 7700 + 13 * W + N, n_keys=W_KEYS[W], prio_levels=levels,
                   pod_levels=None if full_range else (0, 100, 1000, 5000))


def _oracle(orc, c, pods, mv):
    ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp = c
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    return preempt_packed(orc, fc, fm, ac, am, lab, rc[pods], rm[pods], sel[pods], pp[pods], bn, bc, bm, bp, mv)


@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("N", [1, 1023, 1025, 10_007])
def test_preempt_matches_restatement(ks, orc, W, N):
    for full_range in (False, True):  # three tie-heavy levels; the whole int32 range
        c = _cluster(ks, W, N, full_range)
        ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp = c
        assert lab.shape[1] == W
        samples = {P: _sample(P) for P in (1, 7, 4096, P_MAX)}
        union = np.unique(np.concatenate(list(samples.values())))
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            snap.set_bound(bn, bc, bm)
            for mv in (1, 3, 128):
                want = _oracle(orc, c, union, mv)
                where = {int(p): i for i, p in enumerate(union)}
                if mv == 3 and N > 1:
                    assert (want[0]["node_idx"] >= 0).sum() > 20, "the workload must produce plans"
                for P, s in samples.items():  # small P splits the node dimension across gridDim.y
                    got = snap.preempt(rc[:P], rm[:P], sel[:P], pp[:P], bn, bc, bm, bp, mv)
                    idx = [where[int(p)] for p in s]
                    _check(got, (want[0][idx], want[1][idx]), s, f"W={W} N={N} P={P} mv={mv} full={full_range}")


def _edge_run(ks, orc, ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp, mv=8):
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        fc, fm = snap.free()
        got = snap.preempt(rc, rm, sel, pp, bn, bc, bm, bp, mv)
    want = preempt_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, pp, bn, bc, bm, bp, mv)
    _check(got, want)
    return got


def test_edge_cases(ks, orc):
    ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp = crowded(ks, 3000, 700, 4242)
    # no bound pods: nothing to evict (pods that fit nothing get no plan)
    e = np.zeros(0, np.int64)
    got = _edge_run(ks, orc, ac, am, lab, e.astype(np.int32), e, e, e.astype(np.int32), rc * 50, rm, sel, pp)
    assert np.all(got[0]["node_idx"] == -1) and not got[0]["candidates"].any()
    # every bound pod of higher or equal priority
    got = _edge_run(ks, orc, ac, am, lab, bn, bc, bm, np.maximum(bp, 5000), rc, rm, sel, np.minimum(pp, 5000))
    assert np.all(got[0]["node_idx"] == -1)
    # pending priority at the ends of int32, bound priorities across the range
    rng = np.random.default_rng(1)
    bfull = rng.integers(INT32_MIN, INT32_MAX, len(bn), endpoint=True).astype(np.int32)
    ends = np.where(np.arange(len(rc)) % 2 == 0, INT32_MIN, INT32_MAX).astype(np.int32)
    got = _edge_run(ks, orc, ac, am, lab, bn, bc, bm, bfull, rc, rm, sel, ends)
    assert np.all(got[0]["node_idx"][::2] == -1) and (got[0]["node_idx"][1::2] >= 0).any()
    # negative requests, bound and pending
    neg_c = np.where(np.arange(len(bn)) % 5 == 0, -bc // 3, bc)
    neg_m = np.where(np.arange(len(bn)) % 7 == 0, -bm // 2, bm)
    rc2 = np.where(np.arange(len(rc)) % 9 == 0, -rc, rc)
    _edge_run(ks, orc, ac, am, lab, bn, neg_c, neg_m, bp, rc2, rm, sel, pp)
    # one node holding 5 000 bound pods (the walk's worst case), at every cap
    bn5 = np.concatenate([bn, np.full(5000, 3, np.int32)])
    bc5 = np.concatenate([bc, np.full(5000, 7, np.int64)])
    bm5 = np.concatenate([bm, np.full(5000, 1 << 20, np.int64)])
    bp5 = np.concatenate([bp, rng.choice(np.array([0, 100, 1000], np.int32), 5000)])
    for mv in (1, 128):
        _edge_run(ks, orc, ac, am, lab, bn5, bc5, bm5, bp5, rc, rm, sel, pp, mv)
    big = np.array([30_000, 5, 35_001], np.int64)  # needs about 5 000 evictions of 7m on node 3: over every cap
    _edge_run(ks, orc, ac, am, lab, bn5, bc5, bm5, bp5, big, np.zeros(3, np.int64), sel[:3] * 0, np.full(3, 10**6, np.int32),
              128)


def test_range_limits_and_empty_snapshot(ks, orc):
    LC, LM = 1 << 36, 1 << 55
    ac = np.array([LC, LC, 1000], np.int64)
    am = np.array([LM, LM, 1000], np.int64)
    lab = np.zeros((3, 1), np.uint64)
    # node 0: 126 pods of +-2^36 cpu / +-2^55 mem, |sum| = 126 * 2^55 <= 2^62; free stays at the allocatable
    k = 126
    bn = np.zeros(k, np.int32)
    bc = np.where(np.arange(k) % 2 == 0, LC, -LC).astype(np.int64)
    bm = np.where(np.arange(k) % 2 == 0, LM, -LM).astype(np.int64)
    bp = (np.arange(k) % 5).astype(np.int32)
    rc = np.array([LC, LC, -LC, 1], np.int64)
    rm = np.array([LM, 0, LM, LM], np.int64)
    sel = np.zeros((4, 1), np.uint64)
    pp = np.array([3, INT32_MAX, 1, 2], np.int32)
    _edge_run(ks, orc, ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp, 128)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        for extra, code in (([LM, -LM], ks.KS_OK), ([LM, -LM, LM], ks.capi.KS_ERR_RANGE)):  # 128 * 2^55 = 2^62 is the limit
            more = np.concatenate([bn, np.zeros(len(extra), np.int32)]), np.concatenate([bc, np.zeros(len(extra), np.int64)])
            args = (*more, np.concatenate([bm, np.array(extra, np.int64)]), np.zeros(k + len(extra), np.int32))
            if code == ks.KS_OK:
                snap.preempt(rc, rm, sel, pp, *args, 4)
                continue
            with pytest.raises(ks.KsError) as e:
                snap.preempt(rc, rm, sel, pp, *args, 4)
            assert e.value.code == code
        rows, vic = snap.preempt(rc[:0], rm[:0], sel[:0], pp[:0], bn, bc, bm, bp, 4)  # P = 0
        assert rows.shape == (0,) and vic.shape == (0, 4)
        snap.set_nodes(np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 1), np.uint64))
        e0 = np.zeros(0, np.int64)
        rows, vic = snap.preempt(rc, rm, sel, pp, e0.astype(np.int32), e0, e0, e0.astype(np.int32), 4)
        assert np.all(rows["node_idx"] == -1) and np.all(vic == -1) and not rows["feasible_cnt"].any()
        assert np.all(rows["max_victim_priority"] == INT32_MIN) and not rows["victim_priority_sum"].any()


def test_consistency_on_c2_sized_cluster(ks):
    """Checks that do not use the restatement: evicting a plan's victims (set_bound again) makes ks_check_cell OK,
    putting any one victim back makes it fail; feasible_cnt is ks_select's count."""
    ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp = crowded(ks, 100_000, 10_000, 0xC2)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        rows, vic = snap.preempt(rc, rm, sel, pp, bn, bc, bm, bp, 16)
        r = snap.select(rc, rm, sel, flags=ks.KS_SELECT_FORCE_DIRECT)
        assert np.array_equal(rows["feasible_cnt"], r.feasible_cnt)
        assert np.all(rows["node_idx"][r.feasible_cnt > 0] == -1) and np.all(rows["candidates"][r.feasible_cnt > 0] == 0)
        planned = np.nonzero(rows["node_idx"] >= 0)[0]
        assert len(planned) > 1000
        for p in planned[np.linspace(0, len(planned) - 1, 40).astype(np.int64)]:
            n, v = int(rows["node_idx"][p]), vic[p][: rows["n_victims"][p]]
            assert (bn[v] == n).all() and (bp[v] < pp[p]).all()
            keep = np.ones(len(bn), bool)
            keep[v] = False
            snap.set_bound(bn[keep], bc[keep], bm[keep])
            assert snap.check_cell(rc[p], rm[p], sel[p], n) == ks.KS_CELL_OK
            for b in v:
                snap.apply_bind(n, bc[b], bm[b])
                assert snap.check_cell(rc[p], rm[p], sel[p], n) == ks.KS_CELL_NOT_ENOUGH_RESOURCES
                snap.apply_bind(n, -bc[b], -bm[b])
        snap.set_bound(bn, bc, bm)


def test_device_space_on_a_torch_stream_and_cached_graph_selects(ks, orc):
    import torch
    c = _cluster(ks, 2, 1025, False)
    ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp = c
    P, mv = 20_000, 3
    rc, rm, sel, pp = rc[:P], rm[:P], np.ascontiguousarray(sel[:P]), pp[:P]
    dev = torch.device("cuda:0")
    t = [torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(dev) for x in (rc, rm, sel)]
    tp = torch.from_numpy(pp.copy()).to(dev)
    out = torch.full((P, 4), -7, dtype=torch.int64, device=dev)  # 32 bytes per row
    vic = torch.full((P, mv), -7, dtype=torch.int32, device=dev)
    st = torch.cuda.Stream()
    bound = (bn, bc, bm, bp)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        want = snap.preempt(rc, rm, sel, pp, bn, bc, bm, bp, mv)
        torch.cuda.synchronize()
        snap.preempt_raw(P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, tp, bound, mv, out, vic, ks.KS_MEM_DEVICE,
                         stream=st.cuda_stream)
        st.synchronize()
        _check((out.cpu().numpy().view(ks.capi.PREEMPTION_DTYPE).reshape(P), vic.cpu().numpy()), want)
        h_out = np.zeros(P, ks.capi.PREEMPTION_DTYPE)
        snap.preempt_raw(P, rc, rm, sel, ks.KS_MEM_HOST, pp, bound, mv, h_out, None, ks.KS_MEM_HOST)
        assert np.array_equal(h_out, want[0])  # victims skipped
        # interleaved with cached-graph selects: both keep their results
        o_idx, o_score, o_cnt = orc.run_packed(*orc.free_reduce(ac, am, bn, bc, bm), ac, am, lab, rc, rm, sel,
                                               want_mask=False)[:3]
        idx = torch.empty(P, dtype=torch.int32, device=dev)
        score = torch.empty(P, dtype=torch.int64, device=dev)
        cnt = torch.empty(P, dtype=torch.int32, device=dev)
        for rep in range(3):
            idx.fill_(-7)
            torch.cuda.synchronize()
            snap.select_raw(P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, idx, score, cnt, ks.KS_MEM_DEVICE)
            torch.cuda.synchronize()
            assert np.array_equal(idx.cpu().numpy(), o_idx) and np.array_equal(score.cpu().numpy(), o_score)
            assert np.array_equal(cnt.cpu().numpy().view(np.uint32), o_cnt)
            n = P * (rep + 1) // 3  # grows: staging buffers are reallocated between graph replays
            got = snap.preempt(rc[:n], rm[:n], sel[:n], pp[:n], bn, bc, bm, bp, (1, 3, 128)[rep])
            if rep == 1:
                _check(got, (want[0][:n], want[1][:n]))
    s = _sample(P)
    _check(want, _oracle(orc, c, s, mv), s)


def test_host_layer_gv1_objects(ks):
    g = load_golden("gv1.json")
    gold = load_golden("gv1_preempt.json")["gv1"]
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(g["nodes"]), arena.pods(g["bound_pods"]), arena.pods(g["pods"])
    p = gold["pod"]
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        ctx.set_cluster_pods(bound, len(g["bound_pods"]))
        ctx.set_pod_priorities(bound, [0, 1000, 0, 0, 0, 0], len(g["bound_pods"]))  # b2a = 1000; the stray is unknown
        for case in gold["cases"]:
            rows, keys = ctx.preempt_pods(pods, 1, [case["priority"]], gold["max_victims"], first=p)
            assert int(rows["node_idx"][0]) == case["node_idx"] and int(rows["candidates"][0]) == case["candidates"]
            want = [gold["bound_keys"][v] for v in case["victims"]]
            assert keys[0] == (want if want else None)
        assert ctx.node_name(2) == "n2" and ctx.num_bound == 5  # nothing charged


def _obj_cluster(ks):
    ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp = crowded(ks, 400, 300, 515, n_keys=16)
    cl = ks.synth.make(400, 300, 515, n_keys=16, bound_per_node=0)
    nodes_s, _, pods_s = ks.objects.cluster_specs(cl)
    bound_s = [{"name": f"b{i}", "ns": "load", "node_name": nodes_s[n]["name"],
                "containers": [{"cpu": f"{c}m", "memory": str(m)}]} for i, (n, c, m) in enumerate(zip(bn, bc, bm))]
    return nodes_s, bound_s, pods_s, bp, pp


def test_host_layer_against_restatement_after_events(ks, orc):
    nodes_s, bound_s, pods_s, bp, pp = _obj_cluster(ks)
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(nodes_s), arena.pods(bound_s), arena.pods(pods_s)
    P = len(pods_s)
    mirror = [[b["name"], int(q)] for b, q in zip(bound_s, bp)]  # the context's rows: key and priority, in row order

    def swap_remove(i):
        mirror[i] = mirror[-1]
        mirror.pop()

    def check(ctx, mv=8):
        rc, rm, sel = ctx.pack_pods(pods, P)  # first: packing may widen the label dictionary
        ac, am, lab, bn, bc, bm = ctx.export_packed()
        fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
        want = preempt_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, pp, bn, bc, bm, [q for _, q in mirror], mv)
        rows, keys = ctx.preempt_pods(pods, P, pp, mv)
        for f in FIELDS:
            assert np.array_equal(rows[f], want[0][f]), f
        for i in range(P):
            names = [mirror[v][0] for v in want[1][i] if v >= 0]
            assert keys[i] == (["load/" + n for n in names] if want[0]["node_idx"][i] >= 0 else None)
        assert (rows["node_idx"] >= 0).sum() > 10

    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, len(nodes_s))
        ctx.set_cluster_pods(bound, len(bound_s))
        ctx.set_pod_priorities(bound, bp, len(bound_s))
        check(ctx)
        # a deleted pod: swap-remove moves the last row (and its priority) into its place
        ctx.pod_deleted(bound, 10)
        swap_remove(10)
        check(ctx)
        # a known pod bound again (new request): its row moves to the end and keeps its priority
        again = dict(bound_s[20], containers=[{"cpu": "1m", "memory": "1"}])
        ctx.pod_bound(arena.pods([again]))
        pos = [k for k, _ in mirror].index(again["name"])
        prio = mirror[pos][1]
        swap_remove(pos)
        mirror.append([again["name"], prio])
        check(ctx)
        # node events: an allocatable change, then a removal (its pods go, later nodes move down)
        changed = dict(nodes_s[4], allocatable={"cpu": "1", "memory": "1024"})
        ctx.upsert_node(arena.nodes([changed]))
        check(ctx)
        gone = nodes_s[7]["name"]
        node_of = {b["name"]: b["node_name"] for b in bound_s}
        ctx.remove_node(gone)
        i = 0
        while i < len(mirror):
            if node_of[mirror[i][0]] == gone:
                swap_remove(i)
            else:
                i += 1
        check(ctx)


def test_bad_arguments_are_status_codes(ks):
    import ctypes as C
    lib = ks.lib
    rc = np.zeros(4, np.int64)
    sel = np.zeros(4, np.uint64)
    pr = np.zeros(4, np.int32)
    out = np.zeros(4, ks.capi.PREEMPTION_DTYPE)
    bn, bc = np.zeros(2, np.int32), np.zeros(2, np.int64)
    with ks.Snapshot(0) as snap:
        snap.set_nodes([1000], [1000], np.zeros((1, 1), np.uint64))
        pods = ks.capi.ks_pods(4, rc.ctypes.data, rc.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
        good = ks.capi.ks_bound_pods(2, bn.ctypes.data, bc.ctypes.data, bc.ctypes.data, pr.ctypes.data)

        def call(mv=3, s=snap._h, p=pods, prio=pr.ctypes.data, b=good, o=out.ctypes.data, space=ks.KS_MEM_HOST):
            return lib.ks_preempt(s, C.byref(p) if p is not None else None, prio, C.byref(b) if b is not None else None,
                                  mv, o, None, space, None)

        assert call(mv=0) == -5 and call(mv=129) == -5 and call(mv=128) == 0 and call(mv=1) == 0
        assert call(s=None) == -1 and call(p=None) == -1 and call(prio=None) == -1 and call(o=None) == -1
        assert call(b=None) == -1 and call(space=3) == -1
        assert call(b=ks.capi.ks_bound_pods(2, None, bc.ctypes.data, bc.ctypes.data, pr.ctypes.data)) == -1
        bad_node = np.array([0, 1], np.int32)
        assert call(b=ks.capi.ks_bound_pods(2, bad_node.ctypes.data, bc.ctypes.data, bc.ctypes.data, pr.ctypes.data)) == -1
        big = np.array([0, (1 << 36) + 1], np.int64)
        assert call(b=ks.capi.ks_bound_pods(2, bn.ctypes.data, big.ctypes.data, bc.ctypes.data, pr.ctypes.data)) == -5
        empty = ks.capi.ks_pods(0, None, None, None, ks.KS_MEM_HOST)
        assert call(p=empty, prio=None, o=None) == 0
        assert call() == 0 and np.all(out["node_idx"] == -1) and np.all(out["feasible_cnt"] == 1)
    with ks.host.Context(0) as ctx:
        assert lib.ksh_preempt_pods(ctx._h, None, 3, pr.ctypes.data, 4, out.ctypes.data, None, 0, None) == -1
        assert lib.ksh_preempt_pods(ctx._h, None, 0, None, 0, None, None, 0, None) == -5
        assert lib.ksh_preempt_pods(ctx._h, None, 0, None, 4, None, None, 0, None) == 0
