"""Preemption under the full filter (ks_fit_preempt) on the H100: every row, victim slot and unresolvable count bit for
bit against tests/fit_preempt_oracle.py (string-level taints, node affinity and resource maps) across label widths 1-8,
node counts at the tile and chunk edges up to 10 007, queues up to 100 000 pods, R = 0-8, max_victims 1, 3 and 128 with
full-range priorities, many rule classes, a 5 000-pod node and values at the range limits; Q1 against ks_preempt on
crowded clusters, Q3 against ks_select and ks_fit_bind, Q4 with ks_snapshot_set_bound on the shorter list; free[] and
ks_select on both paths unchanged after the call; and every argument error before any device work."""
import ctypes as C

import numpy as np
import pytest

import fit_preempt_oracle as fpo
from helpers import load_golden
from node_bind_oracle import compile_rules
from preempt_oracle import crowded

pytestmark = pytest.mark.gpu

LIM = 1 << 62


def widen(a, W):
    """label bits [rows, w] padded with zero words to W"""
    return np.concatenate([a, np.zeros((a.shape[0], W - a.shape[1]), np.uint64)], axis=1) if W > a.shape[1] else a


def device(ks, d, max_victims, W=None, with_rules=True, with_res=True, snap=None):
    """Snapshot.fit_preempt over cluster_inputs d on a fresh snapshot (or snap, already holding d's nodes and bound)"""
    W = W or d["labels"].shape[1]
    rules = compile_rules(d["node_labels"], d["node_taints"], d["group_rules"]) if with_rules else None
    res = dict(node_free=d["node_free"], pod_req=d["pod_req"], bound_req=d["bound_req"]) if with_res else {}
    args = (d["rc"], d["rm"], widen(d["sel"], W), d["prio"], d["group"] if with_rules else np.full(len(d["rc"]), -1),
            d["G"] if with_rules else 0, d["bn"], d["bc"], d["bm"], d["bp"], max_victims)
    if snap is not None:
        return snap.fit_preempt(*args, rules=rules, **res)
    with ks.Snapshot(0) as s:
        s.set_nodes(d["ac"], d["am"], widen(d["labels"], W))
        s.set_bound(d["bn"], d["bc"], d["bm"])
        return s.fit_preempt(*args, rules=rules, **res)


def same(got, want):
    rows, vic, unres = got
    wr, wv, wu = want
    for f in wr.dtype.names:
        assert np.array_equal(rows[f], wr[f]), f
    assert np.array_equal(vic, wv) and np.array_equal(unres, wu)


def test_golden_plans_and_ks_preempt_contrast(ks):
    for case in load_golden("gv1_fit_preempt.json")["cases"]:
        d = fpo.golden_case(case)
        rows, vic, unres = device(ks, d, case["max_victims"])
        same((rows, vic, unres), fpo.run(d, case["max_victims"]))
        assert int(rows["node_idx"][0]) == case["want"]["node_idx"] and int(unres[0]) == case["want"]["unresolvable"]
        with ks.Snapshot(0) as s:
            s.set_nodes(d["ac"], d["am"], d["labels"])
            s.set_bound(d["bn"], d["bc"], d["bm"])
            prow, _ = s.preempt(d["rc"], d["rm"], d["sel"], d["prio"], d["bn"], d["bc"], d["bm"], d["bp"],
                                case["max_victims"])
        assert {k: int(prow[k][0]) for k in case["preempt_want"]} == case["preempt_want"], case["name"]


@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("N, P", [(1, 300), (31, 200), (1023, 24), (1024, 24), (1025, 24), (4097, 10)])
def test_matches_restatement(ks, W, N, P):
    rng = np.random.default_rng(1000 * W + N)
    d = fpo.random_cluster(rng, N, P, 5, R=3)
    for mv in (1, 3, 128):
        same(device(ks, d, mv, W), fpo.run(d, mv))


def test_big_node_count_and_queue(ks):
    d = fpo.random_cluster(np.random.default_rng(10007), 10007, 12, 6, R=2, full_range=True)
    same(device(ks, d, 128, 2), fpo.run(d, 128))
    d = fpo.random_cluster(np.random.default_rng(100000), 2, 100000, 4, per_node=3, R=3)
    got = device(ks, d, 3)
    same(got, fpo.run(d, 3))
    assert (got[0]["node_idx"] >= 0).sum() > 1000


@pytest.mark.parametrize("R", range(9))
def test_every_resource_count(ks, R):
    d = fpo.random_cluster(np.random.default_rng(77 + R), 300, 60, 8, per_node=6, R=R, full_range=R % 2 == 1)
    for mv in (1, 3, 128):
        same(device(ks, d, mv, with_res=R > 0), fpo.run(d, mv, with_res=R > 0))


def test_many_rule_classes_and_full_range(ks):
    d = fpo.random_cluster(np.random.default_rng(64), 700, 150, 64, per_node=5, R=4, full_range=True)
    assert len({repr(r) for r in d["group_rules"]}) > 30
    for mv in (1, 3, 128):
        same(device(ks, d, mv, 4), fpo.run(d, mv))


def test_five_thousand_pod_node(ks):
    """Node 0 holds 5 000 bound pods of one GPU-less sliver each at full-range priorities; the pods need many victims."""
    rng = np.random.default_rng(5000)
    N = 3
    bound = [(0, 10, 1000, int(rng.integers(-(1 << 31), (1 << 31) - 1, endpoint=True)), {"example.com/x": 1})
             for _ in range(5000)]
    bound += [(1, 4000, 1000, 0, {}), (2, 100, 100, 5, {"example.com/x": 3})]
    alloc = [{"pods": 5000, "example.com/x": 5000}, {"pods": 110}, {"pods": 2, "example.com/x": 3}]
    pods = [dict(cpu=int(c), mem=1000, selector={}, priority=int(pr), group=-1, res={"example.com/x": int(x)})
            for c, pr, x in zip(rng.integers(50, 2000, 40), rng.integers(-(1 << 31), (1 << 31) - 1, 40),
                                rng.integers(0, 200, 40))]
    d = fpo.cluster_inputs([50000, 8000, 8000], [10 ** 8] * 3, [{}] * N, [[]] * N, alloc, bound, pods)
    d.update(node_labels=[{}] * N, node_taints=[[]] * N, group_rules=[], alloc=alloc, bound=bound,
             pod_res=[p["res"] for p in pods], G=0)
    for mv in (1, 3, 128):
        got = device(ks, d, mv)
        same(got, fpo.run(d, mv))
    assert (got[0]["n_victims"] > 20).any()


def test_range_limits(ks):
    """|node_free| + the bound requests at exactly 2^62 is taken (node 0: node_free 2^61, two bound pods of 2^60); one
    more is KS_ERR_RANGE before any device work."""
    X = "example.com/x"
    alloc = [{"pods": 4, X: LIM}, {"pods": 4}]
    bound = [(0, 1000, 1000, 0, {X: LIM // 4}), (0, 1000, 1000, 1, {X: LIM // 4}), (1, 1000, 1000, 0, {})]
    pods = [dict(cpu=100, mem=100, selector={}, priority=p, group=-1, res={X: q})
            for p, q in ((10, 1), (10, LIM // 2), (10, LIM // 2 + 1), (10, LIM), (10, LIM + 1), (1, LIM),
                         (-(1 << 31), 1), (10, 0))]
    d = fpo.cluster_inputs([3000, 1000], [3000, 1000], [{}] * 2, [[]] * 2, alloc, bound, pods)
    d.update(node_labels=[{}] * 2, node_taints=[[]] * 2, group_rules=[], alloc=alloc, bound=bound,
             pod_res=[p["res"] for p in pods], G=0)
    assert d["names"] == ["pods", X] and int(d["node_free"][1, 0]) == LIM // 2
    got = device(ks, d, 4)
    same(got, fpo.run(d, 4))
    assert got[0]["node_idx"].tolist() == [-1, -1, 0, 0, -1, -1, -1, -1]
    assert got[0]["n_victims"].tolist()[2:4] == [1, 2]
    with ks.Snapshot(0) as s:
        s.set_nodes(d["ac"], d["am"], d["labels"])
        s.set_bound(d["bn"], d["bc"], d["bm"])
        for delta in (1, -LIM - LIM // 2 - 1):  # |node_free| 2^61 + 1, then 2^62 + 1
            nf = d["node_free"].copy()
            nf[1, 0] += delta
            with pytest.raises(ks.KsError) as e:
                s.fit_preempt(d["rc"], d["rm"], d["sel"], d["prio"], d["group"], 0, d["bn"], d["bc"], d["bm"],
                              d["bp"], 4, node_free=nf, pod_req=d["pod_req"], bound_req=d["bound_req"])
            assert e.value.code == ks.capi.KS_ERR_RANGE


@pytest.mark.parametrize("full_range", [False, True])
def test_q1_is_ks_preempt(ks, full_range):
    for W_keys, seed in ((8, 1), (16, 2), (32, 3), (64, 4)):
        levels = (None, None) if full_range else ((0, 100, 1000), (0, 100, 1000, 5000))
        ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp = crowded(ks, 3000, 2000 + seed, seed, n_keys=W_keys,
                                                               prio_levels=levels[0], pod_levels=levels[1])
        with ks.Snapshot(0) as s:
            s.set_nodes(ac, am, lab)
            s.set_bound(bn, bc, bm)
            for mv in (1, 3, 128):
                want = s.preempt(rc, rm, sel, pp, bn, bc, bm, bp, mv)
                rows, vic, unres = s.fit_preempt(rc, rm, sel, pp, np.full(len(rc), -1), 0, bn, bc, bm, bp, mv)
                assert all(np.array_equal(rows[f], want[0][f]) for f in rows.dtype.names) and np.array_equal(vic, want[1])
                miss = np.zeros(len(rc), np.int64)
                for i in range(0, len(rc), 500):
                    miss[i:i + 500] = ((sel[i:i + 500, None, :] & ~lab[None, :, :]) != 0).any(axis=2).sum(axis=1)
                assert np.array_equal(unres, miss)
            assert (want[0]["node_idx"] >= 0).sum() > 50


def test_q3_feasible_count_is_select_minus_fit_bind_refusals(ks):
    d = fpo.random_cluster(np.random.default_rng(33), 500, 24, 6, per_node=5, R=4)
    rules = compile_rules(d["node_labels"], d["node_taints"], d["group_rules"])
    N, G = len(d["ac"]), d["G"]
    with ks.Snapshot(0) as s:
        s.set_nodes(d["ac"], d["am"], d["labels"])
        s.set_bound(d["bn"], d["bc"], d["bm"])
        rows, _, _ = device(ks, d, 3, snap=s)
        cnt = s.select(d["rc"], d["rm"], d["sel"], flags=ks.KS_SELECT_FORCE_DIRECT).feasible_cnt
        keys = [(np.zeros(N, np.int32), 1)]
        for p in range(len(d["rc"])):
            sl = slice(p, p + 1)
            out = s.fit_bind(d["rc"][sl], d["rm"][sl], d["sel"][sl], d["group"][sl], G, keys,
                             max_skew=np.zeros((G, 1), np.uint32), rules=rules, node_free=d["node_free"],
                             pod_req=d["pod_req"][sl])
            s.set_bound(d["bn"], d["bc"], d["bm"])  # undo the bind
            refused = out[3][0]
            assert int(rows["feasible_cnt"][p]) == int(cnt[p]) - int(refused[:3].sum()), p
    assert (rows["feasible_cnt"] > 0).any() and (rows["feasible_cnt"] == 0).any()


def test_q4_evict_then_bind_and_nothing_changes(ks):
    d = fpo.random_cluster(np.random.default_rng(44), 400, 60, 5, per_node=6, R=3, full_range=True)
    with ks.Snapshot(0) as s:
        s.set_nodes(d["ac"], d["am"], d["labels"])
        s.set_bound(d["bn"], d["bc"], d["bm"])
        free0 = s.free()
        sel0 = [s.select(d["rc"], d["rm"], d["sel"], flags=f) for f in (ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR)]
        rows, vic, _ = device(ks, d, 128, snap=s)
        assert all(np.array_equal(a, b) for a, b in zip(s.free(), free0))
        for f, r0 in zip((ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR), sel0):
            r = s.select(d["rc"], d["rm"], d["sel"], flags=f)
            assert np.array_equal(r.node_idx, r0.node_idx) and np.array_equal(r.feasible_cnt, r0.feasible_cnt)
        planned = np.nonzero(rows["node_idx"] >= 0)[0]
        assert len(planned) > 5
        for p in planned[:8]:
            v = [int(x) for x in vic[p] if x >= 0]
            keep = np.setdiff1d(np.arange(len(d["bn"])), v)
            e = fpo.cluster_inputs(d["ac"], d["am"], d["node_labels"], d["node_taints"], d["alloc"],
                                   [d["bound"][b] for b in keep],
                                   [dict(cpu=int(d["rc"][p]), mem=int(d["rm"][p]), selector={},
                                         priority=int(d["prio"][p]), group=int(d["group"][p]), res=d["pod_res"][p])],
                                   d["names"])
            e.update(labels=d["labels"], sel=d["sel"][p:p + 1], node_labels=d["node_labels"],
                     node_taints=d["node_taints"], group_rules=d["group_rules"], alloc=d["alloc"],
                     bound=[d["bound"][b] for b in keep], pod_res=[d["pod_res"][p]], G=d["G"])
            s.set_bound(e["bn"], e["bc"], e["bm"])
            assert all(np.array_equal(a, b) for a, b in zip(s.free(), (e["fc"], e["fm"])))
            r2 = device(ks, e, 128, snap=s)
            assert int(r2[0]["feasible_cnt"][0]) > 0 and int(r2[0]["node_idx"][0]) == -1
            assert fpo.fits_after(d, p, int(rows["node_idx"][p]), v)
        s.set_bound(d["bn"], d["bc"], d["bm"])


def test_argument_errors_before_device_work(ks):
    d = fpo.random_cluster(np.random.default_rng(9), 20, 4, 2, R=2)
    rules = compile_rules(d["node_labels"], d["node_taints"], d["group_rules"])
    lib, cap = ks.lib, ks.capi
    P, B, N = len(d["rc"]), len(d["bn"]), len(d["ac"])
    with ks.Snapshot(0) as s:
        s.set_nodes(d["ac"], d["am"], d["labels"])
        s.set_bound(d["bn"], d["bc"], d["bm"])
        free0 = s.free()
        pods = cap.ks_pods(P, d["rc"].ctypes.data, d["rm"].ctypes.data, d["sel"].ctypes.data, ks.KS_MEM_HOST)
        nr, hold = ks.snapshot.node_rules(rules)
        nf, pr, br = (np.ascontiguousarray(d[k]) for k in ("node_free", "pod_req", "bound_req"))
        res = cap.ks_bind_resources(nf.shape[0], nf.ctypes.data, pr.ctypes.data)
        bound = cap.ks_bound_pods(B, d["bn"].ctypes.data, d["bc"].ctypes.data, d["bm"].ctypes.data, d["bp"].ctypes.data)
        out = np.zeros(P, cap.PREEMPTION_DTYPE)
        grp = d["group"].copy()

        def call(pods=pods, group=grp.ctypes.data, G=d["G"], rules=C.byref(nr), res=C.byref(res),
                 prio=d["prio"].ctypes.data, bound=C.byref(bound), breq=br.ctypes.data, mv=4, o=out.ctypes.data):
            return lib.ks_fit_preempt(s._h, C.byref(pods) if pods is not None else None, group, G, rules, res, prio,
                                      bound, breq, mv, o, None, None)
        assert call() == 0
        assert call(mv=0) == cap.KS_ERR_RANGE and call(mv=129) == cap.KS_ERR_RANGE
        assert call(prio=None) == cap.KS_ERR_INVALID and call(o=None) == cap.KS_ERR_INVALID
        assert call(bound=None) == cap.KS_ERR_INVALID and call(group=None) == cap.KS_ERR_INVALID
        assert call(breq=None) == cap.KS_ERR_INVALID
        assert call(G=5000) == cap.KS_ERR_RANGE
        dev_pods = cap.ks_pods(P, d["rc"].ctypes.data, d["rm"].ctypes.data, d["sel"].ctypes.data, ks.KS_MEM_DEVICE)
        assert call(pods=dev_pods) == cap.KS_ERR_INVALID
        bad = grp.copy()
        bad[0] = d["G"]
        assert call(group=bad.ctypes.data) == cap.KS_ERR_INVALID
        bad_b = d["bn"].copy()
        bad_b[0] = N
        b2 = cap.ks_bound_pods(B, bad_b.ctypes.data, d["bc"].ctypes.data, d["bm"].ctypes.data, d["bp"].ctypes.data)
        assert call(bound=C.byref(b2)) == cap.KS_ERR_INVALID
        neg = br.copy()
        neg[0, 0] = -1
        assert call(breq=neg.ctypes.data) == cap.KS_ERR_RANGE
        negp = pr.copy()
        negp[0, 0] = -1
        r2 = cap.ks_bind_resources(nf.shape[0], nf.ctypes.data, negp.ctypes.data)
        assert call(res=C.byref(r2)) == cap.KS_ERR_RANGE
        r9 = cap.ks_bind_resources(9, nf.ctypes.data, pr.ctypes.data)
        assert call(res=C.byref(r9)) == cap.KS_ERR_RANGE
        bad_rules = dict(rules, tolerate_hard=np.full(d["G"], np.uint64(1) << np.uint64(63), np.uint64))
        nr2, hold2 = ks.snapshot.node_rules(bad_rules)
        assert call(rules=C.byref(nr2)) == cap.KS_ERR_INVALID
        heavy = d["bc"].copy()
        heavy[:] = 1 << 36
        b3 = cap.ks_bound_pods(B, d["bn"].ctypes.data, heavy.ctypes.data, d["bm"].ctypes.data, d["bp"].ctypes.data)
        assert call(bound=C.byref(b3)) in (0, cap.KS_ERR_RANGE)
        assert all(np.array_equal(a, b) for a, b in zip(s.free(), free0))
        # nothing to do: no pods, or an empty snapshot
        assert call(pods=cap.ks_pods(0, None, None, None, ks.KS_MEM_HOST), prio=None, o=None) == 0
    with ks.Snapshot(0) as s:
        s.set_nodes(np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 1), np.uint64))
        rows, vic, unres = s.fit_preempt(d["rc"], d["rm"], d["sel"][:, :1], d["prio"], np.full(P, -1), 0,
                                         np.zeros(0, np.int32), np.zeros(0, np.int64), np.zeros(0, np.int64),
                                         np.zeros(0, np.int32), 3)
        assert (rows["node_idx"] == -1).all() and (vic == -1).all() and (unres == 0).all()
        assert (rows["feasible_cnt"] == 0).all() and (rows["max_victim_priority"] == -(1 << 31)).all()


def test_host_layer_end_to_end_after_events(ks):
    """ksh_preempt_fit_pods over objects (labels, taints, allocatable pods and GPUs, running GPU pods at priority 0)
    against the restatement over the same strings, after node, taint and pod events; victims named namespace/name."""
    GPU = "nvidia.com/gpu"
    rng = np.random.default_rng(0xF17)
    taint = {"key": "nvidia.com/gpu", "value": "present", "effect": "NoSchedule"}
    nodes = {}
    for i in range(40):
        gpu = i % 4 == 3
        a = {"cpu": "16", "memory": str(64 << 30), "pods": str(int(rng.integers(2, 8)))}
        if gpu:
            a[GPU] = "8"
        nodes[f"n{i}"] = {"name": f"n{i}", "labels": {"zone": "abc"[i % 3], **({"gpu": "h100"} if gpu else {})},
                          "allocatable": a}
    taints = {nm: [taint] for nm, s in nodes.items() if GPU in s["allocatable"]}
    bound = []
    for i, nm in enumerate(nodes):
        for j in range(int(rng.integers(1, 5))):
            c = {"cpu": f"{int(rng.integers(2000, 5000))}m", "memory": str(int(rng.integers(1, 9)) << 30)}
            if GPU in nodes[nm]["allocatable"] and j < 2:
                c[GPU] = "4"
            bound.append({"name": f"b{i}-{j}", "ns": "batch", "node_name": nm, "containers": [c]})
    bprio = {b["name"]: int(rng.choice([0, 0, 100, 5000])) for b in bound}
    rules = [{"tolerations": [{"key": "nvidia.com/gpu", "operator": "Exists", "effect": "NoSchedule"}]},
             {"required": [[{"key": "zone", "operator": "In", "values": ["a", "b"]}]]}]
    pending = []
    for p in range(48):
        c = {"cpu": f"{int(rng.integers(3000, 12000))}m", "memory": str(int(rng.integers(1, 20)) << 30)}
        g = p % 3 - 1
        if g == 0:
            c[GPU] = str(int(rng.integers(1, 9)))
        pending.append(({"name": f"q{p}", "ns": "train", "containers": [c]}, g))
    arena = ks.objects.ObjectArena()
    pods = arena.pods([q for q, _ in pending])
    group = np.array([g for _, g in pending], np.int32)
    prio = np.full(len(pending), 1000, np.int32)

    def ints(m):
        return {k: int(v) for k, v in m.items() if k not in ("cpu", "memory")}

    def check(ctx, mirror, mv=8):
        rc, rm, sel = ctx.pack_pods(pods, len(pending))
        ac, am, lab, bn, bc, bm = ctx.export_packed()
        order = [ctx.node_name(i) for i in range(ctx.n_nodes)]
        assert [b["node_name"] for b in mirror] == [order[n] for n in bn]
        bl = [(int(n), int(c), int(m), bprio[b["name"]], ints(b["containers"][0])) for n, c, m, b in zip(bn, bc, bm, mirror)]
        d = dict(fc=ac.copy(), fm=am.copy(), labels=lab, sel=sel[:, :lab.shape[1]], rc=rc, rm=rm, prio=prio, group=group,
                 node_labels=[nodes[nm]["labels"] for nm in order], node_taints=[taints.get(nm, []) for nm in order],
                 group_rules=rules, alloc=[ints(nodes[nm]["allocatable"]) for nm in order], bound=bl,
                 pod_res=[ints(q["containers"][0]) for q, _ in pending])
        np.subtract.at(d["fc"], bn, bc)
        np.subtract.at(d["fm"], bn, bm)
        want = fpo.run(d, mv)
        rows, keys = ctx.preempt_fit_pods(pods, len(pending), group, len(rules), prio, mv, group_rules=rules)
        for f in rows.dtype.names:
            assert np.array_equal(rows[f], want[0][f]), f
        for i in range(len(pending)):
            names = ["batch/" + mirror[v]["name"] for v in want[1][i] if v >= 0]
            assert keys[i] == (names if want[0]["node_idx"][i] >= 0 else None)
        return rows

    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(list(nodes.values())), len(nodes))
        ctx.set_node_taints(taints)
        ctx.set_cluster_pods(arena.pods(bound), len(bound))
        ctx.set_pod_priorities(arena.pods(bound), np.array([bprio[b["name"]] for b in bound], np.int32), len(bound))
        mirror = list(bound)
        rows = check(ctx, mirror)
        assert ((rows["node_idx"] >= 0) & (group == 0)).sum() > 3  # GPU pods that preempt running GPU pods
        # a taint event: the GPU pool's taint removed from one node, a NoExecute taint on another
        taints["n3"] = []
        taints["n5"] = [{"key": "maintenance", "value": "true", "effect": "NoExecute"}]
        ctx.set_node_taints({"n3": [], "n5": taints["n5"]})
        check(ctx, mirror)
        # a pod event: a running GPU pod deleted (swap-remove moves the last row into its place)
        k = next(i for i, b in enumerate(mirror) if GPU in b["containers"][0])
        ctx.pod_deleted(arena.pods([mirror[k]]))
        mirror[k] = mirror[-1]
        mirror.pop()
        check(ctx, mirror)
        # a node event: a GPU node's pod limit lowered
        nodes["n7"] = dict(nodes["n7"], allocatable=dict(nodes["n7"]["allocatable"], pods="2"))
        ctx.upsert_node(arena.nodes([nodes["n7"]]))
        check(ctx, mirror)
