"""Drain simulation under the full filter (ks_fit_drain_check) on the H100: placed counts, nodes, scores and refusal words
bit for bit against tests/fit_drain_oracle.py (string-level taints, node affinity and resource maps) across label widths
1-8, node counts on the tile and chunk edges up to 16 897, up to 20 000 candidates, R = 0-8, 64 rule groups, all four
policies, with and without KS_DRAIN_EXCLUDE_CANDIDATES, duplicate candidates, ties across chunks and overlays and a
1024-pod candidate; the refusal pass on a snapshot whose scratch holds earlier calls' data; D1 against ks_drain_check,
also on ks_drain_check's edge values; D4 replayed with ks_snapshot_apply_bind; free[] and ks_select on both paths
unchanged after every call; ksh_drain_fit_nodes end to end after node, taint and pod events; and the argument errors
before any device work."""
import numpy as np
import pytest

import fit_drain_oracle as fdo
from helpers import load_golden
from node_bind_oracle import compile_rules

pytestmark = pytest.mark.gpu


def widen(a, W):
    return np.concatenate([a, np.zeros((a.shape[0], W - a.shape[1]), np.uint64)], axis=1) if W > a.shape[1] else a


def select_state(ks, s, rc, rm, sel):
    """ks_select on both kernel paths for a probe of pods"""
    out = []
    for flags in (ks.capi.KS_SELECT_FORCE_DIRECT, ks.capi.KS_SELECT_FORCE_BITPAR):
        r = s.select(rc, rm, sel, flags=flags)
        out.append((r.node_idx, r.score, r.feasible_cnt))
    return out


def call(ks, s, d, policy=0, flags=0, W=None, with_rules=True, with_res=True):
    """Snapshot.fit_drain_check on snapshot s (holding d's nodes and bound pods); free[] and ks_select on both paths
    are checked unchanged, and with rules and resources NULL the outputs against ks_drain_check (D1)."""
    W = W or d["labels"].shape[1]
    rules = compile_rules(d["node_labels"], d["node_taints"], d["group_rules"]) if with_rules else None
    res = dict(node_free=d["node_free"], pod_req=d["pod_req"]) if with_res else {}
    sel = widen(d["sel"], W)
    probe = slice(0, min(len(d["rc"]), 200))
    before = s.free(), select_state(ks, s, d["rc"][probe], d["rm"][probe], sel[probe])
    out = s.fit_drain_check(d["rc"], d["rm"], sel, d["group"] if with_rules else np.full(len(d["rc"]), -1, np.int32),
                            len(d["group_rules"]) if with_rules else 0, d["node_idx"], d["offset"], policy, flags,
                            rules=rules, **res)
    after = s.free(), select_state(ks, s, d["rc"][probe], d["rm"][probe], sel[probe])
    assert all(np.array_equal(a, b) for a, b in zip(before[0], after[0])), "free[] changed"
    for x, y in zip(before[1], after[1]):
        assert all(np.array_equal(a, b) for a, b in zip(x, y)), "ks_select changed"
    if not with_rules and not with_res:
        want = s.drain_check(d["rc"], d["rm"], sel, d["node_idx"], d["offset"], policy, flags)
        assert all(np.array_equal(a, b) for a, b in zip(out[:3], want)), "D1"
    return out


def load(ks, s, d, W=None):
    s.set_nodes(d["ac"], d["am"], widen(d["labels"], W or d["labels"].shape[1]))
    s.set_bound(d["bn"], d["bc"], d["bm"])


def device(ks, d, policy=0, flags=0, W=None, with_rules=True, with_res=True):
    with ks.Snapshot(0) as s:
        load(ks, s, d, W)
        return call(ks, s, d, policy, flags, W, with_rules, with_res)


def same(got, want):
    for g, w, name in zip(got, want, ("placed", "node_idx", "score", "refused")):
        assert np.array_equal(g, w), name


def test_golden_cases(ks):
    for case in load_golden("gv1_fit_drain.json")["cases"]:
        d = fdo.golden_case(case)
        got = device(ks, d)
        same(got, fdo.fit_drain(d, d["node_idx"], d["offset"]))
        assert got[0].tolist() == case["want"]["placed"] and got[3].tolist() == case["want"]["refused"]


@pytest.mark.parametrize("policy", [0, 1, 3, 4])
def test_against_the_restatement(ks, policy):
    rng = np.random.default_rng(100 + policy)
    for N, D, R, W in ((40, 60, 3, 1), (129, 200, 8, 2), (1025, 300, 1, 4), (4100, 150, 3, 8)):
        d = fdo.random_cluster(rng, N, D, R=R, max_pods=8)
        for flags in (0, 1):
            same(device(ks, d, policy, flags, W), fdo.fit_drain(d, d["node_idx"], d["offset"], policy, flags == 1))
        # R = 0 (res NULL) with rules, and D1 (rules and res NULL)
        same(device(ks, d, policy, 0, W, with_res=False),
             fdo.fit_drain(d, d["node_idx"], d["offset"], policy, with_res=False))
        device(ks, d, policy, 1, W, with_rules=False, with_res=False)


def test_large_candidates_and_duplicates(ks):
    rng = np.random.default_rng(7)
    d = fdo.random_cluster(rng, 600, 3, R=3, max_pods=2)
    big = [dict(cpu=10, mem=1 << 20, selector={}, group=int(g), res={}) for g in rng.integers(-1, 4, 1024)]
    nodes = [dict(cpu=int(c), mem=int(m), labels=l, taints=t, alloc=a) for c, m, l, t, a in
             zip(d["ac"], d["am"], d["node_labels"], d["node_taints"], d["alloc"])]
    e = fdo.cluster(nodes, [], [(5, big), (5, big[:100]), (9, big[:3])], d["names"])
    e["group_rules"] = d["group_rules"]
    for policy in (0, 4):
        got = device(ks, e, policy)
        same(got, fdo.fit_drain(e, e["node_idx"], e["offset"], policy))
    assert got[0][0] > 0


def test_errors_before_any_device_work(ks):
    d = fdo.random_cluster(np.random.default_rng(3), 20, 4, max_pods=3)
    with ks.Snapshot(0) as s:
        s.set_nodes(d["ac"], d["am"], d["labels"])
        s.set_bound(d["bn"], d["bc"], d["bm"])
        P = len(d["rc"])
        base = (d["rc"], d["rm"], d["sel"])

        def code(**kw):
            a = dict(group=d["group"], n_groups=len(d["group_rules"]), node_idx=d["node_idx"], offset=d["offset"],
                     policy=0, flags=0, node_free=d["node_free"], pod_req=d["pod_req"])
            a.update(kw)
            with pytest.raises(ks.KsError) as e:
                s.fit_drain_check(*base, a["group"], a["n_groups"], a["node_idx"], a["offset"], a["policy"],
                                  a["flags"], node_free=a["node_free"], pod_req=a["pod_req"])
            return e.value.code
        assert code(policy=9) == ks.capi.KS_ERR_INVALID
        assert code(flags=2) == ks.capi.KS_ERR_INVALID
        assert code(node_idx=np.full(len(d["node_idx"]), 99, np.int32)) == ks.capi.KS_ERR_INVALID
        assert code(group=np.full(P, 9, np.int32)) == ks.capi.KS_ERR_INVALID
        assert code(n_groups=1 << 20) == ks.capi.KS_ERR_RANGE
        assert code(pod_req=-np.ones_like(d["pod_req"])) == ks.capi.KS_ERR_RANGE
        off = d["offset"].copy()
        off[-1] += 1
        assert code(offset=off) == ks.capi.KS_ERR_INVALID
        many = np.array([0, 1025], np.uint64)
        rc = np.zeros(1025, np.int64)
        with pytest.raises(ks.KsError) as e:
            s.fit_drain_check(rc, rc, np.zeros((1025, d["sel"].shape[1]), np.uint64), np.full(1025, -1, np.int32), 0,
                              np.zeros(1, np.int32), many)
        assert e.value.code == ks.capi.KS_ERR_RANGE
        assert all(np.array_equal(a, b) for a, b in zip(s.free(), (d["fc"], d["fm"])))


def test_many_candidates_and_groups(ks):
    """20 000 candidates (sizes 0-6, duplicates; their pods not bound to them, so that 200 nodes hold them) on 200 nodes,
    and 16 897 nodes, both with 64 rule groups and R = 8; the refusal pass then runs over CTAs that mix stopped and
    drainable candidates, and over several node chunks."""
    rng = np.random.default_rng(41)
    for N, D, flags, bind in ((200, 20_000, 0, False), (16_897, 120, 1, True)):
        d = fdo.random_cluster(rng, N, D, R=8, G=64, max_pods=6, too_big=0.1, bind_drained=bind)
        got = device(ks, d, 4, flags)
        same(got, fdo.fit_drain(d, d["node_idx"], d["offset"], 4, flags == 1))
        size = np.diff(d["offset"]).astype(np.int64)
        assert (got[0] == size).any() and (got[0] < size).any()


def test_refusal_pass_after_other_calls_on_one_snapshot(ks):
    """The stop records live in the snapshot's scratch, which earlier calls fill: a large call with R = 8, then
    ks_drain_check, then smaller calls with other R and D on the same snapshot, each against the restatement."""
    rng = np.random.default_rng(43)
    big = fdo.random_cluster(rng, 300, 6000, R=8, G=16, max_pods=8)
    with ks.Snapshot(0) as s:
        load(ks, s, big)
        same(call(ks, s, big, 1), fdo.fit_drain(big, big["node_idx"], big["offset"], 1))
        s.drain_check(big["rc"], big["rm"], big["sel"], big["node_idx"], big["offset"])
        for R, D, policy in ((1, 2500, 0), (3, 700, 3), (2, 4000, 4)):
            d = fdo.random_cluster(rng, 300, D, R=R, G=8, max_pods=5)
            load(ks, s, d)
            same(call(ks, s, d, policy), fdo.fit_drain(d, d["node_idx"], d["offset"], policy))


def _same_nodes(N, n_gpu_every=7):
    """N identical nodes but for a GPU pool (tainted, 8 GPUs) on every n_gpu_every-th and a cordon on every 11th"""
    nodes = []
    for n in range(N):
        gpu = n % n_gpu_every == 0
        nodes.append(dict(cpu=8000, mem=8 << 30, labels={"gpu": "h100"} if gpu else {},
                          taints=([{"key": "nvidia.com/gpu", "value": "present", "effect": "NoSchedule"}] if gpu else [])
                          + ([fdo.CORDON] if n % 11 == 5 else []),
                          alloc={"pods": 110, **({"nvidia.com/gpu": 8} if gpu else {})}))
    return nodes


@pytest.mark.parametrize("policy", [0, 1, 3, 4])
def test_ties_across_chunks_and_overlays(ks, policy):
    """Equal free values everywhere, so every choice is a tie the lower index breaks; requests of 0 leave an overlay
    node level with untouched ones; candidates on both sides of tile and chunk boundaries."""
    N = 9 * 1024 + 3
    rng = np.random.default_rng(50 + policy)
    cands = []
    for n in rng.choice(np.array([0, 1, 1023, 1024, 1025, 2047, 2048, N - 1]), 250):
        pods = []
        for _ in range(int(rng.integers(0, 25))):
            g = int(rng.integers(-1, 2))
            pods.append(dict(cpu=int(rng.choice([0, 0, 1000, 4000, 8000])), mem=int(rng.choice([0, 0, 1 << 30, 8 << 30])),
                             selector={}, group=g, res={"nvidia.com/gpu": int(rng.integers(0, 3))} if g == 0 else {}))
        cands.append((int(n), pods))
    d = fdo.cluster(_same_nodes(N), [], cands, ["pods", "nvidia.com/gpu"])
    d["group_rules"] = [{"tolerations": [fdo.TOL_GPU]}, {}]
    for flags in (0, 1):
        same(device(ks, d, policy, flags), fdo.fit_drain(d, d["node_idx"], d["offset"], policy, flags == 1))


LC, LM = 1 << 36, 1 << 55


@pytest.mark.parametrize("policy", [0, 1, 3, 4])
def test_d1_on_edge_values(ks, policy):
    """D1 on ks_drain_check's edge values: free at +-limit, allocatable <= 0, requests at the limit, selectors with the
    bit no node carries; ties on equal free values across chunks."""
    rng = np.random.default_rng(60 + policy)
    N = 2500
    ac = rng.choice(np.array([-LC, -1, 0, 1, 1000, LC]), N)
    am = rng.choice(np.array([-LM, -1, 0, 1, 1 << 30, LM]), N)
    lab = rng.integers(0, 1 << 62, (N, 1), dtype=np.uint64)
    D = 150
    node = rng.integers(0, N, D).astype(np.int32)
    node[D // 2] = node[0]
    off = np.concatenate([[0], np.cumsum(rng.integers(0, 13, D))]).astype(np.uint64)
    P = int(off[-1])
    rc = rng.choice(np.array([0, 1, 1000, LC]), P)
    rm = rng.choice(np.array([0, 1, 1 << 30, LM]), P)
    sel = lab[rng.integers(0, N, P)] & rng.integers(0, 1 << 62, (P, 1), dtype=np.uint64)
    sel[rng.random(P) < 0.05, 0] |= np.uint64(1 << 63)
    with ks.Snapshot(0) as s:
        s.set_nodes(ac, am, lab)
        for flags in (0, 1):
            got = s.fit_drain_check(rc, rm, sel, np.full(P, -1, np.int32), 0, node, off, policy, flags)
            want = s.drain_check(rc, rm, sel, node, off, policy, flags)
            assert all(np.array_equal(a, b) for a, b in zip(got[:3], want))
            assert not got[3][got[0] == np.diff(off)].any()
        assert (got[0] < np.diff(off)).any() and (got[0] == np.diff(off)).any()
    # equal free values: every pick a tie, across 9 tiles and their chunks
    N = 9 * 1024 + 3
    ac, am = np.full(N, 8000, np.int64), np.full(N, 8 << 30, np.int64)
    lab = np.zeros((N, 2), np.uint64)
    node = rng.choice(np.array([0, 1023, 1024, 2048, N - 1]), 200).astype(np.int32)
    off = np.concatenate([[0], np.cumsum(rng.integers(0, 30, 200))]).astype(np.uint64)
    P = int(off[-1])
    rc, rm = rng.choice(np.array([0, 0, 1000, 8000]), P), rng.choice(np.array([0, 0, 1 << 30]), P)
    with ks.Snapshot(0) as s:
        s.set_nodes(ac, am, lab)
        got = s.fit_drain_check(rc, rm, np.zeros((P, 2), np.uint64), np.full(P, -1, np.int32), 0, node, off, policy)
        want = s.drain_check(rc, rm, np.zeros((P, 2), np.uint64), node, off, policy)
        assert all(np.array_equal(a, b) for a, b in zip(got[:3], want))


def test_d4_replay_with_apply_bind(ks):
    """Each sampled drainable candidate's moves replayed one at a time: before each, the pod passes the full filter on
    its node against the snapshot's free[] (ks_snapshot_apply_bind charges cpu and memory after each move), node_free
    less the pod_req already moved there, and the string-level taints and node affinity."""
    rng = np.random.default_rng(70)
    d = fdo.random_cluster(rng, 60, 400, R=3, G=8, max_pods=8)
    placed, idx, _, _ = device(ks, d, 0)
    cl = fdo.Cluster(d)
    size = np.diff(d["offset"]).astype(np.int64)
    done = [c for c in range(len(size)) if placed[c] == size[c] and size[c] > 1]
    assert len(done) > 20
    with ks.Snapshot(0) as s:
        s.set_nodes(d["ac"], d["am"], d["labels"])
        for c in done[:40]:
            s.set_bound(d["bn"], d["bc"], d["bm"])
            nf = d["node_free"].copy()
            for p in range(int(d["offset"][c]), int(d["offset"][c + 1])):
                n = int(idx[p])
                fc, fm = s.free()
                assert n != int(d["node_idx"][c])
                assert d["rc"][p] <= fc[n] and d["rm"][p] <= fm[n]
                assert ((d["sel"][p] & ~d["labels"][n]) == 0).all()
                q = d["pod_req"][p]
                assert ((q == 0) | (q <= nf[:, n])).all()
                assert cl.rule_stage(int(d["group"][p]))[n] == fdo.PASS
                s.apply_bind(n, int(d["rc"][p]), int(d["rm"][p]))
                nf[:, n] -= q


def test_integration_example(ks):
    """INTEGRATION.md's GPU-pool consolidation, as written there"""
    GPU = "nvidia.com/gpu"
    gpu_taint = {"key": GPU, "value": "present", "effect": "NoSchedule"}
    cordon = {"key": "node.kubernetes.io/unschedulable", "value": "", "effect": "NoSchedule"}
    arena = ks.objects.ObjectArena()
    nodes = [{"name": "gpu-0", "labels": {"gpu": "h100"},
              "allocatable": {"cpu": "64", "memory": str(512 << 30), "pods": "110", GPU: "8"}},
             {"name": "cpu-1", "allocatable": {"cpu": "16", "memory": str(64 << 30), "pods": "110"}},
             {"name": "cpu-2", "allocatable": {"cpu": "64", "memory": str(512 << 30), "pods": "110"}},
             {"name": "cpu-3", "allocatable": {"cpu": "48", "memory": str(384 << 30), "pods": "110"}}]
    on_gpu0 = [{"name": "trainer-0", "ns": "ml", "node_name": "gpu-0",
                "containers": [{"cpu": "32", "memory": str(256 << 30), GPU: "8"}]}]
    on_cpu1 = [{"name": f"web-{i}", "ns": "shop", "node_name": "cpu-1",
                "containers": [{"cpu": "2", "memory": str(4 << 30)}]} for i in range(2)]
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(nodes), 4)
        ctx.set_cluster_pods(arena.pods(on_gpu0 + on_cpu1), 3)
        ctx.set_node_taints({"gpu-0": [gpu_taint], "cpu-2": [cordon]})
        assert [ctx.node_name(i) for i in range(4)] == ["gpu-0", "cpu-1", "cpu-2", "cpu-3"]
        pods = arena.pods(on_gpu0 + on_cpu1)
        rules = [{"tolerations": [{"key": GPU, "operator": "Exists", "effect": "NoSchedule"}]}, {}]
        placed, node, refused = ctx.drain_fit_nodes(["gpu-0", "cpu-1"], pods, [0, 1, 3], [0, 1, 1], 2,
                                                    group_rules=rules)
        assert placed.tolist() == [0, 2] and node.tolist() == [-1, 3, 3]
        assert refused.tolist() == [[1, 2, 0, 0], [0, 0, 0, 0]]
        old_placed, old_node = ctx.drain_nodes(["gpu-0", "cpu-1"], pods, [0, 1, 3])
        assert old_placed.tolist() == [1, 2] and old_node.tolist() == [2, 2, 2]


def test_host_layer_end_to_end_after_events(ks):
    """ksh_drain_fit_nodes over objects (labels, taints, a cordon, allocatable pods and GPUs, running GPU pods) against
    the restatement over the same strings, after node, taint and pod events."""
    GPU = "nvidia.com/gpu"
    rng = np.random.default_rng(0xD8A1)
    taint = {"key": GPU, "value": "present", "effect": "NoSchedule"}
    nodes = {}
    for i in range(40):
        gpu = i % 4 == 3
        a = {"cpu": "16", "memory": str(64 << 30), "pods": str(int(rng.integers(3, 9)))}
        if gpu:
            a[GPU] = "8"
        nodes[f"n{i}"] = {"name": f"n{i}", "labels": {"zone": "abc"[i % 3], **({"gpu": "h100"} if gpu else {})},
                          "allocatable": a}
    taints = {nm: [taint] for nm, s in nodes.items() if GPU in s["allocatable"]}
    taints["n10"] = [fdo.CORDON]
    bound, bgroup = [], {}
    for i, nm in enumerate(nodes):
        for j in range(int(rng.integers(1, 4))):
            c = {"cpu": f"{int(rng.integers(1000, 4000))}m", "memory": str(int(rng.integers(1, 9)) << 30)}
            g = int(rng.integers(-1, 2))
            if GPU in nodes[nm]["allocatable"] and j < 2:
                c[GPU], g = "3", 0
            bound.append({"name": f"b{i}-{j}", "ns": "batch", "node_name": nm, "containers": [c]})
            bgroup[f"b{i}-{j}"] = g
    rules = [{"tolerations": [{"key": GPU, "operator": "Exists", "effect": "NoSchedule"}]},
             {"required": [[{"key": "zone", "operator": "In", "values": ["a", "b"]}]]}]
    arena = ks.objects.ObjectArena()
    cands = ["n3", "n0", "n7", "n3", "n21", "n10"]

    def ints(m):
        return {k: int(v) for k, v in m.items() if k not in ("cpu", "memory")}

    def check(ctx, mirror, policy=0, flags=0):
        specs, off = [], [0]
        for nm in cands:
            specs += [b for b in mirror if b["node_name"] == nm]
            off.append(len(specs))
        pods = arena.pods(specs)
        group = np.array([bgroup[b["name"]] for b in specs], np.int32)
        placed, node, refused = ctx.drain_fit_nodes(cands, pods, off, group, len(rules), group_rules=rules,
                                                    policy=policy, flags=flags)
        rc, rm, sel = ctx.pack_pods(pods, len(specs))
        ac, am, lab, bn, bc, bm = ctx.export_packed()
        order = [ctx.node_name(i) for i in range(ctx.n_nodes)]
        assert [b["node_name"] for b in mirror] == [order[n] for n in bn]
        d = dict(fc=ac.copy(), fm=am.copy(), ac=ac, am=am, labels=lab, sel=sel[:, :lab.shape[1]], rc=rc, rm=rm,
                 group=group, node_labels=[nodes[nm]["labels"] for nm in order],
                 node_taints=[taints.get(nm, []) for nm in order], group_rules=rules,
                 alloc=[ints(nodes[nm]["allocatable"]) for nm in order],
                 bound=[(int(n), ints(b["containers"][0])) for n, b in zip(bn, mirror)],
                 pod_res=[ints(b["containers"][0]) for b in specs])
        np.subtract.at(d["fc"], bn, bc)
        np.subtract.at(d["fm"], bn, bm)
        want = fdo.fit_drain(d, [order.index(nm) for nm in cands], np.array(off, np.uint64), policy, flags == 1)
        assert np.array_equal(placed, want[0]) and np.array_equal(node, want[1]) and np.array_equal(refused, want[3])
        return placed

    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(list(nodes.values())), len(nodes))
        ctx.set_node_taints(taints)
        ctx.set_cluster_pods(arena.pods(bound), len(bound))
        mirror = list(bound)
        for policy, flags in ((0, 0), (4, 1)):
            check(ctx, mirror, policy, flags)
        # a taint event: n3 leaves the GPU pool's taint, n5 is cordoned
        taints["n3"] = []
        taints["n5"] = [fdo.CORDON]
        ctx.set_node_taints({"n3": [], "n5": taints["n5"]})
        check(ctx, mirror)
        # a pod event: a running GPU pod deleted (swap-remove moves the last row into its place)
        k = next(i for i, b in enumerate(mirror) if GPU in b["containers"][0])
        ctx.pod_deleted(arena.pods([mirror[k]]))
        mirror[k] = mirror[-1]
        mirror.pop()
        check(ctx, mirror)
        # a node event: a GPU node's pod limit lowered
        nodes["n11"] = dict(nodes["n11"], allocatable=dict(nodes["n11"]["allocatable"], pods="1"))
        ctx.upsert_node(arena.nodes([nodes["n11"]]))
        check(ctx, mirror, 4, 1)
