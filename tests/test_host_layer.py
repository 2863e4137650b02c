"""Host layer (C++ behind include/ksched_host.h).  CPU part: the product's own quantity parser and
total_pod_resources against the golden KATs and against the oracle's independent implementation.
GPU part: object-level parity of check_node_validity / select_node_for_pod / reconcile with the faithful oracle."""
import ctypes as C
import json

import numpy as np
import pytest

from helpers import load_golden, mask_bits


def test_product_quantity_parser_matches_golden_and_oracle(ks, orc):
    kats = load_golden("quantity_kats.json")
    for s, want in kats["ok"]:
        rc_c, vc = ks.host.parse_cpu_millicores(s)
        orc_rc, ov = orc.parse_quantity(s)
        if isinstance(want, str):
            assert rc_c == {"INEXACT": -6, "RANGE": -5}[want], s
            continue
        assert orc_rc == 0 and rc_c == 0 and vc == want == ov, s   # cpu unit = 1/1000 = oracle unit
        rc_m, vm = ks.host.parse_memory_bytes(s)
        if want % 1000 == 0:
            assert rc_m == 0 and vm == want // 1000, s
        else:
            assert rc_m == -6, s                                    # sub-byte memory is outside the exact domain
    for s in kats["bad"]:
        assert ks.host.parse_cpu_millicores(s)[0] == -3, s
        assert ks.host.parse_memory_bytes(s)[0] == -3, s


def test_total_pod_resources_and_is_pod_bound_match_oracle(ks, orc):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    pods = arena.pods(g["pods"] + g["bound_pods"])
    for i in range(len(g["pods"])):
        rc, c, m = ks.host.total_pod_resources(pods, i)
        assert (rc, c, m) == (0, g["expected_req_cpu_milli"][i], g["expected_req_mem_bytes"][i])
    for i in range(len(g["pods"]) + len(g["bound_pods"])):
        out = (C.c_int64 * 2)()
        assert orc.lib.orc_total_pod_resources(C.addressof(pods) + i * C.sizeof(pods._type_), out) == 0
        rc, c, m = ks.host.total_pod_resources(pods, i)
        assert (c, m * 1000) == (out[0], out[1])
        assert ks.host.is_pod_bound(pods, i) == bool(orc.lib.orc_is_pod_bound(C.addressof(pods) + i * C.sizeof(pods._type_)))


def test_random_object_totals_match_packed_generator(ks, orc):
    cl = ks.synth.make(200, 50, seed=3)
    _, bound_s, pods_s = ks.objects.cluster_specs(cl)
    arena = ks.objects.ObjectArena()
    pods, bound = arena.pods(pods_s), arena.pods(bound_s)
    for p in range(cl.P):
        assert ks.host.total_pod_resources(pods, p) == (0, cl.req_cpu[p], cl.req_mem[p])
    for b in range(0, cl.B, 7):
        assert ks.host.total_pod_resources(bound, b) == (0, cl.bound_cpu[b], cl.bound_mem[b])


def test_malformed_objects_are_status_codes(ks):
    arena = ks.objects.ObjectArena()
    pods = arena.pods([{"name": "a", "containers": [{"cpu": "one"}]}, {"name": "b", "containers": [{"memory": "1.5"}]}])
    assert ks.host.total_pod_resources(pods, 0)[0] == -3
    assert ks.host.total_pod_resources(pods, 1)[0] == -6
    assert b"memory quantity" in ks.lib.ks_last_error()


# ------------------------------------------------------------------------------------------------ packer, CPU
# A packing-only context (KSH_DEVICE_NONE) turns objects into the SoA / bitmask arrays the device consumes and never
# evaluates a predicate.  The CPU suite checks those arrays by giving them to the oracle's packed flavour and
# comparing with the oracle's object-model (faithful) flavour on the same objects.
def _packed_answer(orc, ctx, pods, P, policy=0):
    rc, rm, sel = ctx.pack_pods(pods, P)           # grows the label dictionary first
    ac, am, lab, bn, bc, bm = ctx.export_packed()   # ... so the node label words use the final dictionary
    assert lab.shape[1] == sel.shape[1] == ctx.label_words
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    return orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, policy=policy, want_codes=True)


def _objects(ks, cl):
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    arena = ks.objects.ObjectArena()
    return arena, arena.nodes(nodes_s), arena.pods(bound_s), arena.pods(pods_s)


@pytest.mark.parametrize("P,N,keys,policy", [(64, 200, 8, 0), (300, 1500, 8, 0), (40, 300, 32, 1), (1, 1, 8, 0)])
def test_packer_output_equals_faithful_oracle(ks, orc, P, N, keys, policy):
    cl = ks.synth.make(P, N, seed=900 + P, n_keys=keys, bound_per_node=3)
    arena, nodes, bound, pods = _objects(ks, cl)
    oc = orc.Cluster(nodes, cl.N, bound, cl.B)
    want = oc.run(pods, P, policy=policy, want_codes=True)
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(nodes, cl.N)
        ctx.set_cluster_pods(bound, cl.B)
        got = _packed_answer(orc, ctx, pods, P, policy)
        assert ctx.label_words <= max(1, cl.label_words)  # only pairs that selectors name get a bit
        ac, am, _, bn, bc, bm = ctx.export_packed()
    for g, w, name in zip(got, want, ("node_idx", "score", "feasible_cnt", "mask", "codes")):
        assert np.array_equal(g, w), name
    # and the numeric columns are the generator's own packed form
    gac, gam, _, gbn, gbc, gbm, _, _, _ = cl.packed()
    assert np.array_equal(ac, gac) and np.array_equal(am, gam)
    assert np.array_equal(bn, gbn) and np.array_equal(bc, gbc) and np.array_equal(bm, gbm)


def test_packer_gv1_and_reference_selector_tests(ks, orc):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(g["nodes"]), arena.pods(g["bound_pods"]), arena.pods(g["pods"])
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(nodes, len(g["nodes"]))
        ctx.set_cluster_pods(bound, len(g["bound_pods"]))
        rc, rm, _ = ctx.pack_pods(pods, len(g["pods"]))
        assert rc.tolist() == g["expected_req_cpu_milli"] and rm.tolist() == g["expected_req_mem_bytes"]
        _, _, _, mask, _ = _packed_answer(orc, ctx, pods, len(g["pods"]))
        ac, am, _, bn, bc, bm = ctx.export_packed()
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    assert fc.tolist() == g["expected_free_cpu_milli"] and fm.tolist() == g["expected_free_mem_bytes"]
    from helpers import rows_to_str
    assert rows_to_str(mask_bits(mask, len(g["nodes"]))) == g["expected_feasible_rows"]
    # the reference's own three nodeSelector tests (src/predicates/test.rs:42-58) through the packer
    k = load_golden("selector_kats.json")
    for case in k["cases"]:
        n_, p_ = arena.nodes([case["node"]]), arena.pods([case["pod"]])
        with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
            ctx.set_nodes(n_, 1)
            _, _, sel = ctx.pack_pods(p_, 1)
            lab = ctx.export_packed()[2]
        match = not np.any(sel[0] & ~lab[0])
        assert match == case["expect"], case["id"]


def test_packer_incremental_events_equal_a_rebuild(ks, orc):
    cl = ks.synth.make(120, 40, seed=11, bound_per_node=2)
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    arena = ks.objects.ObjectArena()
    pods = arena.pods(pods_s)
    first_bound_s = [b for b in bound_s if int(b["node_name"].split("-")[1]) < 30]
    rest_bound_s = [b for b in bound_s if int(b["node_name"].split("-")[1]) >= 30]
    changed = dict(nodes_s[5])
    changed["allocatable"] = {"cpu": "128", "memory": str(1 << 40)}
    gone = [b for b in first_bound_s if b["node_name"] == "node-3"][:2]
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(nodes_s[:30]), 30)
        ctx.set_cluster_pods(arena.pods(first_bound_s), len(first_bound_s))
        ctx.pack_pods(pods, cl.P)  # dictionary exists before the events: it must survive them
        rest_nodes = arena.nodes(nodes_s[30:])
        for i in range(10):
            assert ctx.upsert_node(rest_nodes, i) == 30 + i
        rest_bound = arena.pods(rest_bound_s)
        for i in range(len(rest_bound_s)):
            ctx.pod_bound(rest_bound, i)
        assert ctx.upsert_node(arena.nodes([changed])) == 5
        ctx.remove_node("node-7")
        gone_objs = arena.pods(gone)
        for i in range(len(gone)):
            ctx.pod_deleted(gone_objs, i)
        ctx.pod_deleted(arena.pods([{"name": "never-seen", "ns": "x", "node_name": "node-1"}]))  # ignored
        assert ctx.n_nodes == 39 and ctx.node_name(7) == "node-8" and ctx.node_name(39) is None
        got = _packed_answer(orc, ctx, pods, cl.P)
    final_nodes_s = [changed if n["name"] == "node-5" else n for n in nodes_s if n["name"] != "node-7"]
    gone_names = {g_["name"] for g_ in gone}
    final_bound_s = [b for b in bound_s if b["node_name"] != "node-7" and b["name"] not in gone_names]
    oc = orc.Cluster(arena.nodes(final_nodes_s), len(final_nodes_s), arena.pods(final_bound_s), len(final_bound_s))
    want = oc.run(pods, cl.P, want_codes=True)
    for g_, w, name in zip(got, want, ("node_idx", "score", "feasible_cnt", "mask", "codes")):
        assert np.array_equal(g_, w), name


def test_packing_only_context_never_computes(ks):
    cl = ks.synth.make(4, 6, seed=1)
    arena, nodes, bound, pods = _objects(ks, cl)
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(nodes, cl.N)
        for call in (lambda: ctx.check_node_validity(pods, 0, 0), lambda: ctx.select_nodes(pods, 4),
                     lambda: ctx.select_node_for_pod(pods, 4), lambda: ctx.reconcile(pods, 0)):
            with pytest.raises(ks.KsError) as e:
                call()
            assert e.value.code == -8  # KS_ERR_NO_DEVICE


# ------------------------------------------------------------------------------------------------ GPU
def _cluster_objects(ks, cl):
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    arena = ks.objects.ObjectArena()
    return arena, arena.nodes(nodes_s), arena.pods(bound_s), arena.pods(pods_s)


@pytest.mark.gpu
@pytest.mark.parametrize("P,N,keys,policy", [(64, 200, 8, 0), (300, 1500, 8, 0), (40, 300, 32, 1)])
def test_select_nodes_objects_vs_faithful_oracle(ks, orc, P, N, keys, policy):
    cl = ks.synth.make(P, N, seed=900 + P, n_keys=keys, bound_per_node=3)
    arena, nodes, bound, pods = _cluster_objects(ks, cl)
    oc = orc.Cluster(nodes, cl.N, bound, cl.B)
    oidx, oscore, ocnt, _, ocodes = oc.run(pods, P, policy=policy, want_codes=True)
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, cl.N)
        ctx.set_cluster_pods(bound, cl.B)
        idx, score, cnt = ctx.select_nodes(pods, P, policy=policy)
        assert np.array_equal(idx, oidx) and np.array_equal(score, oscore) and np.array_equal(cnt, ocnt)
        # the dictionary only holds pairs that selectors name: far fewer bits than node label pairs
        assert ctx.label_words <= max(1, cl.label_words)
        for p in range(0, P, 7):
            for n in range(0, N, 13):
                assert ctx.check_node_validity(pods, p, n) == ocodes[p, n]


@pytest.mark.gpu
def test_gv1_objects_through_host_layer(ks, orc):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    nodes, allp, pods = arena.nodes(g["nodes"]), arena.pods(g["bound_pods"]), arena.pods(g["pods"])
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, 5)
        ctx.set_cluster_pods(allp, len(g["bound_pods"]))
        idx, score, cnt = ctx.select_nodes(pods, 10)
        assert list(idx) == g["expected_node_idx_leftover"]
        assert list(cnt) == [r.count("1") for r in g["expected_feasible_rows"]]
        rows = ["".join("1" if ctx.check_node_validity(pods, p, n) == 0 else "0" for n in range(5)) for p in range(10)]
        assert rows == g["expected_feasible_rows"]


@pytest.mark.gpu
def test_reference_selector_tests_through_host_layer(ks):
    """The reference's three tests (src/predicates/test.rs:42-58) on the GPU path: node without status has
    (0,0) allocatable and the fixture pods request nothing, so fit holds and the code isolates the selector."""
    for case in load_golden("selector_kats.json")["cases"]:
        arena = ks.objects.ObjectArena()
        pods, nodes = arena.pods([case["pod"]]), arena.nodes([case["node"]])
        with ks.host.Context(0) as ctx:
            ctx.set_nodes(nodes, 1)
            code = ctx.check_node_validity(pods, 0, 0)
        assert (code == 0) == case["expect"], case["id"]
        assert code in (0, 2)


@pytest.mark.gpu
def test_reconcile_mirror(ks, orc):
    arena = ks.objects.ObjectArena()
    nodes = arena.nodes([{"name": "small", "allocatable": {"cpu": "1", "memory": "1000"}},
                         {"name": "big \"quoted\"", "allocatable": {"cpu": "2", "memory": "4000"}, "labels": {"d": "x"}}])
    pods = arena.pods([
        {"name": "a", "ns": "ns1", "containers": [{"cpu": "1500m", "memory": "3000"}]},
        {"name": "b", "ns": "ns1", "containers": [{"cpu": "600m", "memory": "10"}]},
        {"name": "c", "ns": "ns1", "containers": [{"cpu": "600m", "memory": "10"}]},
        {"name": "bound", "ns": "ns1", "node_name": "small", "containers": [{"cpu": "9", "memory": "9"}]},
        {"name": "sel", "ns": "ns1", "containers": [], "selector": {"d": "y"}},
    ])
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, 2)
        ctx.set_cluster_pods(arena.pods([]), 0)
        rc, node, js = ctx.reconcile(pods, 0)
        assert (rc, node) == (0, 1)
        doc = json.loads(js)
        assert doc == {"apiVersion": "v1", "kind": "Binding", "metadata": {"name": "a", "namespace": "ns1"},
                       "target": {"name": "big \"quoted\""}}
        # capacity was committed: 'big' now has 500m/1000 left, so b goes to 'small', and c fits nowhere
        assert ctx.reconcile(pods, 1)[:2] == (0, 0)
        assert ctx.reconcile(pods, 2)[:2] == (ks.host.KSH_RECONCILE_NO_NODE_FOUND, -1)
        assert ctx.reconcile(pods, 3) == (0, -1, "")          # already bound -> await_change, no binding
        assert ctx.reconcile(pods, 4)[:2] == (ks.host.KSH_RECONCILE_NO_NODE_FOUND, -1)


@pytest.mark.gpu
def test_reconcile_retry_does_not_leak_capacity(ks, orc):
    """A pod that comes back unbound (the caller's POST failed or raced, error_policy requeued it; src/main.rs:105-108,
    :122-125) must not be charged twice: the reference's LIST would never show the failed binding."""
    arena = ks.objects.ObjectArena()
    nodes = arena.nodes([{"name": "n0", "allocatable": {"cpu": "2", "memory": "4000"}},
                         {"name": "n1", "allocatable": {"cpu": "1", "memory": "4000"}}])
    pods = arena.pods([{"name": "a", "ns": "d", "containers": [{"cpu": "1500m", "memory": "1000"}],
                        "metadata_json": '{"name":"a","namespace":"d","uid":"u-1","labels":{"app":"x"}}'},
                       {"name": "b", "ns": "d", "containers": [{"cpu": "1500m", "memory": "1000"}]}])
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, 2)
        ctx.set_cluster_pods(arena.pods([]), 0)
        for _ in range(3):  # the same pod reconciled three times: one row, one charge, always the same answer
            rc, node, js = ctx.reconcile(pods, 0)
            assert (rc, node) == (0, 0) and ctx.num_bound == 1
        # metadata passthrough: the Binding carries the pod's whole ObjectMeta (src/main.rs:88 metadata: pod.metadata.clone())
        assert json.loads(js) == {"apiVersion": "v1", "kind": "Binding", "target": {"name": "n0"},
                                  "metadata": {"name": "a", "namespace": "d", "uid": "u-1", "labels": {"app": "x"}}}
        assert ctx.reconcile(pods, 1)[:2] == (ks.host.KSH_RECONCILE_NO_NODE_FOUND, -1)  # n0 has 500m left, n1 1000m
        ctx.pod_deleted(pods, 0)
        assert ctx.num_bound == 0
        assert ctx.reconcile(pods, 1)[:2] == (0, 0)  # the whole of n0 is back
        # the batch form: a pod of the batch that this context bound earlier is released first, too
        st, nd, _, _ = ctx.reconcile_batch(pods, 2)
        assert ctx.num_bound == 1 and sorted(nd.tolist()) == [-1, 0]
        # duplicate keys in a LIST result: the last row wins, nothing is charged twice
        dup = arena.pods([{"name": "x", "ns": "d", "node_name": "n0", "containers": [{"cpu": "1"}]},
                          {"name": "x", "ns": "d", "node_name": "n0", "containers": [{"cpu": "1"}]}])
        ctx.set_cluster_pods(dup, 2)
        assert ctx.num_bound == 1
        assert ctx.reconcile(pods, 1)[:2] == (ks.host.KSH_RECONCILE_NO_NODE_FOUND, -1)  # n0: 1000m left < 1500m


@pytest.mark.gpu
def test_reconcile_batch_equals_the_streaming_oracle(ks, orc):
    """A drained queue through ksh_reconcile_batch: bound pods skipped, nameless pods refused, the rest bound by the
    micro-batch loop exactly as the oracle's restatement binds the packed batch; every bind is committed (device
    capacity, bound-pod list, Binding body) and visible to what follows."""
    cl = ks.synth.make(400, 25, seed=321, bound_per_node=2)        # few nodes: pods compete, several rounds
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    pods_s = [dict(p) for p in pods_s]
    pods_s[7] = dict(pods_s[7], node_name="node-3")                 # already bound -> skipped
    pods_s[11] = {"name": None, "ns": None, "containers": [{"cpu": "1m"}]}  # no namespace/name -> refused
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(nodes_s), arena.pods(bound_s), arena.pods(pods_s)
    todo = [i for i in range(cl.P) if i not in (7, 11)]
    # expectation: the packer's arrays (packing-only context) through the oracle's streaming restatement
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as pk:
        pk.set_nodes(nodes, cl.N)
        pk.set_cluster_pods(bound, cl.B)
        rc, rm, sel = pk.pack_pods(arena.pods([pods_s[i] for i in todo]), len(todo))
        ac, am, lab, bn, bc, bm = pk.export_packed()
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    oidx, _, orounds = orc.stream_bind_packed(fc, fm, ac, am, lab, rc, rm, sel)
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, cl.N)
        ctx.set_cluster_pods(bound, cl.B)
        status, node, bodies, rounds = ctx.reconcile_batch(pods, cl.P)
        assert rounds == orounds and rounds > 1
        assert (status[7], node[7], bodies[7]) == (0, -1, None)
        assert (status[11], node[11]) == (ks.host.KSH_RECONCILE_BINDING_OBJECT_FAILED, -1)
        assert np.array_equal(node[todo], oidx)
        assert np.array_equal(status[todo], np.where(oidx >= 0, 0, ks.host.KSH_RECONCILE_NO_NODE_FOUND))
        assert (oidx >= 0).any() and (oidx < 0).any()
        for i in todo[:50]:
            if node[i] >= 0:
                assert json.loads(bodies[i]) == {"apiVersion": "v1", "kind": "Binding",
                                                 "metadata": {"name": pods_s[i]["name"], "namespace": pods_s[i].get("ns", "default")},
                                                 "target": {"name": nodes_s[node[i]]["name"]}}
            else:
                assert bodies[i] is None
        # the binds are in the context's bound-pod list and in the device capacity
        xn, xc, xm = ctx.export_packed()[3:]
        assert len(xn) == cl.B + int((oidx >= 0).sum())
        f2c, f2m = orc.free_reduce(ac, am, xn, xc, xm)
        assert np.array_equal(f2c, fc) and np.array_equal(f2m, fm)  # fc/fm were advanced in place by the oracle
        later = arena.pods([{"name": "later", "ns": "d", "containers": [{"cpu": "1m", "memory": "1"}]}])
        feas = (f2c >= 1) & (f2m >= 1)
        want = int(np.argmax(np.where(feas, f2c * (1 << 22) + f2m, np.iinfo(np.int64).min))) if feas.any() else -1
        assert ctx.select_nodes(later, 1)[0][0] == want
        # a second drain of the same queue (the caller's POSTs failed and every pod was requeued): the earlier bindings of
        # these pods are released first, so each pod is charged once, and capacity is never oversubscribed
        status2, node2, _, _ = ctx.reconcile_batch(pods, cl.P)
        xn2, xc2, xm2 = ctx.export_packed()[3:]
        f3c, f3m = orc.free_reduce(ac, am, xn2, xc2, xm2)
        newly = np.nonzero(node2 >= 0)[0]
        assert ((f3c >= 0) | (fc < 0)).all() and ((f3m >= 0) | (fm < 0)).all(), "capacity oversubscribed by the second drain"
        assert len(xn2) == cl.B + len(newly)
        # a tiny Binding buffer: binds still happen, bodies that do not fit are reported as missing
        tiny = arena.pods([{"name": "t1", "ns": "d"}, {"name": "t2", "ns": "d"}])
        st, nd, bd, _ = ctx.reconcile_batch(tiny, 2, json_cap=120)
        assert (st == 0).all() and bd[0] is not None and bd[1] is None


@pytest.mark.gpu
def test_incremental_node_and_pod_events_equal_a_rebuilt_context(ks, orc):
    """upsert/remove node and pod bound/deleted events must leave the context in the state a full rebuild from the
    final objects gives (compared through the faithful oracle on that final cluster)."""
    cl = ks.synth.make(120, 40, seed=11, bound_per_node=2)
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    arena = ks.objects.ObjectArena()
    pods = arena.pods(pods_s)
    # start from the first 30 nodes and their bound pods
    first_nodes = arena.nodes(nodes_s[:30])
    first_bound_s = [b for b in bound_s if int(b["node_name"].split("-")[1]) < 30]
    first_bound = arena.pods(first_bound_s)
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(first_nodes, 30)
        ctx.set_cluster_pods(first_bound, len(first_bound_s))
        # events: 10 more nodes, their bound pods, one node changes size, one node goes away, two pods are deleted
        rest_nodes = arena.nodes(nodes_s[30:])
        for i in range(10):
            assert ctx.upsert_node(rest_nodes, i) == 30 + i
        rest_bound_s = [b for b in bound_s if int(b["node_name"].split("-")[1]) >= 30]
        rest_bound = arena.pods(rest_bound_s)
        for i in range(len(rest_bound_s)):
            ctx.pod_bound(rest_bound, i)
        changed = dict(nodes_s[5])
        changed["allocatable"] = {"cpu": "128", "memory": str(1 << 40)}
        assert ctx.upsert_node(arena.nodes([changed])) == 5
        ctx.remove_node("node-7")
        gone = [b for b in first_bound_s if b["node_name"] == "node-3"][:2]
        gone_objs = arena.pods(gone)
        for i in range(len(gone)):
            ctx.pod_deleted(gone_objs, i)
        ctx.pod_deleted(arena.pods([{"name": "never-seen", "ns": "x", "node_name": "node-1"}]))  # ignored
        assert ctx.n_nodes == 39 and ctx.node_name(7) == "node-8" and ctx.node_name(39) is None
        idx, score, cnt = ctx.select_nodes(pods, cl.P)
        names = [ctx.node_name(i) if i >= 0 else None for i in idx]
    # the same final cluster, built from scratch, through the faithful oracle
    final_nodes_s = [changed if n["name"] == "node-5" else n for n in nodes_s if n["name"] != "node-7"]
    gone_names = {g["name"] for g in gone}
    final_bound_s = [b for b in bound_s if b["node_name"] != "node-7" and b["name"] not in gone_names]
    fn, fb = arena.nodes(final_nodes_s), arena.pods(final_bound_s)
    oc = orc.Cluster(fn, len(final_nodes_s), fb, len(final_bound_s))
    oidx, oscore, ocnt, _, _ = oc.run(pods, cl.P)
    assert np.array_equal(idx, oidx) and np.array_equal(score, oscore) and np.array_equal(cnt, ocnt)
    assert names == [final_nodes_s[i]["name"] if i >= 0 else None for i in oidx]


_THREAD_SNIPPET = r"""
import hashlib, sys
sys.path.insert(0, %r)
import ksched_pkg
ks = ksched_pkg.load()
cl = ks.synth.make(30000, 3000, seed=77, n_keys=32, bound_per_node=10)
nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
arena = ks.objects.ObjectArena()
nodes, bound, pods = arena.nodes(nodes_s), arena.pods(bound_s), arena.pods(pods_s)
h = hashlib.sha256()
with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
    ctx.set_nodes(nodes, cl.N)
    ctx.set_cluster_pods(bound, cl.B)
    for a in ctx.pack_pods(pods, cl.P) + ctx.export_packed():
        h.update(a.tobytes())
    w = ctx.label_words
    bad = list(pods_s)
    bad[20000] = dict(bad[20000], containers=[{"cpu": "two"}])
    bad[5000] = dict(bad[5000], containers=[{"memory": "1.5"}])
    try:
        ctx.pack_pods(arena.pods(bad), cl.P)
        err = "no error"
    except ks.KsError as e:
        err = "%%d %%s" %% (e.code, str(e).split(": ", 1)[1])
print(h.hexdigest(), w, err)
"""


def test_packer_is_identical_for_any_thread_count(ks):
    """Bulk calls run on all host threads; dictionary bits, packed arrays and the reported error (the first failing
    object in array order) must not depend on how many there are."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    outs = []
    for threads in ("1", "3", "8"):
        env = dict(os.environ, KSH_THREADS=threads)
        r = subprocess.run([sys.executable, "-c", _THREAD_SNIPPET % root], capture_output=True, text=True, env=env, timeout=600)
        assert r.returncode == 0, r.stderr
        outs.append(r.stdout.strip())
    assert outs[0] == outs[1] == outs[2], outs
    assert " -6 " in outs[0] and "1.5" in outs[0]  # pod 5000 (memory '1.5', KS_ERR_INEXACT), not pod 20000


def test_packer_event_fuzz_against_a_model(ks, orc):
    """Random informer events (node upsert / remove, pod bound / re-bound / deleted) on a packing-only context vs a
    plain Python model of the cluster; the final state is compared through the faithful oracle."""
    rng = np.random.default_rng(2024)
    cl = ks.synth.make(150, 60, seed=5, bound_per_node=3)
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    arena = ks.objects.ObjectArena()
    pods = arena.pods(pods_s)
    model_nodes = [dict(n) for n in nodes_s[:20]]          # ordered: index = position
    model_bound = {}                                       # (ns, name) -> spec
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(model_nodes), len(model_nodes))
        ctx.set_cluster_pods(arena.pods([]), 0)
        spare_nodes = [dict(n) for n in nodes_s[20:]]
        spare_bound = [dict(b) for b in bound_s]
        for step in range(1500):
            ev = rng.integers(0, 100)
            names = [n["name"] for n in model_nodes]
            if ev < 10 and spare_nodes:                                     # new node
                n = spare_nodes.pop()
                assert ctx.upsert_node(arena.nodes([n])) == len(model_nodes)
                model_nodes.append(n)
            elif ev < 20 and model_nodes:                                   # node changes (size and a label)
                i = int(rng.integers(0, len(model_nodes)))
                n = dict(model_nodes[i])
                n["allocatable"] = {"cpu": str(int(rng.integers(1, 64))), "memory": str(int(rng.integers(1, 64)) << 30)}
                lab = dict(n.get("labels") or {})
                lab["key0"] = f"v{int(rng.integers(0, 8))}"
                n["labels"] = lab
                assert ctx.upsert_node(arena.nodes([n])) == i
                model_nodes[i] = n
            elif ev < 25 and len(model_nodes) > 5:                          # node goes away, with its pods
                i = int(rng.integers(0, len(model_nodes)))
                gone = model_nodes.pop(i)
                ctx.remove_node(gone["name"])
                spare_nodes.append(gone)
                for k in [k for k, b in model_bound.items() if b["node_name"] == gone["name"]]:
                    del model_bound[k]
            elif ev < 75 and spare_bound and names:                         # pod bound (new, or an update of a known pod)
                b = dict(spare_bound[int(rng.integers(0, len(spare_bound)))])
                b["node_name"] = names[int(rng.integers(0, len(names)))]
                ctx.pod_bound(arena.pods([b]))
                model_bound[(b.get("ns"), b["name"])] = b
            elif model_bound:                                               # pod deleted
                keys = list(model_bound)
                k = keys[int(rng.integers(0, len(keys)))]
                ctx.pod_deleted(arena.pods([model_bound.pop(k)]))
            if step % 250 == 249:
                ctx.pack_pods(pods, cl.P)                                   # dictionary grows in between, too
        assert ctx.n_nodes == len(model_nodes)
        assert [ctx.node_name(i) for i in range(ctx.n_nodes)] == [n["name"] for n in model_nodes]
        got = _packed_answer(orc, ctx, pods, cl.P)
    fb = list(model_bound.values())
    oc = orc.Cluster(arena.nodes(model_nodes), len(model_nodes), arena.pods(fb), len(fb))
    want = oc.run(pods, cl.P, want_codes=True)
    for g_, w, name in zip(got, want, ("node_idx", "score", "feasible_cnt", "mask", "codes")):
        assert np.array_equal(g_, w), name


def test_packer_dictionary_compaction_and_duplicate_names(ks):
    arena = ks.objects.ObjectArena()
    alloc = {"cpu": "4", "memory": str(1 << 30)}
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes([{"name": "a", "labels": {"gen": "g0"}, "allocatable": alloc}]), 1)
        # 700 generations of a label: each gets a dictionary bit when a selector names it, the old ones go stale and
        # must be reclaimed instead of overflowing the 511-pair dictionary
        for g in range(700):
            ctx.upsert_node(arena.nodes([{"name": "a", "labels": {"gen": f"g{g}"}, "allocatable": alloc}]))
            want = arena.pods([{"name": "p", "ns": "d", "selector": {"gen": f"g{g}"}},
                               {"name": "q", "ns": "d", "selector": {"gen": f"g{max(g - 1, 0)}"}}])
            _, _, sel = ctx.pack_pods(want, 2)
            lab = ctx.export_packed()[2]
            assert not np.any(sel[0] & ~lab[0])                      # current generation matches
            assert (g == 0) or np.any(sel[1] & ~lab[0])              # the previous one no longer does
        assert ctx.label_words <= 8
        # duplicate names: the first row of a name is the one events and pods address
        ctx.set_nodes(arena.nodes([{"name": "x", "allocatable": alloc}, {"name": "y", "allocatable": alloc},
                                   {"name": "x", "allocatable": alloc}]), 3)
        ctx.pod_bound(arena.pods([{"name": "b", "ns": "d", "node_name": "x", "containers": [{"cpu": "1"}]}]))
        assert ctx.export_packed()[3].tolist() == [0]
        ctx.remove_node("x")                                         # removes row 0; the other "x" is now row 1
        assert [ctx.node_name(i) for i in range(ctx.n_nodes)] == ["y", "x"] and ctx.export_packed()[3].size == 0
        ctx.pod_bound(arena.pods([{"name": "b", "ns": "d", "node_name": "x", "containers": [{"cpu": "1"}]}]))
        ctx.pod_bound(arena.pods([{"name": "b", "ns": "d", "node_name": "y", "containers": [{"cpu": "2"}]}]))  # moved
        bn, bc = ctx.export_packed()[3], ctx.export_packed()[4]
        assert bn.tolist() == [0] and bc.tolist() == [2000]
        assert ctx.upsert_node(arena.nodes([{"name": "z", "allocatable": alloc}])) == 2
        ctx.remove_node("z")
        assert ctx.upsert_node(arena.nodes([{"name": "z", "allocatable": alloc}])) == 2  # a removed name comes back as new


def test_packer_dictionary_is_rebuilt_from_the_batch_when_full(ks):
    """More than 511 distinct (key,value) pairs named by selectors over a context's lifetime while every pair stays
    live on some node (hostname selectors): later batches must still pack - the dictionary only has to cover the
    pairs of the current batch."""
    arena = ks.objects.ObjectArena()
    alloc = {"cpu": "4", "memory": str(1 << 30)}
    n = 700
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes([{"name": f"n{i}", "labels": {"kubernetes.io/hostname": f"n{i}", "zone": f"z{i % 3}"},
                                    "allocatable": alloc} for i in range(n)]), n)
        for lo in range(0, n, 100):  # 7 batches x 100 hostname selectors: 700 live pairs over time
            want = arena.pods([{"name": f"p{i}", "ns": "d", "selector": {"kubernetes.io/hostname": f"n{i}", "zone": f"z{i % 3}"}}
                               for i in range(lo, lo + 100)] + [{"name": "plain", "ns": "d"}])
            _, _, sel = ctx.pack_pods(want, 101)
            lab = ctx.export_packed()[2]
            assert ctx.label_words <= 8 and not sel[100].any()
            for k in range(100):  # pod k matches exactly node lo+k
                match = ~np.any(sel[k][None, :] & ~lab, axis=1)
                assert np.nonzero(match)[0].tolist() == [lo + k]
        # one batch that names more live pairs than the dictionary can hold is refused with a clear status
        big = arena.pods([{"name": f"p{i}", "ns": "d", "selector": {"kubernetes.io/hostname": f"n{i}"}} for i in range(600)])
        with pytest.raises(ks.KsError, match="split the batch"):
            ctx.pack_pods(big, 600)


def test_packer_survives_long_churn(ks, orc):
    """Label values, node names and pods that come and go for a long time (the garbage collection of the interned
    strings runs many times on the way) leave exactly the state of the final objects."""
    arena = ks.objects.ObjectArena()
    alloc = {"cpu": "64", "memory": str(256 << 30)}
    base = [{"name": f"keep-{i}", "labels": {"zone": f"z{i % 3}"}, "allocatable": alloc} for i in range(8)]
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(base), len(base))
        live = {}
        for g in range(6000):
            a = ks.objects.ObjectArena()  # short-lived objects, like the host's own
            base[g % 8] = dict(base[g % 8], labels={"zone": f"z{g % 3}", "rev": f"r{g}"})
            ctx.upsert_node(a.nodes([base[g % 8]]))
            tmp = {"name": f"tmp-{g}", "labels": {"rev": f"t{g}"}, "allocatable": alloc}
            assert ctx.upsert_node(a.nodes([tmp])) == 8
            pod = {"name": f"job-{g}", "ns": "batch", "node_name": f"tmp-{g}" if g % 2 else f"keep-{g % 8}",
                   "containers": [{"cpu": "100m", "memory": "1048576"}]}
            ctx.pod_bound(a.pods([pod]))
            ctx.remove_node(f"tmp-{g}")                    # takes the pods bound to it along
            if g % 2 == 0:
                live[pod["name"]] = pod
            if g % 3 == 0 and live:
                k = next(iter(live))
                ctx.pod_deleted(a.pods([live.pop(k)]))
            if g % 500 == 0:
                ctx.pack_pods(a.pods([{"name": "s", "ns": "d", "selector": {"rev": f"r{g}"}}]), 1)
        for g in range(20000):                             # key arena churn: long pod names bound and deleted
            a = ks.objects.ObjectArena()
            pod = {"name": f"burst-{g}-" + "x" * 40, "ns": "batch", "node_name": f"keep-{g % 8}", "containers": [{"cpu": "1m"}]}
            ctx.pod_bound(a.pods([pod]))
            if g % 1000:
                ctx.pod_deleted(a.pods([pod]))
            else:
                live[pod["name"]] = pod
        assert ctx.n_nodes == 8
        pods_s = [{"name": "a", "ns": "d", "selector": {"rev": "r5999"}, "containers": [{"cpu": "1"}]},
                  {"name": "b", "ns": "d", "selector": {"rev": "r5991"}},           # a label value of the past
                  {"name": "c", "ns": "d", "selector": {"zone": "z0"}, "containers": [{"cpu": "63950m"}]},
                  {"name": "d", "ns": "d"}]
        pods = arena.pods(pods_s)
        got = _packed_answer(orc, ctx, pods, len(pods_s))
    fb = list(live.values())
    oc = orc.Cluster(arena.nodes(base), len(base), arena.pods(fb), len(fb))
    want = oc.run(pods, len(pods_s), want_codes=True)
    for g_, w, name in zip(got, want, ("node_idx", "score", "feasible_cnt", "mask", "codes")):
        assert np.array_equal(g_, w), name
    assert got[2].tolist()[1] == 0 and got[2].tolist()[0] == 1


def test_host_layer_under_sanitizers(tmp_path):
    """csrc/host/ksh_host.cpp built alone (device calls stubbed) with ASan+UBSan: 300k random events against a model,
    the threaded bulk calls (pack_bench) and four threads sharing one context with ThreadSanitizer."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "kube-scheduler-rs-reference_b200", "csrc", "host", "ksh_host.cpp")
    stub = os.path.join(root, "tests", "native", "ksh_stub_device.cpp")
    inc = "-I" + os.path.join(root, "include")
    jobs = [("address,undefined", os.path.join(root, "tests", "native", "ksh_churn.cpp"), [], "churn ok"),
            ("thread", os.path.join(root, "examples", "pack_bench.cpp"), ["2000", "20000", "20000"], "host_packer_objects_per_sec"),
            ("thread", os.path.join(root, "tests", "native", "ksh_concurrent.cpp"), [], "concurrent ok")]
    for san, main_src, args, expect in jobs:
        exe = str(tmp_path / ("t_" + san.split(",")[0] + "_" + os.path.basename(main_src).split(".")[0]))
        r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=" + san, inc, src, stub, main_src, "-pthread", "-o", exe],
                           capture_output=True, text=True)
        if r.returncode != 0 and "sanitize" in r.stderr:
            pytest.skip("sanitizer runtime not available: " + r.stderr.splitlines()[0])
        assert r.returncode == 0, r.stderr
        r = subprocess.run([exe] + args, capture_output=True, text=True, timeout=600, env=dict(os.environ, KSH_THREADS="4"))
        assert r.returncode == 0 and expect in r.stdout, (r.stdout, r.stderr)
        assert "Sanitizer" not in r.stderr and "runtime error" not in r.stderr, r.stderr


def test_object_level_host_layer_against_a_fake_device(tmp_path):
    """The -m gpu host-layer tests (objects -> pack -> device calls -> results, reconcile, events, the reference's
    sampling policy) run here against a scratch libksched.so = the real csrc/host/ksh_host.cpp + a fake device that
    answers the ks_* calls with the oracle's packed flavour (tests/native/ksh_fake_device.cpp).  Checks the host layer's
    side of every device call on machines without a GPU; the product library is not involved."""
    import os
    import shutil
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = "kube-scheduler-rs-reference_b200"
    shadow = tmp_path / "shadow"
    (shadow / pkg).mkdir(parents=True)
    for f in os.listdir(os.path.join(root, pkg)):
        if f.endswith(".py"):
            shutil.copy(os.path.join(root, pkg, f), shadow / pkg / f)
    shutil.copy(os.path.join(root, "ksched_pkg.py"), shadow / "ksched_pkg.py")
    (shadow / "__graft_entry__.py").write_text("def build():\n    pass\n")
    for d in ("include", "oracle", "tests"):
        os.symlink(os.path.join(root, d), shadow / d)
    subprocess.run(["make", "-C", os.path.join(root, "oracle")], check=True, capture_output=True)
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-I" + os.path.join(root, "include"),
                        "-I" + os.path.join(root, "oracle"), os.path.join(root, pkg, "csrc", "host", "ksh_host.cpp"),
                        os.path.join(root, "tests", "native", "ksh_fake_device.cpp"), "-L" + os.path.join(root, "oracle"), "-loracle",
                        "-Wl,-rpath," + os.path.join(root, "oracle"), "-pthread", "-o", str(shadow / pkg / "libksched.so")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    env = {k: v for k, v in os.environ.items() if k != "PYTHONPATH"}
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        "tests/test_host_layer.py", "tests/test_host_calls.py", "tests/test_gpu_parity.py::test_reference_sampling_policy_faithful_objects",
                        "tests/test_gpu_parity.py::test_objects_faithful_oracle_vs_gpu", "tests/test_gpu_parity.py::test_gv1_objects_vs_faithful_oracle"],
                       cwd=str(shadow), capture_output=True, text=True, env=env, timeout=900)
    tail = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else r.stderr
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, r.stdout[-3000:] + r.stderr[-2000:]
