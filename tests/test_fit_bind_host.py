"""Extended resources over objects, without a device (ksh_compile_resources, ksh_reconcile_fit): what the context tracks
per node and per bound pod, after sequences of set_nodes / upsert_node / remove_node / set_cluster_pods / pod_bound /
pod_deleted, against the string restatement in tests/fit_bind_oracle.py; malformed extended quantities leaving every
existing call's return code unchanged and reported only when a batch requests the resource; the batch limits; and
KS_ERR_NO_DEVICE on a packing-only context."""
import numpy as np
import pytest

from fit_bind_oracle import compile_resources

GPU, FPGA, EPH = "nvidia.com/gpu", "example.com/fpga", "ephemeral-storage"
NAMES = (GPU, FPGA, EPH, "hugepages-2Mi")


class Store:
    """The restatement's view of the cluster: nodes by name (allocatable maps of strings) and bound pods by key."""

    def __init__(self):
        self.nodes = {}
        self.pods = {}

    def node_obj(self, name):
        return {"name": name, "allocatable": self.nodes[name]}

    def maps(self, ctx):
        """alloc [N] and bound [(node index, requests)] in the context's node order."""
        order = [ctx.node_name(i) for i in range(ctx.n_nodes)]
        assert sorted(order) == sorted(self.nodes)
        idx = {nm: i for i, nm in enumerate(order)}
        alloc = [{k: int(v) for k, v in self.nodes[nm].items() if k not in ("cpu", "memory")} for nm in order]
        bound = [(idx[p["node_name"]], reqs(p)) for p in self.pods.values() if p["node_name"] in idx]
        return alloc, bound


def reqs(pod):
    out = {}
    for c in pod["containers"]:
        for k, v in (c or {}).items():
            if k not in ("cpu", "memory"):
                out[k] = out.get(k, 0) + int(v)
    return out


def rand_alloc(rng):
    a = {"cpu": "16", "memory": "68719476736"}
    if rng.random() < 0.9:
        a["pods"] = str(int(rng.integers(0, 12)))
    for nm in NAMES:
        if rng.random() < 0.4:
            a[nm] = str(int(rng.integers(0, 9)))
    return a


def rand_pod(rng, name, node=None):
    conts = []
    for _ in range(int(rng.integers(1, 3))):
        c = {"cpu": "100m", "memory": "1048576"}
        for nm in NAMES:
            if rng.random() < 0.3:
                c[nm] = str(int(rng.integers(0, 3)))
        conts.append(c if rng.random() < 0.9 else None)
    p = {"name": name, "ns": "w", "containers": conts}
    if node is not None:
        p["node_name"] = node
    return p


def compare(ks, ctx, arena, store, pending):
    alloc, bound = store.maps(ctx)
    names, free, req = ctx.compile_resources(arena.pods(pending), len(pending))
    wn, wf, wr = compile_resources(alloc, bound, [reqs(p) for p in pending])
    assert names == wn
    assert np.array_equal(free, wf) and np.array_equal(req, wr)
    return names


def test_tracking_against_the_strings(ks):
    rng = np.random.default_rng(0xF1F0)
    arena = ks.objects.ObjectArena()
    for it in range(5):
        store = Store()
        with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
            for i in range(30):
                store.nodes[f"n{i}"] = rand_alloc(rng)
            ctx.set_nodes(arena.nodes([store.node_obj(nm) for nm in store.nodes]), len(store.nodes))
            pods = [rand_pod(rng, f"b{i}", f"n{int(rng.integers(0, 32))}") for i in range(60)]  # n30, n31: unknown
            ctx.set_cluster_pods(arena.pods(pods), len(pods))
            store.pods = {p["name"]: p for p in pods if p["node_name"] in store.nodes}  # unknown nodes: not kept
            for step in range(60):
                pending = [rand_pod(rng, f"q{j}") for j in range(int(rng.integers(0, 6)))]
                compare(ks, ctx, arena, store, pending)
                u = rng.random()
                if u < 0.25:
                    nm = f"n{int(rng.integers(0, 34))}"
                    store.nodes[nm] = rand_alloc(rng)
                    ctx.upsert_node(arena.nodes([store.node_obj(nm)]))
                elif u < 0.35 and store.nodes:
                    nm = sorted(store.nodes)[int(rng.integers(0, len(store.nodes)))]
                    ctx.remove_node(nm)
                    del store.nodes[nm]
                    store.pods = {k: p for k, p in store.pods.items() if p["node_name"] != nm}
                elif u < 0.7 and store.nodes:
                    nm = sorted(store.nodes)[int(rng.integers(0, len(store.nodes)))]
                    p = rand_pod(rng, f"b{int(rng.integers(0, 90))}", nm)  # an existing key replaces its row
                    ctx.pod_bound(arena.pods([p]))
                    store.pods[p["name"]] = p
                elif store.pods:
                    k = sorted(store.pods)[int(rng.integers(0, len(store.pods)))]
                    ctx.pod_deleted(arena.pods([store.pods.pop(k)]))
            if it == 0:  # set_nodes drops every bound row, as for cpu and memory
                ctx.set_nodes(arena.nodes([store.node_obj(nm) for nm in store.nodes]), len(store.nodes))
                store.pods = {}
                compare(ks, ctx, arena, store, [rand_pod(rng, "q")])


def test_names_order_and_missing_allocatable(ks):
    """"pods" first, then names in order of first non-zero request; a node without "pods" takes no pod (free 0 - 0)."""
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes([{"name": "a", "allocatable": {"cpu": "4", "memory": "1024", GPU: "8"}},
                                   {"name": "b", "allocatable": {"cpu": "4", "memory": "1024", "pods": "110",
                                                                  FPGA: "2k"}}]), 2)
        pending = [{"name": "p0", "containers": [{"cpu": "1", GPU: "0"}, {FPGA: "3"}]},
                   {"name": "p1", "containers": [{GPU: "2", FPGA: "1"}]}]
        names, free, req = ctx.compile_resources(arena.pods(pending), 2)
    assert names == ["pods", FPGA, GPU]  # GPU's first request (p0) is 0: FPGA comes first
    assert free.tolist() == [[0, 110], [0, 2000], [8, 0]]
    assert req.tolist() == [[1, 3, 0], [1, 1, 2]]


def test_malformed_quantities_are_recorded_not_rejected(ks):
    """Every existing call returns what it returned before an extended quantity went bad; ksh_compile_resources reports
    KS_ERR_PARSE naming the node or pod only for a batch that requests the resource."""
    arena = ks.objects.ObjectArena()
    ok_node = {"name": "good", "allocatable": {"cpu": "4", "memory": "1024", "pods": "10"}}
    bad_node = {"name": "bad", "allocatable": {"cpu": "4", "memory": "1024", "pods": "10", GPU: "eight"}}
    bad_pod = {"name": "bp", "ns": "w", "node_name": "good", "containers": [{"cpu": "1", FPGA: "1.5.2"}]}
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes([ok_node, bad_node]), 2)
        ctx.upsert_node(arena.nodes([bad_node]))
        ctx.set_cluster_pods(arena.pods([bad_pod]), 1)
        ctx.pod_bound(arena.pods([bad_pod]))
        assert ctx.num_bound == 1
        rc, rm, sel = ctx.pack_pods(arena.pods([bad_pod]), 1)
        assert rc.tolist() == [1000]
        names, free, _ = ctx.compile_resources(arena.pods([{"name": "q", "containers": [{"cpu": "1"}]}]), 1)
        assert names == ["pods"] and sorted(free[0].tolist()) == [9, 10]  # "good" carries the bad pod
        for pending, who in (([{"name": "q", "containers": [{GPU: "1"}]}], "bad"),
                             ([{"name": "q", "containers": [{FPGA: "1"}]}], "w/bp"),
                             ([{"name": "q", "ns": "w", "containers": [{EPH: "1Qi"}]}], "w/q")):
            with pytest.raises(ks.KsError) as e:
                ctx.compile_resources(arena.pods(pending), 1)
            assert e.value.code == ks.capi.KS_ERR_PARSE and who in str(e.value), (pending, str(e.value))
        # two containers whose requests sum past int64: KS_ERR_RANGE, named as a sum, not as a parse error
        big = [{"name": "o", "ns": "w", "containers": [{GPU: "9223372036854775807"}, {GPU: "1"}]}]
        with pytest.raises(ks.KsError) as e:
            ctx.compile_resources(arena.pods(big), 1)
        assert e.value.code == ks.capi.KS_ERR_RANGE and "sum past int64" in str(e.value) and "w/o" in str(e.value)
        ctx.pod_deleted(arena.pods([bad_pod]))
        ctx.remove_node("bad")
        names, _, _ = ctx.compile_resources(arena.pods([{"name": "q", "containers": [{FPGA: "1", GPU: "1"}]}]), 1)
        assert names == ["pods", FPGA, GPU]


def test_batch_limits(ks):
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes([{"name": "a", "allocatable": {"cpu": "4", "memory": "1024"}}]), 1)
        seven = [{"name": f"q{i}", "containers": [{f"example.com/r{i}": "1"}]} for i in range(7)]
        names, _, req = ctx.compile_resources(arena.pods(seven), 7)
        assert len(names) == 8 and req.shape == (7, 8)
        eight = seven + [{"name": "q7", "containers": [{"example.com/r7": "1"}]}]
        with pytest.raises(ks.KsError) as e:  # "pods" and 8 names: split the batch
            ctx.compile_resources(arena.pods(eight), 8)
        assert e.value.code == ks.capi.KS_ERR_RANGE and "split the batch" in str(e.value)
        with pytest.raises(ks.KsError) as e:
            ctx.compile_resources(arena.pods([{"name": "q", "containers": [{GPU: "-1"}]}]), 1)
        assert e.value.code == ks.capi.KS_ERR_RANGE


def test_reconcile_fit_needs_a_device(ks):
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes([{"name": "a", "allocatable": {"cpu": "4", "memory": "1024", "pods": "4"}}]), 1)
        with pytest.raises(ks.KsError) as e:
            ctx.reconcile_fit(arena.pods([{"name": "q", "containers": [{"cpu": "1"}]}]), 1, [0], 1,
                              ["kubernetes.io/hostname"])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
