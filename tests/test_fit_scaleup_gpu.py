"""Scale-up estimate under the full filter (ks_fit_scaleup_estimate) on the GPU: every row, best pick, node ordinal,
refusal word and resource sum bit for bit against the restatement of tests/fit_scaleup_oracle.py, across label widths,
resource counts with non-contiguous request masks, 64 rule groups, template and pod counts up to the limits (a sampled
subset of templates restated), max_nodes 0, 1 and 1024 and ties; E1 against ks_scaleup_estimate, also on its edge
values; the refusal pass after a larger call; the snapshot untouched; the range errors; and the host call end to end."""
import ctypes as C

import numpy as np
import pytest

import fit_scaleup_oracle as fso
from helpers import load_golden

pytestmark = pytest.mark.gpu

LC, LM = 1 << 26, 1 << 45  # template limits: KS_MAX_CPU_MILLI >> 10, KS_MAX_MEM_BYTES >> 10
CASES = load_golden("gv1_fit_scaleup.json")["cases"]


def widen(a, W):
    return np.concatenate([a, np.zeros((a.shape[0], W - a.shape[1]), np.uint64)], axis=1) if W > a.shape[1] else a


def select_state(ks, s, rc, rm, sel):
    out = []
    for flags in (ks.capi.KS_SELECT_FORCE_DIRECT, ks.capi.KS_SELECT_FORCE_BITPAR):
        r = s.select(rc, rm, sel, flags=flags)
        out.append((r.node_idx, r.score, r.feasible_cnt))
    return out


@pytest.fixture(scope="module")
def snap(ks):
    """A snapshot with a cluster on it, whose free[] and ks_select every call must leave unchanged"""
    cl = ks.synth.make(300, 400, seed=0x5CF1, bound_per_node=2)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    with ks.Snapshot(0) as s:
        s.set_nodes(ac, am, lab)
        s.set_bound(bn, bc, bm)
        s._probe = (rc[:200], rm[:200], sel[:200])
        yield s


def run(ks, s, a, W=None, with_rules=True, with_res=True, R=None):
    """Snapshot.fit_scaleup_estimate of to_arrays' a, with free[] and ks_select checked unchanged around the call"""
    W = W or a["labels"].shape[1]
    before = s.free(), select_state(ks, s, *s._probe)
    res = dict(node_free=a["node_free"], pod_req=a["pod_req"]) if with_res else {}
    out = s.fit_scaleup_estimate(a["req_cpu"], a["req_mem"], widen(a["sel"], W), a["alloc_cpu"], a["alloc_mem"],
                                 a["free_cpu"], a["free_mem"], widen(a["labels"], W), a["max_nodes"],
                                 a["group"] if with_rules else np.full(len(a["req_cpu"]), -1, np.int32),
                                 a["n_groups"] if with_rules else 0, rules=a["rules"] if with_rules else None, **res)
    after = s.free(), select_state(ks, s, *s._probe)
    assert all(np.array_equal(x, y) for x, y in zip(before[0], after[0])), "free[] changed"
    for x, y in zip(before[1], after[1]):
        assert all(np.array_equal(p, q) for p, q in zip(x, y)), "ks_select changed"
    if not with_rules and not with_res:  # E1
        want = s.scaleup_estimate(a["req_cpu"], a["req_mem"], widen(a["sel"], W), a["alloc_cpu"], a["alloc_mem"],
                                  a["free_cpu"], a["free_mem"], widen(a["labels"], W), a["max_nodes"])
        assert np.array_equal(out[0], want[0]) and out[1] == want[1] and np.array_equal(out[2], want[2]), "E1"
        assert np.array_equal(out[3][:, 0], want[3][:, 2] + want[3][:, 3]) and not out[3][:, 1:].any(), "E1 words"
    return out


def same(got, want, which=None, pods=None):
    rows, best, node, refused, used = got
    wrows, wbest, wnode, wref, wused = want
    t = slice(None) if which is None else which
    for f in wrows.dtype.names:
        assert np.array_equal(rows[f][t], wrows[f][t]), f
    if which is None:
        assert best == wbest
    assert np.array_equal(node[t], wnode[t])
    p = slice(None) if pods is None else pods
    assert np.array_equal(refused[p], wref[p])
    if used is not None and used.shape[1] == wused.shape[1]:
        assert np.array_equal(used[t], wused[t])


def with_R(d, R):
    """d with its resources cut to the first R names (the pods' other requests dropped)"""
    names = d["names"][:R]
    pods = [dict(q, res={k: v for k, v in q["res"].items() if k in names}) for q in d["pods"]]
    return fso.problem(d["templates"], pods, d["group_rules"], names)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_cases(ks, snap, case):
    d = fso.golden_problem(case)
    got = run(ks, snap, fso.to_arrays(d))
    same(got, fso.fit_scaleup(d))
    assert got[1] == case["want"]["best"]


@pytest.mark.parametrize("W", [1, 2, 4, 8])
def test_label_widths(ks, snap, W):
    d = fso.random_problem(np.random.default_rng(100 + W), 40, 600, extra=2)
    same(run(ks, snap, fso.to_arrays(d), W=W), fso.fit_scaleup(d))


@pytest.mark.parametrize("R", range(0, 9))
def test_resource_counts_and_masks(ks, snap, R):
    """R 0-8: "pods", the GPUs and six further names, each pod requesting a random (non-contiguous) subset"""
    d = with_R(fso.random_problem(np.random.default_rng(200 + R), 48, 800, extra=6), max(R, 1))
    a = fso.to_arrays(d)
    if R == 0:  # an empty resource set: node_free [0, T], pod_req [P, 0]
        a["node_free"], a["pod_req"] = a["node_free"][:0], a["pod_req"][:, :0]
        got = run(ks, snap, a)
        same(got[:4] + (None,), fso.fit_scaleup(d, with_res=False))
        return
    assert len(d["names"]) == R
    masks = {sum(1 << r for r in range(R) if a["pod_req"][p, r]) for p in range(len(d["pods"]))}
    assert R < 3 or any(m & (m + 1) for m in masks)  # some mask with a gap
    same(run(ks, snap, a), fso.fit_scaleup(d))


def test_64_rule_groups(ks, snap):
    d = fso.random_problem(np.random.default_rng(300), 60, 2000, G=64, extra=3)
    same(run(ks, snap, fso.to_arrays(d)), fso.fit_scaleup(d))


@pytest.mark.parametrize("T,P", [(4096, 2048), (700, 65536)])
def test_sizes_with_sampled_templates(ks, snap, T, P):
    """The largest calls: every refusal word of a sample of pods and every row of a sample of templates restated (the
    templates are independent, and so are the pods' words)"""
    rng = np.random.default_rng(T + P)
    d = fso.random_problem(rng, T, P, G=8, extra=3, max_nodes=(0, 6))
    got = run(ks, snap, fso.to_arrays(d))
    tw = sorted(set(rng.choice(T, 6, replace=False).tolist()) | {0, T - 1})
    sub = fso.problem([d["templates"][t] for t in tw], d["pods"], d["group_rules"], d["names"])
    want = fso.fit_scaleup(sub)
    for f in want[0].dtype.names:
        assert np.array_equal(got[0][f][tw], want[0][f]), f
    assert np.array_equal(got[2][tw], want[2]) and np.array_equal(got[4][tw], want[4])
    pw = sorted(set(rng.choice(P, 40, replace=False).tolist()) | {0, P - 1})
    sub = fso.problem(d["templates"], [d["pods"][p] for p in pw], d["group_rules"], d["names"])
    assert np.array_equal(got[3][pw], fso.fit_scaleup(sub, which=[])[3])
    assert (T - got[3].sum(axis=1).astype(np.int64)).sum() == got[0]["eligible"].sum()  # E5, summed


def test_max_nodes_0_1_and_1024_ordinals_filled(ks, snap):
    """max_nodes 0 and 1, and a template whose pod limit makes each of 1100 small pods open a node: 1024 open, 76 left"""
    big = fso.template(64000, 256 << 30, alloc={"pods": 2}, ds=[(0, 0, {})], max_nodes=1024)
    tps = [fso.template(16000, 64 << 30, max_nodes=0), fso.template(16000, 64 << 30, max_nodes=1), big,
           fso.template(64000, 256 << 30, alloc={"pods": 110, "nvidia.com/gpu": 8}, max_nodes=1024)]
    pods = [fso.pod(10, 1 << 20) for _ in range(1100)] + [fso.pod(100, 1 << 20, res={"nvidia.com/gpu": 1})] * 20
    d = fso.problem(tps, pods)
    got = run(ks, snap, fso.to_arrays(d))
    same(got, fso.fit_scaleup(d))
    assert got[0]["nodes"].tolist()[:3] == [0, 1, 1024] and got[0]["placed"][2] == 1024


def test_ties_in_the_order_key(ks, snap):
    """Many pods share a key (the same requests, or requests with the same weighted sum): pod order decides"""
    tps = [fso.template(8000, 32 << 30, alloc={"pods": 7, "example.com/x": 5}, max_nodes=m) for m in (3, 1024)]
    tps.append(fso.template(4000, 8 << 30, alloc={"pods": 110, "example.com/x": 2}, max_nodes=1024))
    pods = []
    for i in range(300):
        k = i % 3
        pods.append(fso.pod(1000 if k else 500, (2 << 30) if k == 2 else (4 << 30) if k == 0 else 2 << 30,
                            res={"example.com/x": 1} if i % 4 == 0 else {}))
    d = fso.problem(tps, pods)
    same(run(ks, snap, fso.to_arrays(d)), fso.fit_scaleup(d))


def test_e1_on_ks_scaleup_estimates_edge_values(ks, snap):
    """Rules and resources NULL: ks_scaleup_estimate's outputs at its edges - zero requests, empty and negative
    capacity, allocatables and requests at the template limits, and a selector on the never-set bit"""
    rng = np.random.default_rng(12)
    P = 1500
    rc = rng.integers(0, LC + 1, P).astype(np.int64)
    rm = rng.integers(0, LM + 1, P).astype(np.int64)
    rc[:100], rm[:100] = LC, LM
    rc[100:400:3], rm[100:400:3] = 0, 0
    rc[400:600], rm[400:600] = rng.integers(0, 4000, 200), rng.integers(0, 8 << 30, 200)
    sel = np.zeros((P, 1), np.uint64)
    sel[::7, 0] = np.uint64(1) << np.uint64(63)  # the never-set bit
    sel[1::11, 0] |= np.uint64(1)
    ac = np.array([LC, LC, 1, LC, LC - 1, 4000, 4000, 4000], np.int64)
    am = np.array([LM, 1, LM, LM - 1, LM, 8 << 30, 8 << 30, 8 << 30], np.int64)
    fc = np.array([LC, 1, 1, LC - 5, LC - 1, 0, -1, -LC], np.int64)
    fm = np.array([LM, 1, LM, LM - 7, LM, 0, 8 << 30, -LM], np.int64)
    lab = np.array([[1], [0], [1], [0], [1], [0], [1], [0]], np.uint64)
    mx = np.array([1024, 1024, 1024, 3, 1024, 1024, 1, 0], np.uint32)
    a = dict(req_cpu=rc, req_mem=rm, sel=sel, alloc_cpu=ac, alloc_mem=am, free_cpu=fc, free_mem=fm, labels=lab,
             max_nodes=mx, group=np.zeros(P, np.int32), n_groups=1, rules=None, node_free=None, pod_req=None)
    got = run(ks, snap, a, with_rules=False, with_res=False)  # E1 checked in run()
    assert got[4].shape == (8, 0) and got[0]["nodes"][7] == 0 and got[0]["eligible"][6] == 0


def test_refusal_pass_after_a_larger_call_with_another_R(ks, snap):
    """Staging holds what a larger call with R = 8 left; a smaller call with R = 2 must read none of it"""
    big = fso.random_problem(np.random.default_rng(400), 300, 6000, G=16, extra=6)
    same(run(ks, snap, fso.to_arrays(big)), fso.fit_scaleup(big))
    small = with_R(fso.random_problem(np.random.default_rng(401), 30, 500, G=4, extra=1), 2)
    same(run(ks, snap, fso.to_arrays(small)), fso.fit_scaleup(small))


def test_node_free_range_and_argument_errors(ks, snap):
    d = fso.golden_problem(CASES[0])
    a = fso.to_arrays(d)
    E = ks.capi

    def code(**kw):
        b = dict(a, **kw)
        try:
            run(ks, snap, b)
        except ks.KsError as e:
            return e.code
        return E.KS_OK
    for v in (1 << 52, -(1 << 52)):
        nf = a["node_free"].copy()
        nf[1, 1] = v
        assert code(node_free=nf) == E.KS_OK
        nf[1, 1] = v + (1 if v > 0 else -1)
        assert code(node_free=nf) == E.KS_ERR_RANGE
    pr = a["pod_req"].copy()
    pr[0, 1] = -1
    assert code(pod_req=pr) == E.KS_ERR_RANGE
    assert code(group=np.array([1], np.int32)) == E.KS_ERR_INVALID  # outside [-1, 1)
    assert code(n_groups=1 << 20, group=np.array([0], np.int32), rules=None) == E.KS_ERR_RANGE
    bad = dict(a["rules"], taint_hard=np.array([0, 1 << 5], np.uint64))  # a taint bit at or above n_taints
    assert code(rules=bad) == E.KS_ERR_INVALID
    mx = a["max_nodes"].copy()
    mx[0] = 1025
    assert code(max_nodes=mx) == E.KS_ERR_RANGE  # ks_scaleup_estimate's checks come first
    nf = np.zeros((9, 2), np.int64)
    assert code(node_free=nf, pod_req=np.zeros((1, 9), np.int64)) == E.KS_ERR_RANGE  # R > 8
    # empty calls: nothing to pack
    rows, best, node, ref, used = snap.fit_scaleup_estimate(np.zeros(0, np.int64), np.zeros(0, np.int64),
                                                            np.zeros((0, 1), np.uint64), a["alloc_cpu"], a["alloc_mem"],
                                                            a["free_cpu"], a["free_mem"], a["labels"], a["max_nodes"],
                                                            np.zeros(0, np.int32), 1, rules=a["rules"],
                                                            node_free=a["node_free"], pod_req=np.zeros((0, 2), np.int64))
    assert best == -1 and len(rows) == 2 and not rows["nodes"].any() and not rows["placed"].any() and not used.any()


def host_problem(spec):
    """The restatement's problem of the object specs the host test and the INTEGRATION.md example pass"""
    def cpu(q):
        return int(q[:-1]) if q.endswith("m") else int(q) * 1000

    def ext(m):
        return {k: int(v) for k, v in m.items() if k not in ("cpu", "memory")}
    tps = []
    for t, taints in zip(spec["templates"], spec["taints"]):
        ds = [(sum(cpu(c["cpu"]) for c in o["containers"]), sum(int(c["memory"]) for c in o["containers"]),
               {k: sum(int(c.get(k, 0)) for c in o["containers"]) for k in ext(o["containers"][0])})
              for o in spec["overhead"] if o["node_name"] == t["name"]]
        tps.append(fso.template(cpu(t["allocatable"]["cpu"]), int(t["allocatable"]["memory"]), t.get("labels"), taints,
                                ext(t["allocatable"]), ds, spec["max_nodes"][len(tps)]))
    pods = [fso.pod(sum(cpu(c["cpu"]) for c in q["containers"]), sum(int(c["memory"]) for c in q["containers"]), g,
                    q.get("selector"), {k: sum(int(c.get(k, 0)) for c in q["containers"]) for k in ext(q["containers"][0])})
            for q, g in zip(spec["pods"], spec["group"])]
    return fso.problem(tps, pods, spec["rules"])


def test_host_call_end_to_end(ks):
    GPU, IT = "nvidia.com/gpu", "node.kubernetes.io/instance-type"
    rng = np.random.default_rng(500)
    templates, taints, overhead = [], [], []
    for t in range(12):
        gpu = t % 3 == 0
        alloc = {"cpu": str(int(rng.integers(8, 97))), "memory": str(int(rng.integers(16, 513)) << 30),
                 "pods": str(int(rng.integers(4, 111)))}
        if gpu:
            alloc[GPU] = "8"
        templates.append({"name": f"t{t}", "labels": {IT: "p4d" if gpu else ["m5", "c5", "r5"][t % 3],
                                                      "zone": "abc"[t % 3], "gen": str(t % 5)}, "allocatable": alloc})
        taints.append([{"key": GPU, "value": "present", "effect": "NoSchedule"}] if gpu else
                      [{"key": "spot", "value": "", "effect": "PreferNoSchedule"}] if t % 4 == 1 else [])
        for i in range(int(rng.integers(0, 3))):
            overhead.append({"name": f"ds-{t}-{i}", "ns": "kube-system", "node_name": f"t{t}",
                             "containers": [{"cpu": "100m", "memory": str(128 << 20)}]})
    pods, group = [], []
    for i in range(400):
        g = int(rng.integers(-1, 3))
        c = {"cpu": f"{int(rng.integers(1, 40)) * 100}m", "memory": str(int(rng.integers(1, 32)) << 28)}
        if g == 0 and rng.random() < 0.6:
            c[GPU] = str(int(rng.integers(1, 9)))
        pods.append({"name": f"p{i}", "ns": "w", "containers": [c],
                     **({"selector": {"zone": "a"}} if rng.random() < 0.1 else {})})
        group.append(g)
    rules = [{"tolerations": [{"key": GPU, "operator": "Exists", "effect": "NoSchedule"}]},
             {"required": [[{"key": IT, "operator": "In", "values": ["m5", "c5"]}]]},
             {"required": [[{"key": "gen", "operator": "Gt", "values": ["2"]}]]}]
    mx = rng.integers(1, 30, 12).astype(np.uint32)
    spec = dict(templates=templates, taints=taints, overhead=overhead, pods=pods, group=group, rules=rules, max_nodes=mx)
    arena = ks.objects.ObjectArena()
    with ks.host.Context(0) as ctx:
        got = ctx.scaleup_fit_estimate(arena.nodes(templates), 12, mx, arena.pods(pods), 400, np.array(group), 3,
                                       group_rules=rules, template_taints=taints, overhead_pods=arena.pods(overhead),
                                       n_overhead=len(overhead))
        assert ctx.n_nodes == 0
    same(got + (None,), fso.fit_scaleup(host_problem(spec)))


def test_integration_example(ks):
    """INTEGRATION.md's scale-up of a GPU training pod, as written there"""
    GPU = "nvidia.com/gpu"
    arena = ks.objects.ObjectArena()
    groups = [{"name": "cpu-pool", "labels": {"node.kubernetes.io/instance-type": "m5.16xlarge"},
               "allocatable": {"cpu": "64", "memory": str(256 << 30), "pods": "110"}},
              {"name": "gpu-pool", "labels": {"node.kubernetes.io/instance-type": "p4d.24xlarge"},
               "allocatable": {"cpu": "96", "memory": str(1152 << 30), "pods": "110", GPU: "8"}}]
    taints = [[], [{"key": GPU, "value": "present", "effect": "NoSchedule"}]]
    trainer = [{"name": "trainer-0", "ns": "ml", "containers": [{"cpu": "8", "memory": str(64 << 30), GPU: "8"}]}]
    rules = [{"tolerations": [{"key": GPU, "operator": "Exists", "effect": "NoSchedule"}]}]
    with ks.host.Context(0) as ctx:
        rows, best, node, refused = ctx.scaleup_fit_estimate(arena.nodes(groups), 2, [10, 4], arena.pods(trainer), 1,
                                                             [0], 1, group_rules=rules, template_taints=taints)
        assert best == 1 and rows["nodes"].tolist() == [0, 1] and rows["utilization"][1] == 6
        assert refused.tolist() == [[0, 1, 0, 0]]  # cpu-pool has no nvidia.com/gpu
        old_rows, old_best, _, _ = ctx.scaleup_estimate(arena.nodes(groups), 2, [10, 4], arena.pods(trainer), 1)
        assert old_best == 0 and old_rows["utilization"].tolist() == [18, 6]
