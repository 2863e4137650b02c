"""Extended resources when binding (ks_fit_bind), without a device: hand-derived queues against the name-map restatement
in tests/fit_bind_oracle.py, identities L2-L5 on the restatements, the C / ctypes / Rust mirrors, and the errors caught
without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from fit_bind_oracle import compile_resources, final_free, fit_bind_packed, fits_request
from node_bind_oracle import node_bind_packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = (1, 3, 4)
GPU_TAINT = {"key": "gpu", "value": "true", "effect": "NoSchedule"}
GPU_TOL = {"tolerations": [{"key": "gpu", "operator": "Exists"}]}
GPU = "nvidia.com/gpu"
MANY = 1 << 40


def run(cpu, alloc, pod_res, group=None, group_rules=({},), taints=None, bound=(), policy=1, mem=64 << 30, rc=1000,
        **kw):
    """Nodes with free cpu `cpu` (allocatable = free), no labels; P pods of rc millicores and 1 GiB."""
    N, P = len(cpu), len(pod_res)
    fc = np.asarray(cpu, np.int64)
    fm = np.full(N, mem, np.int64)
    group = np.zeros(P, np.int32) if group is None else np.asarray(group, np.int32)
    keys = kw.pop("keys", [(np.zeros(N, np.int32), 1)])
    return fit_bind_packed(fc.copy(), fm.copy(), fc, fm, np.zeros((N, 1), np.uint64), np.full(P, rc, np.int64),
                           np.full(P, 1 << 30, np.int64), np.zeros((P, 1), np.uint64), group, len(group_rules), keys,
                           [{}] * N, taints or [[]] * N, list(group_rules), alloc, list(bound), pod_res, policy=policy,
                           **kw)


def test_fits_request():
    # pods 110 with 109 on the node: 109 + 1 > 110 is false, the pod fits; with 110 on it, 111 > 110: "pods"
    assert fits_request({}, {"pods": 110}, {}, 109) == []
    assert fits_request({}, {"pods": 110}, {}, 110) == ["pods"]
    # a zero request is skipped even on a node without the name; a missing allocatable counts as 0
    assert fits_request({GPU: 0}, {"pods": 1}, {}, 0) == []
    assert fits_request({GPU: 1}, {"pods": 1}, {}, 0) == [GPU]
    # 8 GPUs with 4 requested: 4 free, a 4-GPU pod fits, a 5-GPU pod does not
    assert fits_request({GPU: 4}, {"pods": 9, GPU: 8}, {GPU: 4}, 1) == []
    assert fits_request({GPU: 5}, {"pods": 9, GPU: 8}, {GPU: 4}, 1) == [GPU]


def test_gpu_pool_third_four_gpu_pod():
    # node 0: 64 cores, 8 GPUs, tainted gpu=true:NoSchedule; nodes 1-2: 8 cores, no GPU.  Three 4-GPU pods of a group
    # that tolerates the taint.  LEAST_BALANCED prefers node 0 throughout (after two pods it still has 62 of 64 cores
    # free against 8 of 8): without the resources all three land there.
    alloc = [{"pods": 110, GPU: 8}, {"pods": 110}, {"pods": 110}]
    pods = [{GPU: 4}] * 3
    cpu = [64000, 8000, 8000]
    taints = [[GPU_TAINT], [], []]
    free = run(cpu, [{"pods": 110}] * 3, [{}] * 3, group_rules=[GPU_TOL], taints=taints, policy=4)
    assert free[0].tolist() == [0, 0, 0]
    got = run(cpu, alloc, pods, group_rules=[GPU_TOL], taints=taints, policy=4)
    # pods 0 and 1 take 4 + 4 = 8 GPUs of node 0; pod 2: node 0 has 8 - 8 = 0 < 4, nodes 1-2 have 0 < 4: all three nodes
    # pass cpu, memory and selector and fail the GPU, so word 0 = 3 and words 1-4 = 0
    assert got[0].tolist() == [0, 0, -1]
    assert got[3][2].tolist() == [3, 0, 0, 0, 0]
    assert got[3][0].tolist() == [2, 0, 0, 0, 0]  # pod 0: nodes 1 and 2 have no GPU
    names, _, _ = compile_resources(alloc, [], pods)
    assert final_free(alloc, got[6], names).tolist() == [[108, 110, 110], [0, 0, 0]]  # pods 110 - 2, GPUs 8 - 8


def test_pod_limit_loses_to_a_fuller_node():
    # node 0: 32 cores free, pods 2 with 2 bound; node 1: 4 cores free, pods 110.  LEAST_ALLOCATED alone picks node 0
    # (more free); 2 + 1 > 2 refuses it ("Too many pods"), so the pod goes to node 1 and word 0 = 1.
    alloc = [{"pods": 2}, {"pods": 110}]
    bound = [(0, {}), (0, {})]
    assert run([32000, 4000], [{"pods": 110}] * 2, [{}])[0].tolist() == [0]
    got = run([32000, 4000], alloc, [{}], bound=bound)
    assert got[0].tolist() == [1] and got[3][0].tolist() == [1, 0, 0, 0, 0]


def test_negative_free_gpus_take_a_pod_without_gpus():
    # node 0: 2 GPUs, 4 requested by bound pods: free 2 - 4 = -2.  A pod requesting no GPU skips the test (zero
    # request) and binds; a pod requesting 1 GPU fails 1 <= -2.
    alloc = [{"pods": 110, GPU: 2}]
    bound = [(0, {GPU: 3}), (0, {GPU: 1})]
    got = run([8000], alloc, [{}, {GPU: 1}, {GPU: 0}], bound=bound)
    assert got[0].tolist() == [0, -1, 0] and got[3][1].tolist() == [1, 0, 0, 0, 0]
    names, free, req = compile_resources(alloc, bound, [{}, {GPU: 1}, {GPU: 0}])
    assert names == ["pods", GPU] and free.tolist() == [[108], [-2]] and req.tolist() == [[1, 0], [1, 1], [1, 0]]


def test_gpus_and_taint_count_in_word_zero_only():
    # node 0: no GPU and tainted; node 1: 1 GPU.  The pod (no toleration) requests a GPU: node 0 fails the resource
    # first and counts in word 0 only, never in the taint word; node 1 binds.
    got = run([8000, 8000], [{"pods": 110}, {"pods": 110, GPU: 1}], [{GPU: 1}], taints=[[GPU_TAINT], []])
    assert got[0].tolist() == [1] and got[3][0].tolist() == [1, 0, 0, 0, 0]
    # with no GPU anywhere: word 0 = 2, the taint word still 0
    got = run([8000, 8000], [{"pods": 110}] * 2, [{GPU: 1}], taints=[[GPU_TAINT], []])
    assert got[0].tolist() == [-1] and got[3][0].tolist() == [2, 0, 0, 0, 0]


def test_zone_short_of_gpus_pins_the_spread_minimum():
    # zones z0 (nodes 0, 1: 8 GPUs each) and z1 (nodes 2, 3: no GPU), maxSkew 1 on zone.  z1 is eligible (resources play
    # no part in eligibility, as upstream), its count stays 0, so the minimum stays 0.  Pod 0 binds in z0 (count 1);
    # pod 1: z0 nodes fail spread (1 + 1 - 0 = 2 > 1, word 3 = 2), z1 nodes fail the GPU (word 0 = 2): unbound.
    zone = np.array([0, 0, 1, 1], np.int32)
    alloc = [{"pods": 110, GPU: 8}] * 2 + [{"pods": 110}] * 2
    got = run([8000] * 4, alloc, [{GPU: 1}] * 2, keys=[(zone, 2)], max_skew=np.ones((1, 1), np.uint32))
    assert got[0].tolist() == [0, -1]
    assert got[3][1].tolist() == [2, 0, 0, 2, 0]
    assert got[4][0].tolist() == [[1, 0]]


def _case(rng, N=40, G=3, P=25):
    fc = rng.integers(2000, 9000, N).astype(np.int64)
    fm = rng.integers(4, 32, N).astype(np.int64) << 30
    ac, am = fc + rng.integers(0, 2000, N), fm + (rng.integers(0, 4, N) << 30)
    lab = rng.integers(0, 1 << 8, (N, 1)).astype(np.uint64)
    group = rng.integers(-1, G, P).astype(np.int32)
    rc, rm = rng.integers(1, 3000, P).astype(np.int64), rng.integers(0, 8, P).astype(np.int64) << 30
    gsel = rng.integers(0, 4, (G, 1)).astype(np.uint64)
    sel = np.where(group[:, None] >= 0, gsel[np.maximum(group, 0)], 0).astype(np.uint64)
    keys = [((np.arange(N) % 3).astype(np.int32), 3), (np.arange(N, dtype=np.int32), N)]
    skew = rng.integers(0, 3, (G, 2))
    taints = [[GPU_TAINT] if rng.random() < 0.2 else [] for _ in range(N)]
    rules = [GPU_TOL if rng.random() < 0.5 else {} for _ in range(G)]
    return fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, skew, taints, rules


def _both(rng, policy, alloc, pod_res):
    fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, skew, taints, rules = _case(rng)
    N = len(fc)
    alloc = alloc(N, rc)
    pod_res = pod_res(len(rc), rc)
    soft = rng.integers(0, 3, (G, 2))
    a = node_bind_packed(fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, group, G, keys, [{}] * N, taints, rules,
                         max_skew=skew, policy=policy, soft_skew=soft)
    ofc, ofm = fc.copy(), fm.copy()
    b = fit_bind_packed(ofc, ofm, ac, am, lab, rc, rm, sel, group, G, keys, [{}] * N, taints, rules, alloc, [],
                        pod_res, max_skew=skew, policy=policy, soft_skew=soft)
    return a, b, fc, alloc


def _same(a, b, it):
    assert all(np.array_equal(a[i], b[i]) for i in range(3)), it
    assert np.array_equal(b[3][:, 1:], a[3]) and not b[3][:, 0].any(), it
    assert all(np.array_equal(x, y) for x, y in zip(a[4] + a[5], b[4] + b[5])), it


@pytest.mark.parametrize("policy", POLICIES)
def test_l2_zero_requests(policy):
    """L2: every request 0 (and room for every pod) is ks_node_bind's walk; free_r ends where it started, negative
    entries included."""
    rng = np.random.default_rng(0xF170 + policy)
    for it in range(20):
        a, b, _, alloc = _both(rng, policy, lambda N, rc: [{"pods": MANY, GPU: -int(rng.integers(0, 3))}
                                                            for _ in range(N)],
                               lambda P, rc: [{GPU: 0} for _ in range(P)])
        _same(a, b, it)
        assert final_free(alloc, b[6], [GPU]).tolist() == [[r[GPU] for r in alloc]], it


@pytest.mark.parametrize("policy", POLICIES)
def test_l3_conservation(policy):
    """L3: free_r at the end = free_r at the start - the requests of the pods bound on each node."""
    rng = np.random.default_rng(0xF171 + policy)
    bound_any = 0
    for it in range(20):
        fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, skew, taints, rules = _case(rng)
        N, P = len(fc), len(rc)
        alloc = [{"pods": int(rng.integers(0, 4)), GPU: int(rng.integers(-2, 9))} for _ in range(N)]
        bound = [(int(rng.integers(0, N)), {GPU: int(rng.integers(0, 3))}) for _ in range(30)]
        pods = [{GPU: int(q)} for q in rng.integers(0, 3, P)]
        names, free0, req = compile_resources(alloc, bound, pods)
        got = fit_bind_packed(fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, group, G, keys, [{}] * N, taints, rules,
                              alloc, bound, pods, max_skew=skew, policy=policy)
        want = free0.copy()
        for p, n in enumerate(got[0]):
            if n >= 0:
                want[:, n] -= req[p]
        assert np.array_equal(final_free(alloc, got[6], names), want), it
        bound_any += (got[0] >= 0).sum()
    assert bound_any > 0


@pytest.mark.parametrize("policy", POLICIES)
def test_l4_ample_resources(policy):
    """L4: every node_free at least the queue's total request: the walk is ks_node_bind's."""
    rng = np.random.default_rng(0xF172 + policy)
    for it in range(20):
        a, b, _, _ = _both(rng, policy, lambda N, rc: [{"pods": 25, GPU: 75, "example.com/fpga": 50} for _ in range(N)],
                           lambda P, rc: [{GPU: int(rng.integers(0, 4)), "example.com/fpga": 2} for _ in range(P)])
        _same(a, b, it)


@pytest.mark.parametrize("policy", POLICIES)
def test_l5_a_copy_of_cpu(policy):
    """L5: a resource whose request is each pod's cpu request and whose free amount is free_cpu changes nothing."""
    rng = np.random.default_rng(0xF173 + policy)
    for it in range(20):
        fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, skew, taints, rules = _case(rng)
        N = len(fc)
        a = node_bind_packed(fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, group, G, keys, [{}] * N, taints, rules,
                             max_skew=skew, policy=policy)
        alloc = [{"pods": MANY, "cpu-copy": int(fc[n])} for n in range(N)]
        b = fit_bind_packed(fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, group, G, keys, [{}] * N, taints, rules,
                            alloc, [], [{"cpu-copy": int(c)} for c in rc], max_skew=skew, policy=policy)
        _same(a, b, it)


def test_struct_and_constant_mirrors(ks):
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    assert re.search(r"#define KS_BIND_MAX_RESOURCES 8u\b", hdr) and ks.capi.KS_BIND_MAX_RESOURCES == 8
    body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct ks_bind_resources \{(.*?)\} ks_bind_resources;", hdr,
                                               re.S).group(1))
    assert [f[0] for f in ks.capi.ks_bind_resources._fields_] == re.findall(r"(\w+);", body)
    assert C.sizeof(ks.capi.ks_bind_resources) == 24 and ks.capi.ks_bind_resources.pod_req.offset == 16
    assert "ks_fit_bind" in ks.declared_symbols() and hasattr(ks.lib, "ks_fit_bind")
    assert len(ks.lib.ks_fit_bind.argtypes) == 17
    hh = open(os.path.join(ROOT, "include", "ksched_host.h")).read()
    assert re.search(r"#define KSH_RECONCILE_INSUFFICIENT_RESOURCES 8\b", hh)
    assert ks.host.KSH_RECONCILE_INSUFFICIENT_RESOURCES == 8
    for name in ("ksh_compile_resources", "ksh_reconcile_fit"):
        assert name in ks.declared_symbols() and hasattr(ks.lib, name), name


def test_rust_shim_mirror():
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct ks_bind_resources \{(.*?)\} ks_bind_resources;", hdr,
                                               re.S).group(1))
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    rs_body = re.search(r"pub struct ks_bind_resources \{(.*?)\}", rs, re.S).group(1)
    assert re.findall(r"pub (\w+):", rs_body) == re.findall(r"(\w+);", body)
    for fn in ("ks_fit_bind", "ksh_compile_resources", "ksh_reconcile_fit"):
        assert re.search(r"pub fn %s\(" % fn, rs), fn
    assert re.search(r"pub const KSH_RECONCILE_INSUFFICIENT_RESOURCES: c_int = 8;", rs)
    assert re.search(r"pub const KS_BIND_MAX_RESOURCES: u32 = 8;", rs)


def test_errors_without_a_device(ks):
    """A NULL scoring is refused before anything else; a NULL snapshot with a valid scoring is KS_ERR_INVALID whatever
    the resources (the other checks need a snapshot and run in tests/test_fit_bind_gpu.py)."""
    rc_, sel = np.zeros(1, np.int64), np.zeros(1, np.uint64)
    pods = ks.capi.ks_pods(1, rc_.ctypes.data, rc_.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
    grp, dom = np.zeros(1, np.int32), np.zeros(4, np.int32)
    idx = np.empty(1, np.int32)
    sp = ks.capi.ks_spread_multi(1, (C.c_uint32 * 4)(1), (C.c_void_p * 4)(dom.ctypes.data), None, None, None)
    aff = ks.capi.ks_pod_affinity()
    sc = ks.capi.ks_bind_scoring(None, None, None, 1, 2, 2)
    res = ks.capi.ks_bind_resources(9, None, None)
    assert ks.lib.ks_fit_bind(None, C.byref(pods), grp.ctypes.data, 1, C.byref(sp), C.byref(aff), None, None,
                              C.byref(res), 4, idx.ctypes.data, None, None, None, None, None, None) == ks.capi.KS_ERR_INVALID
    assert "NULL scoring" in ks.lib.ks_last_error().decode()
    for r in (None, C.byref(res)):
        assert ks.lib.ks_fit_bind(None, C.byref(pods), grp.ctypes.data, 1, C.byref(sp), C.byref(aff), C.byref(sc),
                                  None, r, 4, idx.ctypes.data, None, None, None, None, None, None) == ks.capi.KS_ERR_INVALID
        assert "NULL scoring" not in ks.lib.ks_last_error().decode()


def test_fit_bind_shapes_are_checked_before_the_call(ks):
    """Snapshot.fit_bind refuses a node_free that is not [R, N] (a 1-D array would otherwise mean R = 0: no resource
    checked) and a pod_req that is not [P, R] (the C call would read past it), with ValueError before any device call.
    The handle is NULL here (no device), so a well-shaped call reaches ks_fit_bind and gets KS_ERR_INVALID."""
    snap = ks.Snapshot.__new__(ks.Snapshot)
    snap._h = None  # N = 0, W = 0
    P = 3
    rc, sel = np.zeros(P, np.int64), np.zeros((P, 0), np.uint64)
    keys = [(np.zeros(0, np.int32), 1)]
    grp = np.zeros(P, np.int32)
    bad = [
        (np.zeros(0, np.int64), np.ones((P, 1), np.int64)),  # 1-D node_free
        (np.zeros((1, 5), np.int64), np.ones((P, 1), np.int64)),  # N = 5 columns, the snapshot has 0 nodes
        (np.zeros((2, 0), np.int64), np.ones((P, 1), np.int64)),  # pod_req one resource short
        (np.zeros((1, 0), np.int64), np.ones((P - 1, 1), np.int64)),  # pod_req one pod short
        (np.zeros((1, 0), np.int64), np.ones(P, np.int64)),  # 1-D pod_req
    ]
    for nf, pr in bad:
        with pytest.raises(ValueError):
            snap.fit_bind(rc, rc, sel, grp, 1, keys, node_free=nf, pod_req=pr)
    with pytest.raises(ValueError):
        snap.fit_bind(rc, rc, sel, grp, 1, keys, node_free=np.zeros((1, 0), np.int64))  # pod_req missing
    with pytest.raises(ks.KsError) as e:
        snap.fit_bind(rc, rc, sel, grp, 1, keys, node_free=np.zeros((1, 0), np.int64), pod_req=np.ones((P, 1), np.int64))
    assert e.value.code == ks.capi.KS_ERR_INVALID
