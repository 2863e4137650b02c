"""Gangs when binding (ks_gang_fit_bind) on the H100, bit for bit: node, total, five parts, five refusals, hard and soft
counts, free[], free_r and placed against tests/gang_fit_bind_oracle.py on small shapes and the hand-derived queues of
tests/golden/gv1_gang_fit_bind.json; M1 and M2 against ks_fit_bind on the bind_edges value families at N of 1, 129,
16,897 and 33,793 and label widths 1-8; M3 against ks_fit_bind on the committed pods of 65,536-pod queues cut into gangs
of 1 to 4,096 pods (rollbacks that cross slice edges, lower a hostname-spread minimum and clear first-pod flags); M4 with
ks_select on both paths; and ksh_reconcile_fit_gangs end to end."""
import json
import os

import numpy as np
import pytest

from affinity_bind_oracle import AFFINITY, ANTI
from bind_edges import FAMILY_N, bind_family, bind_slices, constraints, fit_arrays
from fit_bind_oracle import compile_resources, final_free
from gang_fit_bind_oracle import gang_fit_bind_packed, gangs_of, golden_inputs
from node_bind_oracle import compile_rules, random_cluster
from profile_bind_oracle import PREFERRED
from test_commit_paths_gpu import FAMILIES, _load
from test_fit_bind_gpu import EXTRA, GPU, resources
from test_replicas_gpu import _nodes, load
from test_spread_bind_gpu import key_set, mixed_queue

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = (1, 3, 4)
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "gv1_gang_fit_bind.json")))["cases"]


@pytest.fixture(scope="module")
def sms(ks):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def cut(rng, P, lo, hi):
    """Gang offsets: sizes drawn from [lo, hi], the last one clipped to the queue"""
    sizes = []
    while sum(sizes) < P:
        sizes.append(int(min(rng.integers(lo, hi + 1), P - sum(sizes))))
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)


def same(a, b, tag):
    """Two results of fit_bind / gang_fit_bind: node, score, parts, refused, counts, soft counts, free_r"""
    for i in (0, 1, 2, 3, 6):
        assert np.array_equal(a[i], b[i]), (tag, i, np.nonzero((a[i] != b[i]).reshape(len(a[i]), -1).any(1))[0][:8])
    for i in (4, 5):
        assert all(np.array_equal(x, y) for x, y in zip(a[i], b[i])), (tag, i)


def run_gang(ks, snap, nodes, queue, kw, offset, mm):
    _load(snap, *nodes)  # bound pods within the limits that leave exactly fc / fm, for every value family
    got = snap.gang_fit_bind(*queue, offset, mm, **kw)
    return got, snap.free()


def run_fit(ks, snap, nodes, queue, kw, pods=None):
    _load(snap, *nodes)
    rc, rm, sel, group, G, keys = queue
    kw = dict(kw)
    if pods is not None:
        pods = np.asarray(pods, np.int64)
        rc, rm, sel, group = rc[pods], rm[pods], np.ascontiguousarray(sel[pods]), group[pods]
        if kw.get("pod_req") is not None:
            kw["pod_req"] = np.ascontiguousarray(kw["pod_req"][pods])
    got = snap.fit_bind(rc, rm, sel, group, G, keys, **kw)
    return got, snap.free()


# ------------------------------------------------------------------------------------------- 1. against the restatement
# the last flag adds existing pods and soft_all_keys, so that the call stages every array it can take
CASES = [(1, 1, (1,), 3, 24, False), (2, 129, (3, "host"), 4, 60, False), (4, 2100, (3, "host"), 5, 60, True),
         (8, 16897, (3,), 4, 30, False)]


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("case", CASES, ids=[f"W{c[0]}-N{c[1]}" for c in CASES])
def test_against_the_oracle(ks, case, policy):
    W, N, modes, G, P, every_array = case
    rng = np.random.default_rng([W, N, policy, 0x6A6F])
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, modes)
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 3000), mem=(0, 12 << 30))
    nl, nt, gr = random_cluster(rng, N, G, 3)
    alloc, bound, pod_res = resources(rng, N, P, 3)
    names, free0, req = compile_resources(alloc, bound, pod_res, ["pods"] + [nm for nm in EXTRA if any(
        nm in r for r in pod_res)])
    terms = [(0, ANTI, len(keys) - 1, [0]), (1, AFFINITY, 0, [1]), (2, PREFERRED, 0, [1])]
    soft = np.array([0, 1, 3], np.uint32)[rng.integers(0, 3, (G, len(keys)))]
    offset = cut(rng, P, 1, 6)
    mm = np.minimum(np.diff(offset), rng.integers(0, 4, len(offset) - 1)).astype(np.uint32)
    rc = rc.copy()
    rc[int(offset[1]) - 1] = 1 << 36  # gang 0's last pod fits no node and gang 0 needs every pod: it rolls back
    mm[0] = int(offset[1])
    existing_pods = soft_all = None
    if every_array:
        existing_pods = (rng.integers(0, G, 40).astype(np.int32), rng.integers(0, N, 40).astype(np.int32))
        soft_all = rng.integers(0, 2, G).astype(np.uint8)
    rules = compile_rules(nl, nt, gr)
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got = snap.gang_fit_bind(rc, rm, sel, group, G, keys, offset, mm, terms, existing_pods, skew, mind, ex, policy,
                                 soft_skew=soft, soft_all_keys=soft_all, term_weight=[0, 0, 40], rules=rules,
                                 node_free=free0, pod_req=req)
        gfc, gfm = snap.free()
    ofc, ofm = fc.copy(), fm.copy()
    want = gang_fit_bind_packed(ofc, ofm, ac, am, lab, rc, rm, sel, group, G, keys, nl, nt, gr, alloc, bound, pod_res,
                                offset, mm, terms=terms, existing_pods=existing_pods, max_skew=skew, min_domains=mind,
                                existing=ex, policy=policy, soft_skew=soft, soft_all_keys=soft_all,
                                term_weight=[0, 0, 40])
    for i in range(4):
        assert np.array_equal(got[i], want[i]), i
    for i in (4, 5):
        assert all(np.array_equal(a, b) for a, b in zip(got[i], want[i])), i
    assert np.array_equal(got[6], final_free(alloc, want[6], names)) and np.array_equal(got[7], want[7])
    assert np.array_equal(gfc, ofc) and np.array_equal(gfm, ofm)
    if N > 100:
        assert (want[7] < mm).any() and (want[7] >= mm).any() and (got[0] >= 0).any()
    if every_array:  # both taint masks and a node-affinity expression as well
        assert rules["taint_hard"].any() and rules["taint_soft"].any() and any(t[2] for t in rules["node_terms"])


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_golden(ks, case):
    (fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, nl, nt, gr, alloc, bound, pod_res), kw = golden_inputs(case)
    names, free0, req = compile_resources(alloc, bound, pod_res)
    exp = case["expect"]
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        got = snap.gang_fit_bind(rc, rm, sel, group, G, keys, case["gangs"]["offset"], case["gangs"]["min_member"],
                                 kw.get("terms", ()), None, kw.get("max_skew"), None, kw.get("existing"),
                                 kw["policy"], rules=compile_rules(nl, nt, gr), node_free=free0, pod_req=req)
        gfc, _ = snap.free()
    assert got[0].tolist() == exp["node"] and got[7].tolist() == exp["placed"]
    assert got[3].tolist() == exp["refused"] and gfc.tolist() == exp["free_cpu"]
    assert got[6].tolist() == exp["free_r"] and [c.tolist() for c in got[4]] == exp["counts"]


# ---------------------------------------------------------------------------- 2. M1 and M2 on the bind_edges families
FAM_CASES = list(enumerate(FAMILIES))


@pytest.mark.parametrize("i,fam", FAM_CASES, ids=[f.replace(" ", "_") for f in FAMILIES])
def test_m1_m2_families(ks, sms, i, fam):
    """M1 (every min_member 0, random gangs) and M2 (singleton gangs, min_member 1) are ks_fit_bind bit for bit, with
    placed = the gang's bound pods; N cycles through 1, 129, 16,897 and 33,793, W through 1, 2, 4, 8."""
    N, W = FAMILY_N[i % 4], (1, 2, 4, 8)[(i // 4) % 4]
    policy = POLICIES[i % 3]
    P, G = (120 if N < 1000 else 24), 4
    rng = np.random.default_rng([i, N, W, 0x6A61])
    ac, am, lab, fc, fm, rc, rm, sel, group, keys = bind_family(fam, rng, N, P, W, sms, G)
    skew, mind, ex = constraints(rng, G, keys)
    nf, pr = fit_arrays(resources(rng, N, P, 2 + i % 7))
    kw = dict(terms=[(0, ANTI, 1, [0]), (1, AFFINITY, 0, [1]), (2, PREFERRED, 2, [0, 3])], max_skew=skew,
              min_domains=mind if i % 2 else None, existing=ex if i % 3 else None, policy=policy,
              soft_skew=np.array([0, 1, 3], np.uint32)[rng.integers(0, 3, (G, len(keys)))], term_weight=[0, 0, 60],
              hard_affinity_weight=3, rules=compile_rules(*random_cluster(rng, N, G, 3)), node_free=nf, pod_req=pr)
    nodes, queue = (ac, am, lab, fc, fm), (rc, rm, sel, group, G, keys)
    with ks.Snapshot(0) as snap:
        want, wfree = run_fit(ks, snap, nodes, queue, kw)
        for offset, m in ((cut(rng, P, 1, 9), 0), (np.arange(P + 1, dtype=np.uint64), 1)):
            mm = np.full(len(offset) - 1, m, np.uint32)
            got, gfree = run_gang(ks, snap, nodes, queue, kw, offset, mm)
            same(got, want, f"{fam} N={N} W={W} min {m}")
            assert all(np.array_equal(a, b) for a, b in zip(gfree, wfree))
            assert got[7].tolist() == [int((want[0][g] >= 0).sum()) for g in gangs_of(offset)]


# ------------------------------------------------------------------------------------------------ 3. M3 at full size
def big_queue(rng, N, W, P):
    """A 65,536-pod queue over N nodes: group 0 spreads over hostnames at maxSkew 1, group 1 carries required affinity to
    itself on zone (the first-pod rule), group 2 anti-affinity to itself on zone, group 3 preferred terms; a third of
    the pods ask for GPUs, which a tenth of the nodes have."""
    fc, fm, ac, am, lab = _nodes(rng, N, W)
    keys = key_set(rng, N, (9, "host"))
    G = 5
    rc, rm, sel, group, skew, mind, ex = mixed_queue(rng, N, W, keys, G, P, cpu=(0, 600), mem=(0, 2 << 30))
    skew = np.zeros((G, 2), np.uint32)
    skew[0, 1] = 1
    terms = [(1, AFFINITY, 0, [1]), (2, ANTI, 0, [2]), (3, PREFERRED, 0, [0])]
    nf = np.stack([rng.integers(0, 200, N), np.where(np.arange(N) % 10 == 0, 8, 0)]).astype(np.int64)
    pr = np.stack([np.ones(P), np.where(rng.random(P) < 0.33, rng.integers(1, 5, P), 0)], axis=1).astype(np.int64)
    kw = dict(terms=terms, max_skew=skew, policy=4, term_weight=[0, 0, 50], node_free=nf, pod_req=pr,
              soft_skew=np.array([0, 1, 3], np.uint32)[rng.integers(0, 3, (G, 2))])
    return (ac, am, lab, fc, fm), (rc, rm, sel, group, G, keys), kw


M3_CASES = ["min0", "min1", "size", "random"]


@pytest.mark.parametrize("kind", M3_CASES)
def test_m3_full_queue(ks, sms, kind):
    """M3: 65,536 pods in gangs of 1 to 4,096; the committed gangs' pods and the final state against ks_fit_bind over
    those pods alone.  The rollbacks cross slice edges, lower hostname-spread minima and clear first-pod flags."""
    P, N, W = 65536, 16897, 2
    rng = np.random.default_rng([0x6A63, M3_CASES.index(kind)])
    nodes, queue, kw = big_queue(rng, N, W, P)
    offset = cut(rng, P, 1, 4096) if kind != "min1" else cut(rng, P, 1, 64)
    size = np.diff(offset).astype(np.uint32)
    mm = {"min0": np.zeros_like(size), "min1": np.ones_like(size), "size": size,
          "random": np.minimum(size, rng.integers(0, 4097, len(size))).astype(np.uint32)}[kind]
    with ks.Snapshot(0) as snap:
        got, gfree = run_gang(ks, snap, nodes, queue, kw, offset, mm)
        gangs = gangs_of(offset)
        ok = got[7] >= mm
        C_ = [p for j, g in enumerate(gangs) if ok[j] for p in g]
        R_ = [p for j, g in enumerate(gangs) if not ok[j] for p in g]
        want, wfree = run_fit(ks, snap, nodes, queue, kw, C_)
    assert len(C_) > 0 and (kind in ("min0", "min1") or len(R_) > 0)
    for i in (0, 1, 2, 3):
        assert np.array_equal(got[i][C_], want[i]), i
    for i in (4, 5):
        assert all(np.array_equal(a, b) for a, b in zip(got[i], want[i])), i
    assert np.array_equal(got[6], want[6])
    assert all(np.array_equal(a, b) for a, b in zip(gfree, wfree))
    assert (got[0][R_] == -1).all() and not got[1][R_].any() and not got[2][R_].any()
    if kind == "size":  # rolled-back gangs of hundreds of bound pods, whose nodes span the grid's slices
        assert bind_slices(N, sms)[0] > 1 and (got[7][~ok] > 100).any()


# ----------------------------------------------------------------------------------------- 4. M4: everything rolls back
def test_m4_all_roll_back(ks):
    """Every gang one pod short (min_member = size + ... clipped to size, and an unplaceable last pod): free[], free_r,
    the counts and the soft counts are the inputs, and ks_select on both paths equals a fresh snapshot's."""
    rng = np.random.default_rng(0x6A64)
    N, W, P = 3000, 4, 2000
    nodes, queue, kw = big_queue(rng, N, W, P)
    rc = queue[0].copy()
    offset = cut(rng, P, 2, 300)
    rc[(offset[1:] - 1).astype(np.int64)] = 1 << 36  # the last pod of every gang fits no node
    queue = (rc,) + queue[1:]
    mm = np.diff(offset).astype(np.uint32)
    ac, am, lab, fc, fm = nodes
    sel_rc, sel_rm, sel = queue[0][:256] % 4000, queue[1][:256], np.ascontiguousarray(queue[2][:256])
    with ks.Snapshot(0) as snap, ks.Snapshot(0) as ref:
        got, gfree = run_gang(ks, snap, nodes, queue, kw, offset, mm)
        load(ks, ref, fc, fm, ac, am, lab)
        assert (got[0] == -1).all() and (got[7] > 0).any() and (got[7] < mm).all()
        assert np.array_equal(gfree[0], fc) and np.array_equal(gfree[1], fm)
        assert np.array_equal(got[6], kw["node_free"])
        assert all(not c.any() for c in got[4] + got[5])
        for flags in (ks.KS_SELECT_FORCE_DIRECT, ks.KS_SELECT_FORCE_BITPAR):
            a = snap.select(sel_rc, sel_rm, sel, policy=ks.KS_SCORE_LEAST_ALLOCATED, flags=flags)
            b = ref.select(sel_rc, sel_rm, sel, policy=ks.KS_SCORE_LEAST_ALLOCATED, flags=flags)
            assert np.array_equal(a.node_idx, b.node_idx) and np.array_equal(a.score, b.score), flags


def test_gang_errors_leave_free_unchanged(ks):
    rng = np.random.default_rng(0x6A65)
    nodes, (rc, rm, sel, group, G, keys), kw = big_queue(rng, 200, 1, 10)
    ac, am, lab, fc, fm = nodes
    bad = [([1, 10], [1], ks.capi.KS_ERR_INVALID), ([0, 4, 3, 10], [0, 0, 0], ks.capi.KS_ERR_INVALID),
           ([0, 9], [1], ks.capi.KS_ERR_INVALID), ([0, 0, 10], [0, 0], ks.capi.KS_ERR_RANGE),
           ([0, 4, 10], [5, 0], ks.capi.KS_ERR_RANGE)]
    with ks.Snapshot(0) as snap:
        load(ks, snap, fc, fm, ac, am, lab)
        for off, mm, code in bad:
            with pytest.raises(ks.KsError) as e:
                snap.gang_fit_bind(rc, rm, sel, group, G, keys, off, mm, **kw)
            assert e.value.code == code, (off, mm)
            gfc, gfm = snap.free()
            assert np.array_equal(gfc, fc) and np.array_equal(gfm, fm)


# ---------------------------------------------------------------------------------------- 5. ksh_reconcile_fit_gangs
def test_reconcile_fit_gangs(ks):
    """A training job of 1 launcher and 4 four-GPU workers (min_member 5) and a second gang of 3 such workers that finds
    too few GPUs left.  Gang 0 commits: Binding bodies, and a second call sees its GPUs.  Gang 1 rolls back: status 4, no
    body, its GPUs not recorded.  A running member counts toward min_member; a nameless one gets status 2 and does not.
    After pod_deleted of a committed worker its GPUs come back."""
    arena = ks.objects.ObjectArena()
    N = 5
    nodes = [{"name": f"n{i}", "labels": {"kubernetes.io/hostname": f"n{i}"},
              "allocatable": {"cpu": "32", "memory": "68719476736", "pods": "10", **({GPU: "8"} if i >= 3 else {})}}
             for i in range(N)]
    taint = {"key": "gpu", "value": "true", "effect": "NoSchedule"}
    rules = [{"tolerations": [{"key": "gpu", "operator": "Exists"}]}]
    worker = {"containers": [{"cpu": "1", "memory": "1073741824", GPU: "4"}]}
    pods = ([{"name": "launcher", "containers": [{"cpu": "1", "memory": "1073741824"}]}] +
            [{"name": f"w{i}", **worker} for i in range(4)] + [{"name": f"v{i}", **worker} for i in range(3)])
    group = np.zeros(len(pods), np.int32)
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(arena.nodes(nodes), N)
        ctx.set_node_taints({"n3": [taint], "n4": [taint]})
        names = [ctx.node_name(i) for i in range(N)]
        objs = arena.pods(pods)
        status, node, bodies, placed = ctx.reconcile_fit_gangs(objs, len(pods), group, 1, ["kubernetes.io/hostname"],
                                                                [0, 5, 8], [5, 3], group_rules=rules)
        assert placed.tolist() == [5, 0]
        assert (status[:5] == ks.host.KSH_RECONCILE_OK).all()
        assert sorted(names[n] for n in node[1:5]) == ["n3", "n3", "n4", "n4"]
        for i in range(5):
            assert json.loads(bodies[i])["target"]["name"] == names[node[i]]
        assert (status[5:] == ks.host.KSH_RECONCILE_GANG_UNSATISFIED).all() and (node[5:] == -1).all()
        assert all(b is None for b in bodies[5:])
        _, free_r, _ = ctx.compile_resources(arena.pods([{"name": "x", **worker}]), 1)
        assert free_r[1].tolist() == [0, 0, 0, 0, 0]  # gang 0's 16 GPUs are recorded, gang 1 charged none
        # a running member (bound to n0) counts toward min_member 2; a nameless member gets status 2 and does not count
        more = [{"name": "r0", "node_name": names[0], "containers": [{"cpu": "1"}]}, {"name": None, **worker},
                {"name": "c0", "containers": [{"cpu": "1", "memory": "1048576"}]}]
        status2, node2, bodies2, placed2 = ctx.reconcile_fit_gangs(arena.pods(more), 3, np.zeros(3, np.int32), 1,
                                                                   ["kubernetes.io/hostname"], [0, 3], [2],
                                                                   group_rules=rules)
        assert status2.tolist() == [ks.host.KSH_RECONCILE_OK, ks.host.KSH_RECONCILE_BINDING_OBJECT_FAILED,
                                    ks.host.KSH_RECONCILE_OK]
        assert node2[0] == -1 and node2[2] >= 0 and placed2.tolist() == [1]
        # the same gang with min_member 3: one running, one schedulable, the nameless one not counted: too few
        status3, _, _, placed3 = ctx.reconcile_fit_gangs(arena.pods(more[:2] + [{**more[2], "name": "c1"}]), 3,
                                                         np.zeros(3, np.int32), 1, ["kubernetes.io/hostname"], [0, 3],
                                                         [3], group_rules=rules)
        assert status3[2] == ks.host.KSH_RECONCILE_GANG_UNSATISFIED and placed3.tolist() == [0]
        # a committed worker deleted: its 4 GPUs are free again
        done = arena.pods([{"name": "w0", "node_name": names[node[1]], **worker}])
        ctx.pod_deleted(done)
        _, free_r, _ = ctx.compile_resources(arena.pods([{"name": "x", **worker}]), 1)
        assert free_r[1].tolist() == [4 if i == node[1] else 0 for i in range(N)]
