"""Topology spread for replica placement (ks_place_replicas_spread), CPU part: the restatement of tests/spread_oracle.py
against the existing replica plans where the skew rule cannot bind (one domain for all nodes, or a skew above every
count) under every policy; the hostname identity; the hand-derived GV-1 plans of tests/golden/gv1_spread.json; every
blocked_domain case; the C / ctypes / numpy / Rust mirrors of the row; ksh_context_topology_domains on a packing-only
context; and the errors caught without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from helpers import load_golden
from policy_oracle import PLAN
from replicas_oracle import merge_packed
from spread_oracle import SPREAD_PLAN_DTYPE, spread_packed
from test_replicas import random_cluster

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = (0, 1, 3, 4)


def replica_plan(policy, fc, fm, ac, am, labels, rc, rm, sel, R):
    if policy in (0, 1):
        return merge_packed(fc, fm, ac, am, labels, rc, rm, sel, R, policy)
    return PLAN[policy](fc, fm, ac, am, labels, rc, rm, sel, R)


def assert_same_plan(got, want, ctx):
    rows, node, score, off, _ = got
    w_rows, w_node, w_score, w_off = want
    for f in ("placed", "nodes", "max_per_node", "last_score"):
        assert np.array_equal(rows[f], w_rows[f]), (ctx, f)
    assert np.array_equal(node, w_node) and np.array_equal(score, w_score) and np.array_equal(off, w_off), ctx


@pytest.mark.parametrize("policy", POLICIES)
def test_unbinding_rule_gives_the_replica_plan(policy):
    """One domain for all nodes (any skew), or every node in some domain with max_skew >= R + max(existing): the rule
    never binds, so the plan is ks_place_replicas' plan."""
    rng = np.random.default_rng(0x5B7EAD + policy)
    for it in range(400):
        fc, fm, ac, am, labels, rc, rm, sel, R = random_cluster(rng)
        N, T = len(fc), len(rc)
        want = replica_plan(policy, fc, fm, ac, am, labels, rc, rm, sel, R)
        one = spread_packed(fc, fm, ac, am, labels, rc, rm, sel, R, np.zeros(N), 1,
                            rng.integers(1, 4, T), policy=policy)
        assert_same_plan(one, want, (it, "one domain"))
        D = int(rng.integers(1, N + 2))
        dom = rng.integers(0, D, N)
        ex = rng.integers(0, 5, (T, D))
        skew = R.astype(np.int64) + ex.max(axis=1)
        wide = spread_packed(fc, fm, ac, am, labels, rc, rm, sel, R, dom, D, np.maximum(skew, 1), existing=ex,
                             policy=policy)
        assert_same_plan(wide, want, (it, "wide skew"))
        for t in range(T):  # the counts are the existing pods plus the copies per domain
            a, b = int(wide[3][t]), int(wide[3][t + 1])
            placed = wide[1][a:b][wide[1][a:b] >= 0]
            assert np.array_equal(wide[4][t], ex[t] + np.bincount(dom[placed], minlength=D)), (it, t)


@pytest.mark.parametrize("policy", POLICIES)
def test_hostname_spreads_over_distinct_nodes_in_copy_zero_order(policy):
    """node_domain[n] = n, max_skew 1, no existing pods: one copy per node with room, in order of copy 0's score (ties
    to the lower node), then a second round only once every eligible node holds one."""
    rng = np.random.default_rng(0x4057 + policy)
    for it in range(300):
        fc, fm, ac, am, labels, rc, rm, sel, R = random_cluster(rng, r_max=10)
        N = len(fc)
        rows, node, score, off, cnt = spread_packed(fc, fm, ac, am, labels, rc, rm, sel, R, np.arange(N), N,
                                                    np.ones(len(rc), np.uint32), policy=policy)
        first = replica_plan(policy, fc, fm, ac, am, labels, rc, rm, sel, np.ones(len(rc), np.uint32))
        for t in range(len(rc)):
            a, b = int(off[t]), int(off[t + 1])
            placed = node[a:b][node[a:b] >= 0]
            k = min(len(placed), int(rows["eligible_domains"][t]))
            assert len(set(placed[:k].tolist())) == k, (it, t)  # distinct nodes while a round lasts
            if len(placed):  # copy 0 is ks_place_replicas' copy 0
                assert placed[0] == first[1][t] and score[a] == first[2][t], (it, t)
            assert (score[a:a + k][:-1] >= score[a + 1:a + k]).all(), (it, t)  # copy-0 scores, descending
            assert cnt[t].max(initial=0) <= rows["min_count"][t] + 1, (it, t)  # no node ahead of the minimum by 2


def test_gv1_spread_golden(ks):
    g = load_golden("gv1.json")
    want = load_golden("gv1_spread.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        ac, am, lab = ctx.export_packed()[:3]
        rc, rm, sel = ctx.pack_pods(arena.pods(g["pods"]), len(g["pods"]))
    names = [p["name"] for p in g["pods"]]
    for case in want["cases"]:
        i = names.index(case["spec"])
        rows, node, score, off, cnt = spread_packed(ac, am, ac, am, lab, rc[i:i + 1], rm[i:i + 1], sel[i:i + 1],
                                                    [case["replicas"]], want["node_domain"], want["n_domains"],
                                                    [case["max_skew"]], [case["min_domains"]], policy=0)
        assert node.tolist() == case["node"] and score.tolist() == case["score"], case["_why"]
        assert {f: int(rows[f][0]) for f in case["row"]} == case["row"], case["_why"]
        assert cnt[0].tolist() == case["counts"], case["_why"]


def _flat(N, cpu=4, mem=4):
    v = np.full(N, cpu, np.int64), np.full(N, mem, np.int64)
    return v[0], v[1], v[0], v[1], np.zeros((N, 1), np.uint64)


def test_blocked_domain_cases():
    """-1 when every copy is placed, when no domain is eligible (the selector excludes every node, or no node has a
    domain), and when minDomains holds m at 0 with every domain at max_skew; otherwise the lowest admitted full domain."""
    fc, fm, ac, am, lab = _flat(6)
    dom = np.array([0, 0, 1, 1, 2, 2])

    def plan(R, dom=dom, D=3, skew=1, mind=None, ex=None, sel=0, f=fc):
        return spread_packed(f, fm, ac, am, lab, [1], [1], np.array([[sel]], np.uint64), [R], dom, D, [skew],
                             mind, ex, 0)[0][0]

    r = plan(6)
    assert r["placed"] == 6 and r["blocked_domain"] == -1 and r["min_count"] == 2
    r = plan(3, sel=1)  # no node carries bit 0
    assert r["placed"] == 0 and r["eligible_domains"] == 0 and r["blocked_domain"] == -1
    r = plan(3, dom=np.full(6, -1))
    assert r["placed"] == 0 and r["eligible_domains"] == 0 and r["blocked_domain"] == -1
    r = plan(9, mind=[4])  # three eligible domains < 4: m stays 0, one copy per domain
    assert r["placed"] == 3 and r["min_count"] == 0 and r["blocked_domain"] == -1
    full = fc.copy()
    full[[2, 3]] = 0  # domain 1 eligible but without room: it holds m at 0
    r = plan(9, f=full)
    assert r["placed"] == 2 and r["min_count"] == 0 and r["blocked_domain"] == 1
    full[[0, 1]] = 0  # domains 0 and 1 full: the lower one is named
    r = plan(9, f=full)
    assert r["placed"] == 1 and r["blocked_domain"] == 0
    r = plan(9, mind=[4], f=np.where(dom == 1, 0, fc))  # minDomains with a full domain still admitted: it is named
    assert r["placed"] == 2 and r["blocked_domain"] == 1
    r = plan(9, ex=np.array([[5, 0, 0]]))  # existing above m + skew: domain 0 starts excluded, 1 and 2 fill to 5
    assert r["placed"] == 9 and r["blocked_domain"] == -1
    r = plan(0)
    assert r["placed"] == 0 and r["blocked_domain"] == -1 and r["eligible_domains"] == 3


def test_plan_struct_mirrors(ks):
    """ks_spread_plan: 32 bytes; the ctypes struct, the numpy record and the Rust shim list the header's fields, and
    ks_spread's fields match too."""
    assert C.sizeof(ks.capi.ks_spread_plan) == 32 and ks.capi.SPREAD_PLAN_DTYPE.itemsize == 32
    assert ks.capi.SPREAD_PLAN_DTYPE == SPREAD_PLAN_DTYPE
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    for struct in ("ks_spread_plan", "ks_spread"):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), hdr, re.S).group(1)
        c_fields = re.findall(r"\b\**([a-z_]+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
        assert c_fields == [f[0] for f in getattr(ks.capi, struct)._fields_], struct
        rbody = re.search(r"pub struct %s \{(.*?)\n\}" % struct, rs, re.S).group(1)
        assert re.findall(r"pub ([a-z_0-9]+):", rbody) == c_fields, struct
    assert list(SPREAD_PLAN_DTYPE.names) == [f[0] for f in ks.capi.ks_spread_plan._fields_]
    for name, value in (("KS_SPREAD_MAX_DOMAINS", 1 << 20), ("KS_SPREAD_MAX_EXISTING", 1 << 24),
                        ("KS_SPREAD_MAX_COUNTS", 1 << 26)):
        assert getattr(ks.capi, name) == value
        assert re.search(r"pub const %s: u(32|64) = ([^;]+);" % name, rs), name
    for fn in ("ks_place_replicas_spread", "ksh_place_replicas_spread", "ksh_context_topology_domains"):
        assert fn in ks.declared_symbols() and hasattr(ks.lib, fn), fn


def _node(name, labels):
    return {"name": name, "labels": labels, "allocatable": {"cpu": "4", "memory": "8589934592"}}


def test_topology_domains_on_a_packing_only_context(ks):
    """Dense ids by first appearance in node order, -1 without the key; upserts and removals renumber."""
    Z = "topology.kubernetes.io/zone"
    arena = ks.objects.ObjectArena()
    nodes = [_node("n0", {Z: "b"}), _node("n1", {Z: "a", "x": "1"}), _node("n2", None), _node("n3", {Z: "b"}),
             _node("n4", {"zone": "a"})]
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(nodes), len(nodes))
        dom, values = ctx.topology_domains(Z)
        assert dom.tolist() == [0, 1, -1, 0, -1] and values == ["b", "a"]
        dom, values = ctx.topology_domains("kubernetes.io/hostname")
        assert dom.tolist() == [-1] * 5 and values == []
        dom, values = ctx.topology_domains("x")
        assert dom.tolist() == [-1, 0, -1, -1, -1] and values == ["1"]
        ctx.remove_node("n0")  # later nodes move down one index, and "a" now appears first
        dom, values = ctx.topology_domains(Z)
        assert dom.tolist() == [0, -1, 1, -1] and values == ["a", "b"]
        ctx.upsert_node(arena.nodes([_node("n2", {Z: "c"})]))  # replaced in place
        ctx.upsert_node(arena.nodes([_node("n5", {Z: "a"})]))  # appended
        dom, values = ctx.topology_domains(Z)
        assert dom.tolist() == [0, 1, 2, -1, 0] and values == ["a", "c", "b"]
        n = ctx.n_nodes
        d = C.c_uint32()
        out = np.empty(n, np.int32)
        buf = C.create_string_buffer(4)
        off = np.empty(n, np.int64)
        assert ks.lib.ksh_context_topology_domains(ctx._h, Z.encode(), out.ctypes.data, C.byref(d), buf, 4,
                                                   off.ctypes.data) == 0
        assert d.value == 3 and off[:3].tolist() == [0, 2, -1]  # "a\0c\0" fills the 4 bytes
        assert buf.raw == b"a\0c\0"
        assert ks.lib.ksh_context_topology_domains(ctx._h, None, out.ctypes.data, C.byref(d), None, 0, None) == \
            ks.capi.KS_ERR_INVALID


def test_errors_without_a_device(ks):
    """A NULL snapshot is refused on the host; the object-level call on a packing-only context is KS_ERR_NO_DEVICE
    (the other argument and range errors need a snapshot and are checked on the GPU)."""
    out = (ks.capi.ks_spread_plan * 2)()
    rc_, rm_, sel = np.zeros(1, np.int64), np.zeros(1, np.int64), np.zeros(1, np.uint64)
    pods = ks.capi.ks_pods(1, rc_.ctypes.data, rm_.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
    rep, skew, dom = np.ones(1, np.uint32), np.ones(1, np.uint32), np.zeros(4, np.int32)
    sp = ks.capi.ks_spread(1, dom.ctypes.data, skew.ctypes.data, None, None)
    assert ks.lib.ks_place_replicas_spread(None, C.byref(pods), rep.ctypes.data, C.byref(sp), 0, out, None, None,
                                           None) == ks.capi.KS_ERR_INVALID
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        with pytest.raises(ks.KsError) as e:
            ctx.place_replicas_spread(arena.pods(g["pods"][:2]), 2, [3, 1], "zone", [1, 1])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
