"""Topology spread when binding (ks_spread_bind), CPU part: the restatement of tests/spread_bind_oracle.py against the
hand-derived GV-1 queues of tests/golden/gv1_spread_bind.json; both identities of include/ksched.h (unconstrained pods
are ks_gang_bind with singleton groups, one fully constrained group is ks_place_replicas_spread_multi's copy list)
between the restatements; the skew rule at each placed pod's turn; the refusal counts; the C / ctypes / Rust mirrors;
and the errors caught without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from gang_oracle import gang_bind_packed
from helpers import load_golden
from policy_oracle import Oracle
from spread_bind_oracle import skew_ok_at_each_turn, spread_bind_packed
from spread_multi_oracle import spread_multi_packed
from spread_oracle import spread_packed
from test_replicas import random_cluster

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = (0, 1, 3, 4)


def _random_keys(rng, N, K):
    keys = []
    for _ in range(K):
        D = int(rng.integers(1, N + 2))
        dom = rng.integers(0, D, N)
        dom[rng.random(N) < 0.1] = -1
        keys.append((dom, D))
    return keys


def _queue(rng, rc, rm, sel, G, P):
    """P pods drawn from the specs rc / rm / sel; pod p of group g >= 0 is spec g % T (one selector per group), -1 = a
    random spec."""
    T = len(rc)
    group = rng.integers(-1, G, P) if G else np.full(P, -1)
    spec = np.where(group >= 0, group % T, rng.integers(0, T, P))
    return rc[spec], rm[spec], sel[spec], group


@pytest.mark.parametrize("policy", POLICIES)
def test_unconstrained_is_gang_bind_with_singletons(orc, policy):
    """Identity 1: every pod in group -1, or every max_skew 0: the nodes, scores and final free[] of ks_gang_bind with one
    singleton group per pod and min_member 0; nothing is refused."""
    rng = np.random.default_rng(0x5B1 + policy)
    for it in range(120):
        fc, fm, ac, am, labels, rc, rm, sel, _ = random_cluster(rng)
        N = len(fc)
        K = int(rng.integers(1, 4))
        keys = _random_keys(rng, N, K)
        G = int(rng.integers(0, 4))
        P = int(rng.integers(1, 20))
        qc, qm, qs, group = _queue(rng, rc, rm, sel, G, P)
        if it % 2:
            group[:] = -1
        gfc, gfm = fc.copy(), fm.copy()
        want = gang_bind_packed(Oracle(orc), gfc, gfm, ac, am, labels, qc, qm, qs, np.arange(P + 1, dtype=np.uint64),
                                np.zeros(P, np.uint32), policy)
        bfc, bfm = fc.copy(), fm.copy()
        node, score, refused, counts = spread_bind_packed(bfc, bfm, ac, am, labels, qc, qm, qs, group, keys,
                                                          np.zeros((G, K)), policy=policy)
        assert np.array_equal(node, want[0]) and np.array_equal(score, want[1]), it
        assert np.array_equal(bfc, gfc) and np.array_equal(bfm, gfm), it
        assert not refused.any() and all(not c.any() for c in counts), it


@pytest.mark.parametrize("policy", POLICIES)
def test_one_group_is_the_replica_plan(policy):
    """Identity 2: one group of R identical pods that constrains every key binds ks_place_replicas_spread_multi's copy
    list with its counts, and leaves free[] as committing that list would; K = 1 against ks_place_replicas_spread."""
    rng = np.random.default_rng(0x5B2 + policy)
    for it in range(150):
        fc, fm, ac, am, labels, rc, rm, sel, R = random_cluster(rng, t_max=1, r_max=20)
        N, R = len(fc), int(R[0])
        K = 1 if it % 3 == 0 else int(rng.integers(1, 4))
        keys = _random_keys(rng, N, K)
        skew = rng.integers(1, 4, (1, K))
        mind = rng.integers(0, 4, (1, K))
        ex = [rng.integers(0, 4, (1, d)) for _, d in keys]
        want = spread_multi_packed(fc, fm, ac, am, labels, rc, rm, sel, [R], keys, skew, mind, ex, policy)
        bfc, bfm = fc.copy(), fm.copy()
        node, score, refused, counts = spread_bind_packed(bfc, bfm, ac, am, labels, np.repeat(rc, R), np.repeat(rm, R),
                                                          np.repeat(sel, R, axis=0), np.zeros(R, np.int64), keys, skew,
                                                          mind, ex, policy)
        assert np.array_equal(node, want[1]) and np.array_equal(score, want[2]), it
        assert all(np.array_equal(a, b) for a, b in zip(counts, want[4])), it
        cfc, cfm = fc.copy(), fm.copy()
        for n in node[node >= 0]:
            cfc[n] -= rc[0]
            cfm[n] -= rm[0]
        assert np.array_equal(bfc, cfc) and np.array_equal(bfm, cfm), it
        if K == 1:
            one = spread_packed(fc, fm, ac, am, labels, rc, rm, sel, [R], *keys[0], skew[:, 0], mind[:, 0], ex[0],
                                policy)
            assert np.array_equal(node, one[1]) and np.array_equal(score, one[2]), it


@pytest.mark.parametrize("policy", POLICIES)
def test_skew_rule_and_refusals_at_each_turn(policy):
    """Mixed queues (no minDomains): every placed pod of a constrained group keeps each constrained key within its skew at
    its turn; an unconstrained pod refuses nothing; a pod left unbound with a feasible node refused every feasible node;
    refused never exceeds the feasible count at the pod's turn."""
    rng = np.random.default_rng(0x5B3 + policy)
    for it in range(120):
        fc, fm, ac, am, labels, rc, rm, sel, _ = random_cluster(rng, n_max=12)
        N = len(fc)
        K = int(rng.integers(1, 4))
        keys = _random_keys(rng, N, K)
        G = int(rng.integers(1, 5))
        P = int(rng.integers(1, 40))
        qc, qm, qs, group = _queue(rng, rc, rm, sel, G, P)
        skew = rng.integers(0, 3, (G, K))
        ex = [rng.integers(0, 3, (G, d)) for _, d in keys]
        bfc, bfm = fc.copy(), fm.copy()
        node, _, refused, _ = spread_bind_packed(bfc, bfm, ac, am, labels, qc, qm, qs, group, keys, skew, None, ex,
                                                 policy)
        assert skew_ok_at_each_turn(labels, qs, group, keys, skew, node, ex) is None, it
        f_c, f_m = fc.copy(), fm.copy()
        for p in range(P):
            feasible = int(((qc[p] <= f_c) & (qm[p] <= f_m) & ((qs[p][None, :] & ~labels) == 0).all(axis=1)).sum())
            assert refused[p] <= feasible, (it, p)
            if group[p] < 0 or not skew[group[p]].any():
                assert refused[p] == 0, (it, p)
            if node[p] < 0:
                assert refused[p] == feasible, (it, p)
            else:
                f_c[node[p]] -= qc[p]
                f_m[node[p]] -= qm[p]


def test_gv1_spread_bind_golden(ks):
    g = load_golden("gv1.json")
    want = load_golden("gv1_spread_bind.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        ac, am, lab = ctx.export_packed()[:3]
        rc, rm, sel = ctx.pack_pods(arena.pods(g["pods"]), len(g["pods"]))
    names = [p["name"] for p in g["pods"]]
    N = len(g["nodes"])
    key_of = {"zone": (want["zone_domain"], want["n_zones"]), "host": (list(range(N)), N)}
    for case in want["cases"]:
        runs = [case] + ([dict(case, **case["reordered"])] if "reordered" in case else [])
        for c in runs:
            i = [names.index(p) for p in c["pods"]]
            keys = [key_of[k] for k in c["keys"]]
            ex = None if "existing" not in c else [np.array([e[k] for e in c["existing"]]) for k in range(len(keys))]
            fc, fm = ac.copy(), am.copy()
            node, score, refused, counts = spread_bind_packed(fc, fm, ac, am, lab, rc[i], rm[i], sel[i], c["group"],
                                                              keys, c["max_skew"], c.get("min_domains"), ex, policy=0)
            assert node.tolist() == c["node"] and score.tolist() == c["score"], c["_why"]
            if c is case:
                assert refused.tolist() == c["refused"], c["_why"]
                assert [cn.tolist() for cn in counts] == c["counts"], c["_why"]
        if "reordered" in case:  # interleaving another workload changes the zone of workload 0's first pod
            assert case["node"][1] != case["reordered"]["node"][0], case["_why"]


def test_struct_and_constant_mirrors(ks):
    """KS_SPREAD_BIND_MAX_PODS / _GROUPS and KSH_RECONCILE_SPREAD_UNSATISFIED in the headers, the ctypes module and the
    Rust shim; both calls declared, exported and bound in Rust."""
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    hhdr = open(os.path.join(ROOT, "include", "ksched_host.h")).read()
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    assert "#define KS_SPREAD_BIND_MAX_PODS 65536u" in hdr and "#define KS_SPREAD_BIND_MAX_GROUPS 4096u" in hdr
    assert ks.capi.KS_SPREAD_BIND_MAX_PODS == 65536 and ks.capi.KS_SPREAD_BIND_MAX_GROUPS == 4096
    assert re.search(r"pub const KS_SPREAD_BIND_MAX_PODS: u32 = 65536;", rs)
    assert re.search(r"pub const KS_SPREAD_BIND_MAX_GROUPS: u32 = 4096;", rs)
    assert re.search(r"#define KSH_RECONCILE_SPREAD_UNSATISFIED 5\b", hhdr)
    assert ks.host.KSH_RECONCILE_SPREAD_UNSATISFIED == 5
    assert re.search(r"pub const KSH_RECONCILE_SPREAD_UNSATISFIED: c_int = 5;", rs)
    for fn in ("ks_spread_bind", "ksh_reconcile_spread"):
        assert fn in ks.declared_symbols() and hasattr(ks.lib, fn), fn
        assert re.search(r"pub fn %s\(" % fn, rs), fn
    # the ctypes prototype takes the header's ten arguments
    assert len(ks.lib.ks_spread_bind.argtypes) == 10 and len(ks.lib.ksh_reconcile_spread.argtypes) == 17


def test_errors_without_a_device(ks):
    """A NULL snapshot is refused on the host; the object-level call is KS_ERR_RANGE for a key count outside [1, 4] and
    KS_ERR_INVALID for a group outside [-1, n_groups) before it needs the device, and KS_ERR_NO_DEVICE on a
    packing-only context."""
    rc_, sel = np.zeros(1, np.int64), np.zeros(1, np.uint64)
    pods = ks.capi.ks_pods(1, rc_.ctypes.data, rc_.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
    grp, skew, dom = np.zeros(1, np.int32), np.ones(1, np.uint32), np.zeros(4, np.int32)
    idx = np.empty(1, np.int32)
    sp = ks.capi.ks_spread_multi(1, (C.c_uint32 * 4)(1), (C.c_void_p * 4)(dom.ctypes.data), skew.ctypes.data, None, None)
    assert ks.lib.ks_spread_bind(None, C.byref(pods), grp.ctypes.data, 1, C.byref(sp), 0, idx.ctypes.data, None, None,
                                 None) == ks.capi.KS_ERR_INVALID
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        p = arena.pods(g["pods"][:2])
        with pytest.raises(ks.KsError) as e:
            ctx.reconcile_spread(p, 2, [0, -1], 1, ["zone"], [1])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
        with pytest.raises(ks.KsError) as e:
            ctx.reconcile_spread(p, 2, [0, 1], 1, ["zone"], [1])
        assert e.value.code == ks.capi.KS_ERR_INVALID
        keys = (C.c_char_p * 5)(*[b"k"] * 5)
        ones, st, nd = np.ones(10, np.uint32), np.empty(2, np.int32), np.empty(2, np.int32)
        for k in (0, 5):
            assert ks.lib.ksh_reconcile_spread(ctx._h, C.addressof(p), 2, grp.ctypes.data, 0, C.cast(keys, C.c_void_p), k,
                                               ones.ctypes.data, None, None, None, 0, st.ctypes.data, nd.ctypes.data,
                                               None, 0, None) == ks.capi.KS_ERR_RANGE
