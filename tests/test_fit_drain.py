"""Drain simulation under the full filter (ks_fit_drain_check), CPU part: the restatement of tests/fit_drain_oracle.py
against the hand-derived cases of tests/golden/gv1_fit_drain.json, identities D1 (against drain_oracle.drain_packed),
D2, D3, D4 and D5 between restatements, the C / ctypes / Rust mirrors, and the argument errors caught before any device
work."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import fit_drain_oracle as fdo
from drain_oracle import drain_packed
from helpers import load_golden
from policy_oracle import Oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = load_golden("gv1_fit_drain.json")["cases"]


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden_cases(case, orc):
    d = fdo.golden_case(case)
    placed, idx, _, refused = fdo.fit_drain(d, d["node_idx"], d["offset"])
    assert placed.tolist() == case["want"]["placed"] and idx.tolist() == case["want"]["node_idx"]
    assert refused.tolist() == case["want"]["refused"]
    # what ks_drain_check, blind to the new filters, makes of the same candidates
    dp, di, _ = drain_packed(orc, d["fc"], d["fm"], d["ac"], d["am"], d["labels"], d["rc"], d["rm"], d["sel"],
                             d["node_idx"], d["offset"])
    assert dp.tolist() == case["drain_want"]["placed"] and di.tolist() == case["drain_want"]["node_idx"]


@pytest.mark.parametrize("policy", [0, 1, 3, 4])
@pytest.mark.parametrize("exclude", [False, True])
def test_d1_without_rules_and_resources_is_ks_drain_check(orc, policy, exclude):
    o = Oracle(orc)
    for seed in range(2):
        d = fdo.random_cluster(np.random.default_rng(seed), 30, 12)
        want = drain_packed(o, d["fc"], d["fm"], d["ac"], d["am"], d["labels"], d["rc"], d["rm"], d["sel"],
                            d["node_idx"], d["offset"], policy, exclude)
        got = fdo.fit_drain(d, d["node_idx"], d["offset"], policy, exclude, with_rules=False, with_res=False)
        assert all(np.array_equal(a, b) for a, b in zip(got[:3], want))


def test_d2_a_copy_of_cpu_changes_nothing():
    for seed in range(4):
        d = fdo.random_cluster(np.random.default_rng(10 + seed), 30, 12)
        d["rc"] = np.maximum(d["rc"], 1)
        a = fdo.fit_drain(d, d["node_idx"], d["offset"])
        e = dict(d)
        bound_cpu = np.zeros(len(d["fc"]), np.int64)
        np.add.at(bound_cpu, d["bn"], d["bc"])
        e["alloc"] = [dict(m, **{"cpu-copy": int(c)}) for m, c in zip(d["alloc"], d["ac"])]
        e["bound"] = [(n, dict(r, **{"cpu-copy": int(c)})) for (n, r), c in zip(d["bound"], d["bc"])]
        e["pod_res"] = [dict(r, **{"cpu-copy": int(c)}) for r, c in zip(d["pod_res"], d["rc"])]
        b = fdo.fit_drain(e, e["node_idx"], e["offset"])
        assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_d3_no_rule_and_ample_resources_is_d1():
    for seed in range(4):
        d = fdo.random_cluster(np.random.default_rng(20 + seed), 30, 12)
        for n in d["node_taints"]:
            n.clear()
        d["group_rules"] = [{} for _ in d["group_rules"]]
        big = 1 << 40
        d["alloc"] = [{k: big for k in list(a) + ["pods"]} for a in d["alloc"]]
        for a in d["alloc"]:
            for r in d["names"]:
                a[r] = big
        full = fdo.fit_drain(d, d["node_idx"], d["offset"])
        bare = fdo.fit_drain(d, d["node_idx"], d["offset"], with_rules=False, with_res=False)
        assert all(np.array_equal(x, y) for x, y in zip(full, bare))


def test_d4_replay_and_d5_words_sum_to_the_destinations():
    drainable = stopped = 0
    for seed in range(6):
        d = fdo.random_cluster(np.random.default_rng(30 + seed), 25, 15)
        for exclude in (False, True):
            placed, idx, _, refused = fdo.fit_drain(d, d["node_idx"], d["offset"], exclude=exclude)
            size = np.diff(d["offset"]).astype(np.int64)
            for c in range(len(size)):
                if placed[c] == size[c]:
                    assert fdo.replay_ok(d, d["node_idx"], d["offset"], c, idx)
                    assert refused[c].sum() == 0
                    drainable += 1
                else:
                    assert refused[c].sum() == fdo.destinations(d, d["node_idx"], c, exclude)
                    stopped += 1
    assert drainable > 10 and stopped > 10


def test_struct_and_prototype_mirrors(ks):
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    decl = re.search(r"int ks_fit_drain_check\((.*?)\);", hdr, re.S).group(1)
    assert len(re.sub(r"/\*.*?\*/", "", decl, flags=re.S).split(",")) == 13
    assert "ks_fit_drain_check" in ks.declared_symbols() and hasattr(ks.lib, "ks_fit_drain_check")
    assert len(ks.lib.ks_fit_drain_check.argtypes) == 13
    hh = open(os.path.join(ROOT, "include", "ksched_host.h")).read()
    decl = re.search(r"int ksh_drain_fit_nodes\((.*?)\);", hh, re.S).group(1)
    assert len(re.sub(r"/\*.*?\*/", "", decl, flags=re.S).split(",")) == 13
    assert len(ks.lib.ksh_drain_fit_nodes.argtypes) == 13
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    for name in ("ks_fit_drain_check", "ksh_drain_fit_nodes"):
        m = re.search(rf"pub fn {name}\((.*?)\) -> c_int;", rs, re.S)
        assert m and len(m.group(1).split(",")) == 13, name


def test_errors_without_a_device(ks):
    """A NULL snapshot is KS_ERR_INVALID before anything is read (the checks that need a snapshot run in
    tests/test_fit_drain_gpu.py); Snapshot.fit_drain_check refuses wrongly shaped arrays with ValueError first."""
    rc_, sel = np.zeros(1, np.int64), np.zeros(1, np.uint64)
    pods = ks.capi.ks_pods(1, rc_.ctypes.data, rc_.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
    grp, node, off = np.zeros(1, np.int32), np.zeros(1, np.int32), np.array([0, 1], np.uint64)
    cand = ks.capi.ks_drain_candidates(1, node.ctypes.data, off.ctypes.data)
    placed, idx = np.zeros(1, np.uint32), np.zeros(1, np.int32)
    assert ks.lib.ks_fit_drain_check(None, C.byref(pods), grp.ctypes.data, 1, None, None, C.byref(cand), 0, 0,
                                     placed.ctypes.data, idx.ctypes.data, None, None) == ks.capi.KS_ERR_INVALID
    assert "snapshot is NULL" in ks.lib.ks_last_error().decode()
    snap = ks.Snapshot.__new__(ks.Snapshot)
    snap._h = None  # N = 0
    P = 3
    rc, sel = np.zeros(P, np.int64), np.zeros((P, 0), np.uint64)
    g, nd, of = np.zeros(P, np.int32), np.zeros(1, np.int32), np.array([0, P], np.uint64)
    bad = [
        dict(node_free=np.zeros(0, np.int64), pod_req=np.ones((P, 1), np.int64)),  # 1-D node_free
        dict(node_free=np.zeros((1, 5), np.int64), pod_req=np.ones((P, 1), np.int64)),  # 5 columns, 0 nodes
        dict(node_free=np.zeros((2, 0), np.int64), pod_req=np.ones((P, 1), np.int64)),  # pod_req short
        dict(node_free=np.zeros((1, 0), np.int64), pod_req=np.ones((P - 1, 1), np.int64)),  # one pod short
        dict(node_free=np.zeros((1, 0), np.int64), pod_req=None),  # pod_req missing
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            snap.fit_drain_check(rc, rc, sel, g, 1, nd, of, **kw)
    with pytest.raises(ValueError):
        snap.fit_drain_check(rc, rc, sel, g[:2], 1, nd, of)  # group short
    with pytest.raises(ValueError):
        snap.fit_drain_check(rc, rc, sel, g, 1, nd, of[:1])  # offset short
    with pytest.raises(ks.KsError) as e:
        snap.fit_drain_check(rc, rc, sel, g, 1, nd, of)
    assert e.value.code == ks.capi.KS_ERR_INVALID


def test_host_layer_errors_on_a_packing_only_context(ks):
    """ksh_drain_fit_nodes: NULL arguments, offsets, groups, node names and group_rules shapes are refused before the
    device check; a well-formed call on a packing-only context is KS_ERR_NO_DEVICE."""
    lib = ks.lib
    arena = ks.objects.ObjectArena()
    pods = arena.pods([{"name": f"q{i}", "ns": "w", "node_name": "a", "containers": [{"cpu": "1", "nvidia.com/gpu": "8"}]}
                       for i in range(3)])
    grp = np.zeros(3, np.int32)
    off = np.array([0, 3], np.uint64)
    placed, node, ref = np.zeros(1, np.uint32), np.zeros(3, np.int32), np.zeros(4, np.uint32)
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes([{"name": "a", "allocatable": {"cpu": "4", "memory": "1024", "pods": "4"}}]), 1)
        names = (C.c_char_p * 1)(b"a")
        h, P = ctx._h, C.addressof(pods)

        def call(c=h, nm=C.addressof(names), p=P, o=off.ctypes.data, g=grp.ctypes.data, G=1, pl=placed.ctypes.data,
                 ni=node.ctypes.data):
            return lib.ksh_drain_fit_nodes(c, nm, 1, p, o, g, G, None, 0, 0, pl, ni, ref.ctypes.data)

        for bad in (dict(c=None), dict(nm=None), dict(p=None), dict(o=None), dict(g=None), dict(pl=None),
                    dict(ni=None)):
            assert call(**bad) == ks.capi.KS_ERR_INVALID, bad
        assert call(G=0) == ks.capi.KS_ERR_INVALID  # group 0 outside [-1, 0)
        other = (C.c_char_p * 1)(b"zz")
        assert call(nm=C.addressof(other)) == ks.capi.KS_ERR_INVALID  # not in the store
        assert call() == ks.capi.KS_ERR_NO_DEVICE
        with pytest.raises(ValueError):
            ctx.drain_fit_nodes(["a"], pods, off, grp, 1, group_rules=[{}, {}])
        with pytest.raises(ValueError):
            ctx.drain_fit_nodes(["a"], pods, off, grp[:2], 1)
        with pytest.raises(ks.KsError) as e:
            ctx.drain_fit_nodes(["a"], pods, off, grp, 1, group_rules=[{}])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
