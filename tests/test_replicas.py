"""Replica placement (ks_place_replicas), CPU part: the merge restatement of tests/replicas_oracle.py against the
one-copy-at-a-time restatement on thousands of random small clusters (both policies, LEAST_ALLOCATED plateaus, ties,
allocatable <= 0, negative free, zero requests, one zero request, selectors); the hand-derived GV-1 plans of
tests/golden/gv1_replicas.json; argument errors caught before any device work; and the C / ctypes / Rust mirrors of the
row."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from helpers import load_golden
from replicas_oracle import PLAN_DTYPE, U64_MAX, merge_packed, sequential_packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def random_cluster(rng, n_max=8, t_max=4, r_max=12):
    """A small cluster whose values are multiples of small units, so scores tie and LEAST_ALLOCATED plateaus."""
    N, T = int(rng.integers(1, n_max + 1)), int(rng.integers(1, t_max + 1))
    uc, um = int(rng.choice([1, 7, 250])), int(rng.choice([1, 3, 1 << 20]))
    ac = rng.choice([-2, 0, 1, 4, 8, 16], N).astype(np.int64) * uc
    am = rng.choice([-1, 0, 2, 4, 16], N).astype(np.int64) * um
    fc = (rng.integers(-2, 17, N) * uc).astype(np.int64)
    fm = (rng.integers(-1, 17, N) * um).astype(np.int64)
    if rng.random() < 0.5:  # identical nodes: every score ties across nodes
        fc[:], fm[:], ac[:], am[:] = fc[0], fm[0], ac[0], am[0]
    labels = rng.integers(0, 4, (N, 1)).astype(np.uint64)
    rc = (rng.integers(0, 4, T) * uc).astype(np.int64)
    rm = (rng.integers(0, 4, T) * um).astype(np.int64)
    zero = rng.random(T)
    rc[zero < 0.15] = 0
    rm[(zero > 0.1) & (zero < 0.25)] = 0
    sel = np.where(rng.random((T, 1)) < 0.3, rng.integers(1, 4, (T, 1)), 0).astype(np.uint64)
    R = rng.integers(0, r_max + 1, T).astype(np.uint32)
    return fc, fm, ac, am, labels, rc, rm, sel, R


def test_merge_equals_one_copy_at_a_time(orc):
    rng = np.random.default_rng(0x5EED)
    cases = 0
    for it in range(2500):
        fc, fm, ac, am, labels, rc, rm, sel, R = random_cluster(rng)
        for policy in (0, 1):
            got = merge_packed(fc, fm, ac, am, labels, rc, rm, sel, R, policy)
            want = sequential_packed(orc, fc, fm, ac, am, labels, rc, rm, sel, R, policy)
            for a, b in zip(got, want):
                assert np.array_equal(a, b), (it, policy, got, want)
            cases += len(rc)
    assert cases > 10000


def test_zero_request_is_unbounded_and_stays_on_one_node():
    fc, fm = np.array([4, 9, 9], np.int64), np.array([4, 9, 9], np.int64)
    rows, node, score, _ = merge_packed(fc, fm, fc, fm, np.zeros((3, 1)), [0], [0], np.zeros((1, 1)), [5])
    assert int(rows["capacity"][0]) == U64_MAX and node.tolist() == [1] * 5 and rows["max_per_node"][0] == 5


def test_one_zero_request_divides_by_the_other():
    fc, fm = np.array([5, 3], np.int64), np.array([0, 0], np.int64)
    rows, node, _, _ = merge_packed(fc, fm, fc, fm + 1, np.zeros((2, 1)), [2], [0], np.zeros((1, 1)), [9])
    assert rows["capacity"][0] == 3 and rows["placed"][0] == 3 and node[:3].tolist() == [0, 0, 1]


def test_capacity_below_replicas_pads_with_minus_one():
    fc, fm = np.array([3, 2], np.int64), np.array([8, 8], np.int64)
    rows, node, score, off = merge_packed(fc, fm, fc, fm, np.zeros((2, 1)), [1, 1], [1, 1], np.zeros((2, 1)), [9, 2])
    assert rows["capacity"].tolist() == [5, 5] and rows["placed"].tolist() == [5, 2]
    assert node[5:9].tolist() == [-1] * 4 and score[5:9].tolist() == [0] * 4 and off.tolist() == [0, 9, 11]


def test_gv1_replicas_golden(ks, orc):
    g = load_golden("gv1.json")
    want = load_golden("gv1_replicas.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        ac, am, lab = ctx.export_packed()[:3]
        rc, rm, sel = ctx.pack_pods(arena.pods(g["pods"]), len(g["pods"]))
    names = [p["name"] for p in g["pods"]]
    idx = [names.index(p) for p in want["specs"]]
    fc, fm = orc.free_reduce(ac, am, np.zeros(0, np.int32), np.zeros(0, np.int64), np.zeros(0, np.int64))
    for policy, plan in (("leftover", 0), ("least_allocated", 1)):
        R = np.array(want["replicas"], np.uint32)
        rows, node, score, off = merge_packed(fc, fm, ac, am, lab, rc[idx], rm[idx], sel[idx], R, plan)
        seq = sequential_packed(orc, fc, fm, ac, am, lab, rc[idx], rm[idx], sel[idx], R, plan)
        assert all(np.array_equal(a, b) for a, b in zip((rows, node, score, off), seq))
        for t, w in enumerate(want[policy]):
            assert {f: int(rows[f][t]) for f in w["row"]} == w["row"], (policy, t)
            a, b = int(off[t]), int(off[t + 1])
            assert node[a:b].tolist() == w["node"] and score[a:b].tolist() == w["score"], (policy, t)


def test_plan_struct_mirrors(ks):
    """ks_replica_plan: 32 bytes; the ctypes struct, the numpy record and the Rust shim list the header's fields."""
    assert C.sizeof(ks.capi.ks_replica_plan) == 32 and ks.capi.REPLICA_PLAN_DTYPE.itemsize == 32
    assert ks.capi.REPLICA_PLAN_DTYPE == PLAN_DTYPE
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    body = re.search(r"typedef struct ks_replica_plan \{(.*?)\} ks_replica_plan;", hdr, re.S).group(1)
    c_fields = re.findall(r"\b([a-z_]+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert c_fields == [f[0] for f in ks.capi.ks_replica_plan._fields_] == list(PLAN_DTYPE.names)
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    rbody = re.search(r"pub struct ks_replica_plan \{(.*?)\n\}", rs, re.S).group(1)
    assert re.findall(r"pub ([a-z_0-9]+):", rbody) == c_fields
    for name, value in (("KS_REPLICAS_MAX_SPECS", 4096), ("KS_REPLICAS_MAX", 65536), ("KS_REPLICAS_MAX_TOTAL", 1 << 24)):
        assert getattr(ks.capi, name) == value
        assert re.search(r"pub const %s: u32 = ([^;]+);" % name, rs), name
    assert "ks_place_replicas" in ks.declared_symbols() and hasattr(ks.lib, "ks_place_replicas")
    assert "ksh_place_replicas" in ks.declared_symbols() and hasattr(ks.lib, "ksh_place_replicas")


def _pods(ks, n, rc=0, rm=0):
    a = np.full(max(n, 1), rc, np.int64), np.full(max(n, 1), rm, np.int64), np.zeros(max(n, 1), np.uint64)
    return ks.capi.ks_pods(n, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, ks.KS_MEM_HOST), a


def test_argument_errors_before_any_device_work(ks):
    """A NULL snapshot is refused on the host, without a device (the other argument errors are checked on the GPU,
    where a snapshot can be created)."""
    out = (ks.capi.ks_replica_plan * 4)()
    pods, keep = _pods(ks, 1)
    rep = np.ones(4, np.uint32)
    assert ks.lib.ks_place_replicas(None, C.byref(pods), rep.ctypes.data, 0, out, None, None) == ks.capi.KS_ERR_INVALID


def test_no_device_context(ks):
    """A packing-only host context has no snapshot: the object-level call is KS_ERR_NO_DEVICE."""
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        with pytest.raises(ks.KsError) as e:
            ctx.place_replicas(arena.pods(g["pods"][:2]), 2, [3, 1])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE


def test_widest_score_range_one_copy_at_a_time(orc):
    """The restatements agree where LEAST_ALLOCATED scores are widest: an allocatable of 1 B with 2^55 B free."""
    fc, fm = np.array([1000, 1000, 1000], np.int64), np.array([1 << 55, 1 << 30, 1 << 30], np.int64)
    ac, am = np.array([1000, 1000, 1000], np.int64), np.array([1, 1 << 30, 1 << 30], np.int64)
    lab, sel = np.zeros((3, 1), np.uint64), np.zeros((1, 1), np.uint64)
    for policy in (0, 1):
        for r in (1, 15, 16, 30):
            got = merge_packed(fc, fm, ac, am, lab, [100], [1 << 20], sel, [r], policy)
            want = sequential_packed(orc, fc.copy(), fm.copy(), ac, am, lab, np.array([100]), np.array([1 << 20]), sel,
                                     [r], policy)
            assert all(np.array_equal(a, b) for a, b in zip(got, want)), (policy, r)
    assert got[2][0] > 1 << 60  # copy 0 under LEAST_ALLOCATED: 2^55 B left of a 1-byte allocatable
