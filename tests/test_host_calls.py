"""The object-level calls of include/ksched_host.h at their edges: what each of the 13 calls that need the device does
on a packing-only context (code, message, and whether it packed first), the argument errors each one checks and in
which order, what a library without an optional device entry reports, and the string-list outputs under a buffer
that is too small.  The -m gpu tests here also run against the host layer linked with a fake device
(tests/native/ksh_fake_device.cpp, which has none of the optional entries) in test_host_layer.py."""
import ctypes as C

import numpy as np
import pytest

from helpers import string_list_cases

NODES = [{"name": "n0", "labels": {"zone": "a", "disk": "ssd"}, "allocatable": {"cpu": "4", "memory": "8Gi"}},
         {"name": "n1", "labels": {"zone": "b"}, "allocatable": {"cpu": "2", "memory": "4Gi"}},
         {"name": "n2", "labels": {"zone": "a"}, "allocatable": {"cpu": "1", "memory": "2Gi"}}]
PENDING = [{"name": "p0", "ns": "d", "containers": [{"cpu": "500m", "memory": "1Gi"}], "selector": {"zone": "a"}},
           {"name": "p1", "ns": "d", "containers": [{"cpu": "1", "memory": "1Gi"}], "selector": {"disk": "ssd"}}]
BOUND = [{"name": "b0", "ns": "d", "node_name": "n0", "containers": [{"cpu": "1", "memory": "1Gi"}]}]
NO_DEVICE = "packing-only context (KSH_DEVICE_NONE): no device snapshot, nothing is computed on the host"


class Call:
    """One ksh_* call through the bare ABI (no binding code in between), on a context with NODES set."""

    def __init__(self, ks, ctx):
        self.ks, self.lib, self.h = ks, ks.lib, ctx._h
        self.arena = ks.objects.ObjectArena()
        self.pods = self.arena.pods(PENDING)
        self.bound = self.arena.pods(BOUND)
        self.templates = self.arena.nodes(NODES[:1])
        self.keep = []

    def buf(self, n, dtype):
        a = np.zeros(max(int(n), 1), dtype)
        self.keep.append(a)
        return a.ctypes.data

    def __call__(self, name, n):
        b, lib, h, P = self.buf, self.lib, self.h, C.addressof(self.pods)
        I32, I64, U32, U64 = np.int32, np.int64, np.uint32, np.uint64
        if name == "check_node_validity":
            return lib.ksh_check_node_validity(h, P, 0)
        if name == "select_nodes":
            return lib.ksh_select_nodes(h, P, n, 0, b(n, I32), b(n, I64), b(n, U32))
        if name == "rank_nodes":
            return lib.ksh_rank_nodes(h, P, n, 0, 2, b(2 * n, I32), b(2 * n, I64), b(n, U32))
        if name == "select_node_for_pod":
            return lib.ksh_select_node_for_pod(h, P, n, 5, 7, 0, b(n, I32), b(n, U32), b(5 * n, I32), b(5 * n, np.uint8))
        if name == "reconcile":
            node = C.c_int32()
            return lib.ksh_reconcile(h, P, 0, C.byref(node), C.create_string_buffer(256), 256)
        if name == "reconcile_batch":
            return lib.ksh_reconcile_batch(h, P, n, 0, b(n, I32), b(n, I32), b(4096, np.uint8), 4096, b(n, I64), None)
        if name == "reconcile_gangs":
            off = np.array([0, n] if n else [0], U64)
            mm = np.array([1] if n else [], U32)
            self.keep += [off, mm]
            return lib.ksh_reconcile_gangs(h, P, n, off.ctypes.data, len(off) - 1, mm.ctypes.data, 0, b(n, I32), b(n, I32),
                                           b(1, U32), b(4096, np.uint8), 4096, b(n, I64))
        if name == "explain_pods":
            return lib.ksh_explain_pods(h, P, n, b(4 * n, U32), b(4096, np.uint8), 4096, b(n, I64))
        if name == "preempt_pods":
            return lib.ksh_preempt_pods(h, P, n, b(n, I32), 4, b(4 * n, U64), b(4096, np.uint8), 4096, b(n, I64))
        if name == "drain_nodes":
            names = (C.c_char_p * 1)(b"n0")
            off = np.array([0, 1] if n else [0], U64)
            self.keep += [names, off]
            return lib.ksh_drain_nodes(h, C.addressof(names), min(n, 1), C.addressof(self.bound), off.ctypes.data, 0, 0,
                                       b(1, U32), b(1, I32))
        if name == "place_replicas":
            return lib.ksh_place_replicas(h, P, n, b(n, U32) if not n else np.full(n, 2, U32).ctypes.data, 0,
                                          b(3 * n, U64), None, None)
        if name == "place_replicas_spread":
            rep = np.full(max(n, 1), 2, U32)
            self.keep.append(rep)
            return lib.ksh_place_replicas_spread(h, P, n, rep.ctypes.data, b"zone", rep.ctypes.data, None, None, None, 0,
                                                 b(4 * n, U64), None, None, None)
        if name == "scaleup_estimate":
            best = C.c_int32()
            mx = np.full(1, 4, U32)
            self.keep.append(mx)
            return lib.ksh_scaleup_estimate(h, C.addressof(self.templates), min(n, 1), mx.ctypes.data, None, 0, P, n,
                                            b(4, U64), C.addressof(best), None, None)
        raise KeyError(name)


CALLS = ["check_node_validity", "select_nodes", "rank_nodes", "select_node_for_pod", "reconcile", "reconcile_batch",
         "reconcile_gangs", "explain_pods", "preempt_pods", "drain_nodes", "place_replicas", "place_replicas_spread",
         "scaleup_estimate"]


def _outcome(ks, device, name, n):
    with ks.host.Context(device) as ctx:
        ctx.set_nodes(ks.objects.ObjectArena().nodes(NODES), len(NODES))
        rc = Call(ks, ctx)(name, n)
        msg = ks.lib.ks_last_error().decode() if rc < 0 else ""
        return rc, msg, ctx.label_words, ctx.export_packed()[2].tolist()


# Packing-only context: (n > 0, n == 0) -> (code, message, node label words after the call).  The calls without a
# snapshot check of their own pack the batch before upload() refuses, which gives the selector pairs dictionary bits
# (zone=a bit 0, disk=ssd bit 1); the others refuse first.
NONE = [[0], [0], [0]]
ONE = [[1], [0], [1]]   # pod 0 alone
BOTH = [[3], [0], [1]]
PACKING_ONLY = {
    "check_node_validity": ((-8, NO_DEVICE, ONE), None),
    "select_nodes": ((-8, NO_DEVICE, BOTH), (0, "", NONE)),
    "rank_nodes": ((-8, NO_DEVICE, NONE), (-8, NO_DEVICE, NONE)),
    "select_node_for_pod": ((-8, NO_DEVICE, BOTH), (0, "", NONE)),
    "reconcile": ((-8, NO_DEVICE, ONE), None),
    "reconcile_batch": ((-8, NO_DEVICE, BOTH), (0, "", NONE)),
    "reconcile_gangs": ((-8, NO_DEVICE, NONE), (-8, NO_DEVICE, NONE)),
    "explain_pods": ((-8, NO_DEVICE, NONE), (-8, NO_DEVICE, NONE)),
    "preempt_pods": ((-8, NO_DEVICE, NONE), (-8, NO_DEVICE, NONE)),
    "drain_nodes": ((-8, NO_DEVICE, NONE), (-8, NO_DEVICE, NONE)),
    "place_replicas": ((-8, NO_DEVICE, NONE), (-8, NO_DEVICE, NONE)),
    "place_replicas_spread": ((-8, NO_DEVICE, NONE), (-8, NO_DEVICE, NONE)),
    "scaleup_estimate": ((-8, NO_DEVICE, NONE), (-8, NO_DEVICE, NONE)),
}


@pytest.mark.parametrize("name", CALLS)
def test_packing_only_outcome(ks, name):
    for n, want in zip((2, 0), PACKING_ONLY[name]):
        if want is None:  # one pod by definition
            continue
        rc, msg, w, lab = _outcome(ks, ks.host.KSH_DEVICE_NONE, name, n)
        assert (rc, msg, w, lab) == want[:2] + (1, want[2]), (name, n)


# A library whose device side lacks an optional entry (the fake device has none of them): (n > 0, n == 0) -> (code,
# message, node label words after the call).  Only these eight calls use the optional entries.
STAND_IN = {
    "rank_nodes": ((-8, "this library has no ks_select_topk", NONE), (-8, "this library has no ks_select_topk", NONE)),
    "reconcile_gangs": ((-8, "this library has no ks_gang_bind", NONE), (-8, "this library has no ks_gang_bind", NONE)),
    "explain_pods": ((-8, "this library has no ks_explain", NONE), (-8, "this library has no ks_explain", NONE)),
    "preempt_pods": ((-8, "this library has no ks_preempt", NONE), (-8, "this library has no ks_preempt", NONE)),
    "drain_nodes": ((-8, "this library has no ks_drain_check", NONE), (-8, "this library has no ks_drain_check", NONE)),
    "place_replicas": ((-8, "this library has no ks_place_replicas", NONE),
                       (-8, "this library has no ks_place_replicas", NONE)),
    "place_replicas_spread": ((-8, "this library has no ks_place_replicas_spread", NONE),
                              (-8, "this library has no ks_place_replicas_spread", NONE)),
    "scaleup_estimate": ((-8, "this library has no ks_scaleup_estimate", NONE),
                         (-8, "this library has no ks_scaleup_estimate", NONE)),
}
ENTRY = {"rank_nodes": "ks_select_topk", "reconcile_gangs": "ks_gang_bind", "explain_pods": "ks_explain",
         "preempt_pods": "ks_preempt", "drain_nodes": "ks_drain_check", "place_replicas": "ks_place_replicas",
         "place_replicas_spread": "ks_place_replicas_spread", "scaleup_estimate": "ks_scaleup_estimate"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(STAND_IN))
def test_library_without_the_entry(ks, name):
    if hasattr(ks.lib, ENTRY[name]):
        pytest.skip(f"this library defines {ENTRY[name]}")
    for n, want in zip((2, 0), STAND_IN[name]):
        rc, msg, w, lab = _outcome(ks, 0, name, n)
        assert (rc, msg, w, lab) == want[:2] + (1, want[2]), (name, n)


def _errors(ks, ctx):
    """(call, expected code, expected message) for every argument check, each case breaking the earliest check that it
    names and, where a later check exists, also a later one: the first check in the call's order must win."""
    lib, h = ks.lib, ctx._h
    arena = ks.objects.ObjectArena()
    pods = arena.pods(PENDING)
    P = C.addressof(pods)
    bound = arena.pods(BOUND + [{"name": "x", "ns": "d", "containers": []}])
    B = C.addressof(bound)
    z = np.zeros(4096, np.int64)
    Z = z.ctypes.data
    keep = []

    def arr(*v):
        a = np.array(v, np.uint64)
        keep.append(a)
        return a.ctypes.data

    def names(*v):
        a = (C.c_char_p * max(len(v), 1))(*v)
        keep.append(a)
        return C.addressof(a)

    dup = arena.nodes([NODES[0], NODES[0]])
    unbound_over = arena.pods([{"name": "o", "ns": "d", "containers": []}])
    lost_over = arena.pods([{"name": "o", "ns": "d", "node_name": "elsewhere", "containers": []}])
    bad_cpu = arena.nodes([{"name": "t", "allocatable": {"memory": "1"}}])
    tmpl = arena.nodes(NODES[:1])
    R, I = -5, -1
    AFTER = True  # checked after the device check: a library without the call's optional entry refuses first
    cases = [
        ("check_node_validity", lambda: lib.ksh_check_node_validity(None, P, 9), I, "NULL argument"),
        ("check_node_validity", lambda: lib.ksh_check_node_validity(h, P, 3), I, "node index out of range"),
        ("select_nodes", lambda: lib.ksh_select_nodes(h, None, 1, 0, Z, Z, Z), I, "NULL argument"),
        ("rank_nodes", lambda: lib.ksh_rank_nodes(h, None, 1, 0, 0, Z, Z, Z), I, "NULL argument"),
        ("rank_nodes", lambda: lib.ksh_rank_nodes(h, P, 1, 0, 0, None, Z, Z), R, "k must be in [1, 32]", AFTER),
        ("rank_nodes", lambda: lib.ksh_rank_nodes(h, P, 1, 0, 33, None, Z, Z), R, "k must be in [1, 32]", AFTER),
        ("rank_nodes", lambda: lib.ksh_rank_nodes(h, P, 1, 0, 1, None, Z, Z), I, "out_node_idx is NULL", AFTER),
        ("select_node_for_pod", lambda: lib.ksh_select_node_for_pod(h, None, 1, 5, 0, 0, Z, Z, Z, Z), I, "NULL argument"),
        ("reconcile", lambda: lib.ksh_reconcile(h, P, 0, None, None, 0), I, "NULL argument"),
        ("reconcile_batch", lambda: lib.ksh_reconcile_batch(h, P, 1, 0, None, Z, None, 0, None, None), I, "NULL argument"),
        ("reconcile_gangs", lambda: lib.ksh_reconcile_gangs(h, P, 2, None, 1, Z, 0, Z, Z, None, None, 0, None), I,
         "NULL argument"),
        ("reconcile_gangs", lambda: lib.ksh_reconcile_gangs(h, P, 2, arr(1, 0), 1, Z, 0, Z, Z, None, None, 0, None), I,
         "group_offset[0] must be 0"),
        ("reconcile_gangs", lambda: lib.ksh_reconcile_gangs(h, P, 2, arr(0, 2, 1), 2, Z, 0, Z, Z, None, None, 0, None), I,
         "group offsets decrease"),
        ("reconcile_gangs", lambda: lib.ksh_reconcile_gangs(h, P, 2, arr(0, 0, 2), 2, Z, 0, Z, Z, None, None, 0, None), R,
         "a group has 0 pods (1..1024)"),
        ("reconcile_gangs", lambda: lib.ksh_reconcile_gangs(h, P, 2, arr(0, 1), 1, arr(2), 0, Z, Z, None, None, 0, None),
         R, "min_member above the group's size"),
        ("reconcile_gangs", lambda: lib.ksh_reconcile_gangs(h, P, 2, arr(0, 1), 1, Z, 0, Z, Z, None, None, 0, None), I,
         "group_offset[n_groups] must be n_pods"),
        ("explain_pods", lambda: lib.ksh_explain_pods(h, P, 1, None, None, 0, None), I, "NULL argument"),
        ("preempt_pods", lambda: lib.ksh_preempt_pods(h, P, 1, None, 0, Z, None, 0, None), I, "NULL argument"),
        ("preempt_pods", lambda: lib.ksh_preempt_pods(h, P, 1, Z, 0, Z, None, 0, None), R, "max_victims must be in [1, 128]"),
        ("preempt_pods", lambda: lib.ksh_preempt_pods(h, P, 1, Z, 129, Z, None, 0, None), R,
         "max_victims must be in [1, 128]"),
        ("drain_nodes", lambda: lib.ksh_drain_nodes(h, names(b"n0"), 1, B, None, 0, 0, Z, Z), I, "NULL argument"),
        ("drain_nodes", lambda: lib.ksh_drain_nodes(h, names(b"n0"), 1, B, arr(1, 1), 0, 0, Z, Z), I,
         "pod_offset[0] must be 0"),
        ("drain_nodes", lambda: lib.ksh_drain_nodes(h, names(b"n0", b"n1"), 2, None, arr(0, 2, 1), 0, 0, Z, Z), I,
         "pod offsets decrease"),
        ("drain_nodes", lambda: lib.ksh_drain_nodes(h, names(b"n0"), 1, None, arr(0, 1), 0, 0, Z, Z), I, "NULL argument"),
        ("drain_nodes", lambda: lib.ksh_drain_nodes(h, names(None), 1, B, arr(0, 1), 0, 0, Z, Z), I,
         "candidate 0: node name is NULL"),
        ("drain_nodes", lambda: lib.ksh_drain_nodes(h, names(b"n9"), 1, B, arr(0, 1), 0, 0, Z, Z), I,
         "candidate 0: node \"n9\" is not in the store"),
        ("drain_nodes", lambda: lib.ksh_drain_nodes(h, names(b"n0"), 1, B, arr(0, 2), 0, 0, Z, Z), I,
         "pod 1 (d/x) has spec.nodeName \"\", not its candidate's node \"n0\""),
        ("place_replicas", lambda: lib.ksh_place_replicas(h, P, 1, None, 0, Z, None, None), I, "NULL argument"),
        ("place_replicas_spread", lambda: lib.ksh_place_replicas_spread(h, P, 1, Z, None, Z, None, None, None, 0, Z, None,
                                                                        None, None), I, "NULL argument"),
        ("place_replicas_spread", lambda: lib.ksh_place_replicas_spread(h, P, 1, Z, b"zone", Z, None, None, arr(0, 1), 0,
                                                                        Z, None, None, None), I,
         "NULL existing_node_names"),
        ("place_replicas_spread", lambda: lib.ksh_place_replicas_spread(h, P, 1, Z, b"zone", Z, None, names(b"n0"),
                                                                        arr(1, 0), 0, Z, None, None, None), I,
         "existing offsets decrease"),
        ("scaleup_estimate", lambda: lib.ksh_scaleup_estimate(h, C.addressof(tmpl), 1, Z, None, 0, P, 1, Z, None, None,
                                                              None), I, "NULL argument"),
        ("scaleup_estimate", lambda: lib.ksh_scaleup_estimate(h, C.addressof(tmpl), 1, Z, None, 0, P, 65537, Z, Z, None,
                                                              None), R, "more than 65536 pods or 4096 templates"),
        ("scaleup_estimate", lambda: lib.ksh_scaleup_estimate(h, C.addressof(dup), 2, Z, None, 0, P, 1, Z, Z, None, None),
         I, "template 1: duplicate name \"n0\""),
        ("scaleup_estimate", lambda: lib.ksh_scaleup_estimate(h, C.addressof(bad_cpu), 1, Z, None, 0, P, 1, Z, Z, None,
                                                              None), -7,
         "template 0: node 't': allocatable has no cpu (reference panics, predicates.rs:29)"),
        ("scaleup_estimate", lambda: lib.ksh_scaleup_estimate(h, C.addressof(tmpl), 1, Z, C.addressof(unbound_over), 1, P,
                                                              1, Z, Z, None, None), I,
         "overhead pod 0 (d/o) has no spec.nodeName naming its template"),
        ("scaleup_estimate", lambda: lib.ksh_scaleup_estimate(h, C.addressof(tmpl), 1, Z, C.addressof(lost_over), 1, P, 1,
                                                              Z, Z, None, None), I,
         "overhead pod 0 (d/o) names unknown template \"elsewhere\""),
        ("scaleup_estimate", lambda: lib.ksh_scaleup_estimate(h, C.addressof(tmpl), 1, Z, None, 0, B, 1, Z, Z, None, None),
         I, "pod 0 (d/b0) has spec.nodeName \"n0\": not a pending pod"),
    ]
    return cases, (keep, z, pods, bound, dup, unbound_over, lost_over, bad_cpu, tmpl, arena)


@pytest.mark.gpu
def test_argument_errors_in_order(ks):
    seen = set()
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(ks.objects.ObjectArena().nodes(NODES), len(NODES))
        cases, keep = _errors(ks, ctx)
        for name, call, code, text, *after in cases:
            if after and not hasattr(ks.lib, ENTRY[name]):
                code, text = -8, "this library has no " + ENTRY[name]
            rc = call()
            assert (rc, ks.lib.ks_last_error().decode()) == (code, text), name
            seen.add(name)
    assert seen == set(CALLS)


def test_topology_domain_names_under_a_small_buffer(ks):
    arena = ks.objects.ObjectArena()
    nodes = arena.nodes([{"name": "a", "labels": {"zone": "eu-west-long-zone-name"}},
                         {"name": "b", "labels": {"zone": "us"}},
                         {"name": "c", "labels": {"rack": "r1"}},
                         {"name": "d", "labels": {"zone": "ap-south"}}])
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(nodes, 4)
        dom, values = ctx.topology_domains("zone")
        assert dom.tolist() == [0, 1, -1, 2] and values == ["eu-west-long-zone-name", "us", "ap-south"]
        for cap, want in string_list_cases(values):
            d = np.empty(4, np.int32)
            n = C.c_uint32()
            buf = C.create_string_buffer(max(cap, 1))
            off = np.full(3, -7, np.int64)
            assert ks.lib.ksh_context_topology_domains(ctx._h, b"zone", d.ctypes.data, C.byref(n), buf, cap,
                                                       off.ctypes.data) == 0
            assert n.value == 3 and d.tolist() == dom.tolist()
            got = [None if o < 0 else C.string_at(C.addressof(buf) + int(o)).decode() for o in off]
            assert got == want, cap
            assert off.tolist() == [-1 if w is None else off[i] for i, w in enumerate(want)]
        # no buffer or no offsets: the offsets are not written
        off = np.full(3, -7, np.int64)
        assert ks.lib.ksh_context_topology_domains(ctx._h, b"zone", d.ctypes.data, C.byref(n), None, 64,
                                                   off.ctypes.data) == 0
        assert off.tolist() == [-7, -7, -7]


@pytest.mark.gpu
def test_reconcile_batch_bodies_under_a_small_buffer(ks):
    arena = ks.objects.ObjectArena()
    nodes = arena.nodes([{"name": "n0", "allocatable": {"cpu": "8", "memory": "8Gi"}}])
    pods_s = [{"name": "long", "ns": "d", "containers": [{"cpu": "1"}],
               "metadata_json": '{"name":"long","namespace":"d","labels":{"app":"' + "x" * 80 + '"}}'},
              {"name": "bound", "ns": "d", "node_name": "n0", "containers": []},
              {"name": "s", "ns": "d", "containers": [{"cpu": "1"}]},
              {"name": "mid", "ns": "d", "containers": [{"cpu": "1"}]}]
    full = None
    for step in range(4):
        with ks.host.Context(0) as ctx:
            ctx.set_nodes(nodes, 1)
            ctx.set_cluster_pods(arena.pods([]), 0)
            if full is None:
                st, nd, full, _ = ctx.reconcile_batch(arena.pods(pods_s), 4)
                assert st.tolist() == [0, 0, 0, 0] and nd.tolist() == [0, -1, 0, 0] and full[1] is None
                cases = string_list_cases(full)
                continue
            cap, want = cases[step - 1]
            st, nd, bodies, _ = ctx.reconcile_batch(arena.pods(pods_s), 4, json_cap=cap)
            assert st.tolist() == [0, 0, 0, 0] and nd.tolist() == [0, -1, 0, 0]
            assert bodies == want, cap
            assert ctx.num_bound == 3  # the bodies that did not fit are still bound
