"""Scale-up estimate (ks_scaleup_estimate), CPU part: the restatement of tests/scaleup_oracle.py against the hand-derived
GV-1 example of tests/golden/gv1_scaleup.json and against its special cases (max_nodes 1 is one first-fit bin,
identical pods take ceil nodes, the cpu:memory ratio of the allocatable sets the order, a pod after the node limit can
still fit an open node); argument errors caught before any device work; and the C / ctypes / Rust mirrors of the two
structs."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from helpers import load_golden
from scaleup_oracle import best_template, pack_template, scaleup_packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS_ERR_PARSE, KS_ERR_MISSING = -3, -7  # include/ksched.h


def _gv1_pods(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        rc, rm, _ = ctx.pack_pods(arena.pods(g["pods"]), len(g["pods"]))
    return [p["name"] for p in g["pods"]], rc, rm


def test_gv1_scaleup_golden(ks, orc):
    names, rc, rm = _gv1_pods(ks)
    g = load_golden("gv1_scaleup.json")
    assert names == g["pods"]
    t = g["templates"]
    ac, am = np.array(t["alloc_cpu"], np.int64), np.array(t["alloc_mem"], np.int64)
    fc, fm = np.array(t["free_cpu"], np.int64), np.array(t["free_mem"], np.int64)
    sel = np.zeros((len(rc), 1), np.uint64)
    rows, best, node, why = scaleup_packed(orc, ac, am, fc, fm, np.zeros((2, 1), np.uint64), t["max_nodes"], rc, rm, sel)
    for i, want in enumerate(g["rows"]):
        assert {f: int(rows[f][i]) for f in want} == want
    assert best == g["best"] and node.tolist() == g["node"]
    for i, name in enumerate(names):
        assert why[i].tolist() == g["reasons"].get(name, g["reasons"]["others"]), name
    for i, order in enumerate(g["order"]):  # the walk order: by the wide key, descending, then the pod index
        elig = [names.index(p) for p in order]
        key = [int(rc[p]) * int(am[i]) + int(rm[p]) * int(ac[i]) for p in elig]
        assert sorted(zip([-k for k in key], elig)) == list(zip([-k for k in key], elig))


def test_max_nodes_1_is_one_first_fit_bin(ks, orc):
    rng = np.random.default_rng(1)
    rc = rng.integers(0, 3000, 400).astype(np.int64)
    rm = rng.integers(0, 8 << 30, 400).astype(np.int64)
    row, where = pack_template(rc, rm, np.arange(400), 16000, 64 << 30, 16000, 64 << 30, 1)
    # one bin: walk the key order and take every pod that still fits
    order = sorted(range(400), key=lambda p: (-(int(rc[p]) * (64 << 30) + int(rm[p]) * 16000), p))
    left_c, left_m, took = 16000, 64 << 30, []
    for p in order:
        if rc[p] <= left_c and rm[p] <= left_m:
            left_c, left_m = left_c - rc[p], left_m - rm[p]
            took.append(p)
    assert sorted(where) == sorted(took) and set(where.values()) == {0} and row[:3] == (1, len(took), 400)


def test_identical_pods_take_ceil_nodes():
    rc, rm = np.full(1000, 700, np.int64), np.full(1000, 1 << 30, np.int64)
    for ac, am, per in ((4000, 64 << 30, 5), (64000, 4 << 30, 4), (7000, 10 << 30, 10)):
        row, _ = pack_template(rc, rm, np.arange(1000), ac, am, ac, am, 1024)
        assert row[0] == -(-1000 // per) and row[1] == 1000


def test_cpu_memory_ratio_sets_the_order():
    """A cpu-heavy and a memory-heavy pod swap places between a 1:1 and a 4:1 template (cpu m : memory B units)."""
    rc, rm = np.array([400, 100], np.int64), np.array([100, 300], np.int64)
    key = lambda ac, am: sorted(range(2), key=lambda p: (-(int(rc[p]) * am + int(rm[p]) * ac), p))
    assert key(1000, 1000) == [0, 1] and key(4000, 1000) == [1, 0]
    _, w1 = pack_template(rc, rm, [0, 1], 1000, 1000, 400, 300, 1)
    _, w2 = pack_template(rc, rm, [0, 1], 4000, 1000, 400, 300, 1)
    assert list(w1) == [0] and list(w2) == [1]  # the first pod walked takes the single node, the other no longer fits


def test_limit_reached_then_a_smaller_pod_fits():
    rc = np.array([3000, 3000, 3000, 500], np.int64)
    rm = np.array([1, 1, 1, 1], np.int64)
    row, where = pack_template(rc, rm, np.arange(4), 4000, 1 << 30, 4000, 1 << 30, 2)
    assert where == {0: 0, 1: 1, 3: 0} and row[:3] == (2, 3, 4)


def test_best_template_rule():
    dt = np.dtype([("nodes", np.uint32), ("placed", np.uint32), ("utilization", np.int32)])
    rows = np.array([(3, 5, 90), (2, 5, 90), (1, 5, 91), (9, 6, 10), (0, 0, 0)], dt)
    assert best_template(rows) == 3
    rows["placed"][3] = 5
    assert best_template(rows) == 2
    rows["utilization"][2] = 90
    assert best_template(rows) == 2  # fewest nodes
    rows["nodes"][2] = 2
    assert best_template(rows) == 1  # lowest index
    assert best_template(np.zeros(3, dt)) == -1


def test_scaleup_needs_a_snapshot(ks):
    E = ks.capi
    rc = np.zeros(1, np.int64)
    lab = np.zeros(1, np.uint64)
    mx = np.ones(1, np.uint32)
    out = (E.ks_scaleup_option * 1)()
    best = C.c_int32(0)
    pods = E.ks_pods(1, rc.ctypes.data, rc.ctypes.data, lab.ctypes.data, ks.KS_MEM_HOST)
    tm = E.ks_node_templates(1, 1, rc.ctypes.data, rc.ctypes.data, rc.ctypes.data, rc.ctypes.data, lab.ctypes.data,
                             mx.ctypes.data)
    assert ks.lib.ks_scaleup_estimate(None, C.byref(pods), C.byref(tm), C.addressof(out), C.addressof(best), None,
                                      None) == E.KS_ERR_INVALID
    assert "snapshot" in ks.lib.ks_last_error().decode()


def test_struct_mirrors_c_ctypes_rust(ks):
    cap = ks.capi
    assert C.sizeof(cap.ks_node_templates) == 64 and C.sizeof(cap.ks_scaleup_option) == 32
    assert cap.SCALEUP_OPTION_DTYPE.itemsize == 32
    assert [(n, cap.SCALEUP_OPTION_DTYPE.fields[n][1]) for n in cap.SCALEUP_OPTION_DTYPE.names] == \
        [(f[0], getattr(cap.ks_scaleup_option, f[0]).offset) for f in cap.ks_scaleup_option._fields_]
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    for name in ("KS_SCALEUP_MAX_NODES", "KS_SCALEUP_MAX_PODS", "KS_SCALEUP_MAX_TEMPLATES"):
        assert re.search(rf"#define {name} (\d+)u", hdr).group(1) == str(getattr(cap, name))
    src = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    for name in ("KS_SCALEUP_MAX_NODES", "KS_SCALEUP_MAX_PODS", "KS_SCALEUP_MAX_TEMPLATES"):
        assert re.search(rf"pub const {name}: u32 = (\d+);", src).group(1) == str(getattr(cap, name))
    for struct, rust in (("ks_node_templates", [("n", "u64"), ("label_words", "u32"), ("alloc_cpu", "*const i64"),
                                                ("alloc_mem", "*const i64"), ("free_cpu", "*const i64"),
                                                ("free_mem", "*const i64"), ("labels", "*const u64"),
                                                ("max_nodes", "*const u32")]),
                         ("ks_scaleup_option", [("nodes", "u32"), ("placed", "u32"), ("eligible", "u32"),
                                                ("utilization", "i32"), ("used_cpu", "i64"), ("used_mem", "i64")])):
        body = re.search(rf"typedef struct {struct} \{{(.*?)\}} {struct};", hdr, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = [n for decl in body.split(";") for n in re.findall(r"\**([a-z_]+)\s*(?:,|$)", decl.strip())]
        assert names == [f[0] for f in getattr(cap, struct)._fields_], struct
        body = re.search(rf"pub struct {struct} \{{(.*?)\n\}}", src, re.S).group(1)
        assert re.findall(r"pub ([a-z_]+): ([^,]+),", body) == rust, struct
    fns = set(re.findall(r"pub fn (ksh?_[a-z0-9_]+)\(", src))
    assert {"ks_scaleup_estimate", "ksh_context_snapshot"} <= fns and hasattr(ks.lib, "ks_scaleup_estimate")
    wrapper = open(os.path.join(ROOT, "examples", "rust_shim", "ksched.rs")).read()
    assert "pub fn scaleup_estimate(" in wrapper


def _host_case():
    """Three templates of node groups (instance type and zone labels), two DaemonSet pods each, pending pods with and
    without selectors."""
    tmpl = [{"name": f"group-{i}", "labels": {"node.kubernetes.io/instance-type": t, "zone": z},
             "allocatable": {"cpu": f"{c}m", "memory": str(m)}}
            for i, (t, z, c, m) in enumerate([("m5.xlarge", "a", 4000, 16 << 30), ("m5.2xlarge", "a", 8000, 32 << 30),
                                              ("r5.xlarge", "b", 4000, 32 << 30)])]
    ds = [{"name": f"ds-{k}-{i}", "node_name": f"group-{i}", "containers": [{"cpu": "100m", "memory": str(200 << 20)}]}
          for i in range(3) for k in range(2)]
    rng = np.random.default_rng(0x5CA1E)
    pods = []
    for p in range(400):
        spec = {"name": f"p{p}", "containers": [{"cpu": f"{int(rng.integers(50, 3000))}m",
                                                 "memory": str(int(rng.integers(1, 12 << 30)))}]}
        r = p % 5
        if r == 1:
            spec["selector"] = {"node.kubernetes.io/instance-type": "m5.2xlarge"}  # only a template carries it
        elif r == 2:
            spec["selector"] = {"zone": "b"}
        elif r == 3:
            spec["selector"] = {"disk": "ssd"}  # no template carries it
        pods.append(spec)
    return tmpl, [12, 5, 30], ds, pods


def test_host_layer_argument_errors_before_device_work(ks):
    E = ks.capi
    tmpl, mx, ds, pods = _host_case()
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        def code(t=tmpl, m=mx, o=ds, p=pods):
            with pytest.raises(ks.KsError) as e:
                ctx.scaleup_estimate(arena.nodes(t) if t else None, len(t), m, arena.pods(p) if p else None, len(p),
                                     arena.pods(o) if o else None, len(o))
            return e.value.code, str(e.value)

        assert code()[0] == E.KS_ERR_NO_DEVICE  # well formed: reaches the device check
        c, msg = code(t=tmpl + [dict(tmpl[0])], m=mx + [1])
        assert c == E.KS_ERR_INVALID and "duplicate" in msg and "group-0" in msg
        c, msg = code(o=ds + [{"name": "stray", "node_name": "group-9", "containers": []}])
        assert c == E.KS_ERR_INVALID and "group-9" in msg and "stray" in msg
        c, msg = code(o=ds + [{"name": "unbound", "containers": []}])
        assert c == E.KS_ERR_INVALID and "unbound" in msg
        c, msg = code(p=pods + [{"name": "bound", "node_name": "n1", "containers": []}])
        assert c == E.KS_ERR_INVALID and "bound" in msg and "spec.nodeName" in msg
        c, msg = code(t=tmpl[:2] + [{"name": "g", "allocatable": {"cpu": "4"}}])
        assert c == KS_ERR_MISSING and "memory" in msg
        assert code(t=tmpl[:2] + [{"name": "g", "allocatable": {"cpu": "4x", "memory": "1"}}])[0] == KS_ERR_PARSE
        assert code(p=pods + [{"name": "bad", "containers": [{"cpu": "1", "memory": "12Qi"}]}])[0] == KS_ERR_PARSE
        many = [{"name": f"t{i}", "labels": {f"k{i}": "v"}, "allocatable": {"cpu": "1", "memory": "1"}} for i in range(512)]
        sel = [{"name": f"q{i}", "selector": {f"k{i}": "v"}, "containers": []} for i in range(512)]
        c, msg = code(t=many, m=[1] * 512, o=[], p=sel)
        assert c == E.KS_ERR_RANGE and "511" in msg
        assert code(t=many[:511], m=[1] * 511, o=[], p=sel)[0] == E.KS_ERR_NO_DEVICE  # 511 pairs still fit
        assert code(t=[], m=[], o=[], p=[])[0] == E.KS_ERR_NO_DEVICE
        with pytest.raises(ValueError):
            ctx.scaleup_estimate(arena.nodes(tmpl), 3, [1, 2], None, 0)
        assert ctx.export_packed()[0].shape == (0,)  # the context's store is untouched
