"""Taints and node affinity over objects, without a device (ksh_context_set_node_taints, ksh_compile_node_rules,
ksh_reconcile_nodes): the host's compilation of tolerations and requirement operators evaluated per (group, node)
against the string restatement in tests/node_bind_oracle.py on random label maps (hostname keys of more than 64
domains included), taint bookkeeping across upsert, remove and set_nodes, the requirements API validation rejects, the
C / ctypes / Rust mirrors, and KS_ERR_NO_DEVICE on a packing-only context."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from node_bind_oracle import intolerable_soft, preferred_raw, random_cluster, required_ok, untolerated_hard

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CP = {"key": "node-role.kubernetes.io/control-plane", "value": "", "effect": "NoSchedule"}
ALLOC = {"cpu": "8", "memory": "34359738368"}


def _ctx(ks, labels, taints=None):
    arena = ks.objects.ObjectArena()
    ctx = ks.host.Context(ks.host.KSH_DEVICE_NONE)
    objs = [{"name": f"n{i}", "labels": lab, "allocatable": ALLOC} for i, lab in enumerate(labels)]
    ctx.set_nodes(arena.nodes(objs), len(objs))
    if taints is not None:
        ctx.set_node_taints({f"n{i}": ts for i, ts in enumerate(taints)})
    return ctx, arena


def _want(labels, taints, rules):
    G, N = len(rules), len(labels)
    want = (np.zeros((G, N), np.uint8), np.zeros((G, N), np.uint8), np.zeros((G, N), np.uint32),
            np.zeros((G, N), np.uint32))
    for g, r in enumerate(rules):
        tols = r.get("tolerations", ())
        for n in range(N):
            want[0][g, n] = untolerated_hard(taints[n], tols)
            want[1][g, n] = required_ok(r, labels[n])
            want[2][g, n] = intolerable_soft(taints[n], tols)
            want[3][g, n] = preferred_raw(r, labels[n])
    return want


def test_compilation_against_the_strings(ks):
    rng = np.random.default_rng(0x90F0)
    for it in range(6):
        N, G = 150, 6
        labels, taints, rules = random_cluster(rng, N, G, int(rng.choice([0, 1, 3, 64])))
        for n, lab in enumerate(labels):  # a hostname key of more than 64 domains, one node without it
            if n != 100:
                lab["host"] = f"h{n}"
            lab["num"] = ["+3", "-2", "007", "1e3", " 4", "9223372036854775808", "5"][n % 7]
        rules[0].setdefault("required", []).append([{"key": "host", "operator": "NotIn", "values": ["h3", "h140"]}])
        rules[1]["required"] = [[{"key": "host", "operator": "In", "values": ["h70", "h130", "h7"]}],
                                [{"key": "host", "operator": "DoesNotExist"}]]
        rules[2]["preferred"] = [(40, [{"key": "num", "operator": "Gt", "values": ["2"]}]),
                                 (60, [{"key": "num", "operator": "Lt", "values": ["-1"]}])]
        rules[3]["required"] = [[{"key": "num", "operator": "Lt", "values": ["+8"]}]]
        ctx, _ = _ctx(ks, labels, taints)
        with ctx:
            got = ctx.compile_node_rules(rules)
        want = _want(labels, taints, rules)
        for i in range(4):
            assert np.array_equal(got[i], want[i]), (it, i, np.argwhere(got[i] != want[i])[:5])
        assert want[1][1, 100] and want[1][1, 70] and not want[1][1, 71]  # the absent bit in the set's third word


def test_taints_follow_the_node_name(ks):
    """Kept by name: they survive an upsert of that name, go with remove_node, are cleared by set_nodes; unknown names
    are ignored."""
    labels = [{}] * 4
    ctx, arena = _ctx(ks, labels)
    with ctx:
        ctx.set_node_taints({"n1": [CP], "n3": [CP], "nope": [CP]})
        assert ctx.compile_node_rules([{}])[0].tolist() == [[0, 1, 0, 1]]
        ctx.upsert_node(arena.nodes([{"name": "n1", "labels": {"x": "y"}, "allocatable": ALLOC}]))
        assert ctx.compile_node_rules([{}])[0].tolist() == [[0, 1, 0, 1]]
        ctx.remove_node("n1")
        assert ctx.compile_node_rules([{}])[0].tolist() == [[0, 0, 1]]
        ctx.upsert_node(arena.nodes([{"name": "n1", "labels": {}, "allocatable": ALLOC}]))  # back, without taints
        assert ctx.compile_node_rules([{}])[0].tolist() == [[0, 0, 1, 0]]
        ctx.set_node_taints({"n3": []})
        assert not ctx.compile_node_rules([{}])[0].any()
        ctx.set_node_taints({"n0": [CP]})
        objs = [{"name": f"n{i}", "labels": {}, "allocatable": ALLOC} for i in range(4)]
        ctx.set_nodes(arena.nodes(objs), 4)
        assert not ctx.compile_node_rules([{}])[0].any()
        # tolerated by Exists with an empty key; a PreferNoSchedule toleration does not tolerate a NoSchedule taint
        ctx.set_node_taints({"n0": [CP]})
        rules = [{"tolerations": [{"key": "", "operator": "Exists"}]},
                 {"tolerations": [{"key": CP["key"], "operator": "Exists", "effect": "PreferNoSchedule"}]}]
        assert ctx.compile_node_rules(rules)[0][:, 0].tolist() == [0, 1]


@pytest.mark.parametrize("req", [
    {"key": "a", "operator": "Near", "values": ["x"]},
    {"key": "a", "operator": "In", "values": []},
    {"key": "a", "operator": "NotIn", "values": []},
    {"key": "a", "operator": "Gt", "values": []},
    {"key": "a", "operator": "Gt", "values": ["1", "2"]},
    {"key": "a", "operator": "Lt", "values": ["x1"]},
    {"key": "a", "operator": "Exists", "values": ["x"]},
    {"key": "a", "operator": "DoesNotExist", "values": ["x"]},
    {"key": "", "operator": "Exists"},
], ids=lambda q: f"{q['operator']}-{len(q.get('values', ()))}-{q['key'] or 'nokey'}")
def test_requirements_api_validation_rejects(ks, req):
    ctx, _ = _ctx(ks, [{"a": "1"}])
    with ctx:
        with pytest.raises(ks.KsError) as e:
            ctx.compile_node_rules([{"required": [[req]]}])
        assert e.value.code == ks.capi.KS_ERR_INVALID


def test_other_rejections(ks):
    ctx, _ = _ctx(ks, [{"a": "1"}] * 3)
    with ctx:
        for tol in ({"key": "a", "operator": "Gte"}, {"key": "a", "operator": "Exists", "value": "v"}):
            with pytest.raises(ks.KsError) as e:
                ctx.compile_node_rules([{"tolerations": [tol]}])
            assert e.value.code == ks.capi.KS_ERR_INVALID
        for bad in ({"key": "", "value": "", "effect": "NoSchedule"}, {"key": "k", "value": "", "effect": "Never"}):
            with pytest.raises(ks.KsError) as e:
                ctx.set_node_taints({"n0": [bad]})
            assert e.value.code == ks.capi.KS_ERR_INVALID
        ctx.set_node_taints({f"n{i}": [{"key": f"t{i}-{j}", "value": "", "effect": "NoSchedule"} for j in range(30)]
                             for i in range(3)})  # 90 distinct taints
        with pytest.raises(ks.KsError) as e:
            ctx.compile_node_rules([{}])
        assert e.value.code == ks.capi.KS_ERR_RANGE
        ctx.set_node_taints({f"n{i}": [] for i in range(3)})
        many = [[{"key": f"k{i}", "operator": "Exists"}] for i in range(17)]
        with pytest.raises(ks.KsError) as e:
            ctx.compile_node_rules([{"required": many}])
        assert e.value.code == ks.capi.KS_ERR_RANGE
        ctx.compile_node_rules([{"required": many[:16]}])  # 16 keys: at the cap


def test_reconcile_nodes_needs_a_device(ks):
    ctx, arena = _ctx(ks, [{"a": "1"}])
    with ctx:
        with pytest.raises(ks.KsError) as e:
            ctx.reconcile_nodes(arena.pods([{"name": "p0", "containers": []}]), 1, [0], 1, ["a"],
                                group_rules=[{}])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE


def test_host_mirrors(ks):
    hdr = open(os.path.join(ROOT, "include", "ksched_host.h")).read()
    assert re.search(r"#define KSH_RECONCILE_NODE_RULES_UNSATISFIED 7\b", hdr)
    assert ks.host.KSH_RECONCILE_NODE_RULES_UNSATISFIED == 7
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    assert re.search(r"pub const KSH_RECONCILE_NODE_RULES_UNSATISFIED: c_int = 7;", rs)
    for name in ("ksh_taint", "ksh_toleration", "ksh_node_selector_requirement", "ksh_node_rules"):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), hdr, re.S).group(1)
        fields = re.findall(r"(\w+);", re.sub(r"/\*.*?\*/", "", body))
        assert [f[0] for f in getattr(ks.host, name)._fields_] == fields, name
        rs_body = re.search(r"pub struct %s \{(.*?)\}" % name, rs, re.S).group(1)
        assert re.findall(r"pub (\w+):", rs_body) == fields, name
    assert C.sizeof(ks.host.ksh_node_rules) == 64  # 2 pointers, u32 + pad, 4 pointers, 2 u32
    for fn, n_args in (("ksh_context_set_node_taints", 5), ("ksh_compile_node_rules", 7), ("ksh_reconcile_nodes", 20)):
        assert hasattr(ks.lib, fn) and len(getattr(ks.lib, fn).argtypes) == n_args, fn
        assert re.search(r"pub fn %s\(" % fn, rs), fn
