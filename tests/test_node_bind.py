"""Taints and node affinity when binding (ks_node_bind), without a device: hand-derived queues against the string-level
restatement in tests/node_bind_oracle.py, identities K2-K4 on the restatements, the compiled masks and domain sets
against the string evaluation on random label maps, the C / ctypes mirrors, and the errors caught without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from node_bind_oracle import (compile_rules, intolerable_soft, node_bind_packed, preferred_raw, random_cluster,
                              required_ok, untolerated_hard)
from profile_bind_oracle import profile_bind_packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = (1, 3, 4)
CP = {"key": "node-role.kubernetes.io/control-plane", "value": "", "effect": "NoSchedule"}


def flat(N, cpu=8000, mem=32 << 30):
    """N identical empty nodes without label bits: every policy score ties, so the rules alone pick the node."""
    fc = np.full(N, cpu, np.int64)
    fm = np.full(N, mem, np.int64)
    return fc, fm, fc.copy(), fm.copy(), np.zeros((N, 1), np.uint64)


def run(N, node_labels, node_taints, group_rules, group, keys=None, policy=1, **kw):
    fc, fm, ac, am, lab = flat(N)
    P = len(group)
    rc, rm = np.full(P, 1000, np.int64), np.full(P, 1 << 30, np.int64)
    keys = keys or [(np.zeros(N, np.int32), 1)]
    return node_bind_packed(fc, fm, ac, am, lab, rc, rm, np.zeros((P, 1), np.uint64), group, len(group_rules), keys,
                            node_labels, node_taints, group_rules, policy=policy, **kw)


def test_control_plane_taint_then_exists_with_empty_key():
    # node 0 carries the control-plane taint; group 0 tolerates nothing, group 1 tolerates everything by Exists with an
    # empty key.  Pod 0 (group 0): node 0 refused (word 0 = 1), node 1 binds (lower index of the rest).  Pod 1
    # (group 1): both nodes pass; LEAST_ALLOCATED prefers node 0, which pod 0 left empty.
    got = run(2, [{}, {}], [[CP], []], [{}, {"tolerations": [{"key": "", "operator": "Exists"}]}], [0, 1])
    assert got[0].tolist() == [1, 0]
    assert got[3][:, 0].tolist() == [1, 0]


def test_notin_on_a_node_without_the_key_and_gt_against_a_non_integer():
    # NotIn zone {z0}: node 0 (z0) fails, node 1 (no zone) passes -> word 1 = 1, binds node 1.
    # gen Gt 2: node 0 gen "x3" does not parse and never matches, node 1 gen 3 matches -> binds node 1.
    labels = [{"zone": "z0", "gen": "x3"}, {"gen": "3"}]
    notin = {"required": [[{"key": "zone", "operator": "NotIn", "values": ["z0"]}]]}
    gt = {"required": [[{"key": "gen", "operator": "Gt", "values": ["2"]}]]}
    got = run(2, labels, [[], []], [notin, gt], [0, 1])
    assert got[0].tolist() == [1, 1] and got[3][:, 1].tolist() == [1, 1]


def test_an_empty_required_term_matches_nothing():
    got = run(3, [{}] * 3, [[]] * 3, [{"required": [[]]}], [0])
    assert got[0].tolist() == [-1] and got[3][0].tolist() == [0, 3, 0, 0]


def test_prefer_no_schedule_max_zero_and_max_two():
    # max 0: every node tt = 100.  Node taints 2, 1, 0 PreferNoSchedule: max 2, tt = 100 - 100 * raw / 2 = 0, 50, 100;
    # the nodes are equal in every other score, so node 2 wins by 3 * 50 over node 1
    s1 = {"key": "a", "value": "", "effect": "PreferNoSchedule"}
    s2 = {"key": "b", "value": "", "effect": "PreferNoSchedule"}
    got = run(3, [{}] * 3, [[]] * 3, [{}], [0])
    assert got[2][0, 3] == 100
    got = run(3, [{}] * 3, [[s1, s2], [s1], []], [{}], [0])
    assert got[0].tolist() == [2] and got[2][0, 3] == 100
    # tolerating s1 for PreferNoSchedule leaves raw 1, 0, 0: max 1, node 1 wins the tie by index
    got = run(3, [{}] * 3, [[s1, s2], [s1], []], [{"tolerations": [{"key": "a", "operator": "Exists",
                                                                    "effect": "PreferNoSchedule"}]}], [0])
    assert got[0].tolist() == [1] and got[2][0, 3] == 100


def test_preferred_affinity_max_zero():
    # no node matches the preferred term: max 0 -> na = 0 everywhere (DefaultNormalizeScore without reverse)
    g = {"preferred": [(50, [{"key": "zone", "operator": "In", "values": ["z9"]}])]}
    got = run(2, [{"zone": "z0"}, {}], [[], []], [g], [0])
    assert got[0].tolist() == [0] and got[2][0, 4] == 0
    # weights 30 and 70 on nodes 0 and 1: max 70, na = 100 * 30 // 70 = 42 and 100; node 1 wins
    g = {"preferred": [(30, [{"key": "zone", "operator": "In", "values": ["z0"]}]),
                       (70, [{"key": "zone", "operator": "DoesNotExist"}])]}
    got = run(2, [{"zone": "z0"}, {}], [[], []], [g], [0])
    assert got[0].tolist() == [1] and got[2][0, 4] == 100


def test_honor_a_zone_failing_the_affinity_does_not_block():
    # zones z0, z1, z2 of 2 nodes; z2 is being drained (pool NotIn drain fails there).  maxSkew 1 on zone: eligible
    # domains are z0 and z1 only, so 4 pods go 2 and 2.  Counting z2 would pin the minimum at 0 and refuse pods 3-4.
    N = 6
    zone = (np.arange(N) // 2).astype(np.int32)
    labels = [{"zone": f"z{z}", "pool": "drain" if z == 2 else "live"} for z in zone]
    g = {"required": [[{"key": "pool", "operator": "NotIn", "values": ["drain"]}]]}
    got = run(N, labels, [[]] * N, [g], [0] * 4, keys=[(zone, 3)], max_skew=np.ones((1, 1), np.uint32))
    assert (got[0] >= 0).all() and sorted(zone[got[0]].tolist()) == [0, 0, 1, 1]


def _case(rng, N=40, G=3, P=25):
    fc = rng.integers(2000, 9000, N).astype(np.int64)
    fm = rng.integers(4, 32, N).astype(np.int64) << 30
    ac, am = fc + rng.integers(0, 2000, N), fm + (rng.integers(0, 4, N) << 30)
    lab = rng.integers(0, 1 << 8, (N, 1)).astype(np.uint64)
    group = rng.integers(-1, G, P).astype(np.int32)
    rc, rm = rng.integers(0, 3000, P).astype(np.int64), rng.integers(0, 8, P).astype(np.int64) << 30
    gsel = rng.integers(0, 4, (G, 1)).astype(np.uint64)
    sel = np.where(group[:, None] >= 0, gsel[np.maximum(group, 0)], 0).astype(np.uint64)
    keys = [((np.arange(N) % 3).astype(np.int32), 3), (np.arange(N, dtype=np.int32), N)]
    skew = rng.integers(0, 3, (G, 2))
    return fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, skew


@pytest.mark.parametrize("policy", POLICIES)
def test_k2_no_rules_is_profile_bind(policy):
    rng = np.random.default_rng(0x90E0 + policy)
    for it in range(30):
        fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, skew = _case(rng)
        N = len(fc)
        soft = rng.integers(0, 3, (G, 2))
        want = profile_bind_packed(fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, group, G, keys, max_skew=skew,
                                   policy=policy, soft_skew=soft)
        got = node_bind_packed(fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, group, G, keys, [{}] * N, [[]] * N,
                               [{}] * G, max_skew=skew, policy=policy, soft_skew=soft)
        bound = want[0] >= 0
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1] + 300 * bound), it
        assert np.array_equal(got[2][:, :3], want[2]) and np.array_equal(got[3][:, 2:], want[3]), it
        assert not got[3][:, :2].any() and (got[2][bound, 3] == 100).all() and not got[2][:, 4].any(), it
        assert all(np.array_equal(a, b) for a, b in zip(got[4] + got[5], want[4] + want[5])), it


@pytest.mark.parametrize("policy", POLICIES)
def test_k3_required_in_is_a_node_selector(policy):
    """A required term `color In {blue}` binds as a nodeSelector on the label bit that marks the blue nodes."""
    rng = np.random.default_rng(0x90E1 + policy)
    for it in range(30):
        fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, skew = _case(rng)
        N = len(fc)
        blue = rng.random(N) < 0.5
        labels = [{"color": "blue"} if b else ({"color": "red"} if rng.random() < 0.5 else {}) for b in blue]
        lab2 = lab.copy()
        lab2[:, 0] = (lab2[:, 0] & ~np.uint64(1 << 40)) | np.where(blue, np.uint64(1 << 40), np.uint64(0))
        sel2 = sel.copy()
        pinned = rng.random(G) < 0.6
        sel2[(group >= 0) & pinned[np.maximum(group, 0)], 0] |= np.uint64(1 << 40)
        rules = [{"required": [[{"key": "color", "operator": "In", "values": ["blue"]}]]} if pinned[g] else {}
                 for g in range(G)]
        a = node_bind_packed(fc.copy(), fm.copy(), ac, am, lab2, rc, rm, sel, group, G, keys, labels, [[]] * N, rules,
                             max_skew=skew, policy=policy)
        b = node_bind_packed(fc.copy(), fm.copy(), ac, am, lab2, rc, rm, sel2, group, G, keys, labels, [[]] * N,
                             [{}] * G, max_skew=skew, policy=policy)
        assert np.array_equal(a[0], b[0]), it


@pytest.mark.parametrize("policy", POLICIES)
def test_k4_a_taint_everyone_tolerates(policy):
    rng = np.random.default_rng(0x90E2 + policy)
    for it in range(30):
        fc, fm, ac, am, lab, rc, rm, sel, group, G, keys, skew = _case(rng)
        N = len(fc)
        group = np.maximum(group, 0)  # group -1 tolerates nothing: every pod here belongs to a group that tolerates
        sel = np.where(group[:, None] >= 0, sel[np.argmax(group[:, None] == group[None, :], axis=1)], 0).astype(np.uint64)
        taints = [[CP] if rng.random() < 0.5 else [] for _ in range(N)]
        tol = [{"tolerations": [{"key": CP["key"], "operator": "Exists", "effect": "NoSchedule"}]}] * G
        a = node_bind_packed(fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, group, G, keys, [{}] * N, taints, tol,
                             max_skew=skew, policy=policy)
        b = node_bind_packed(fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, group, G, keys, [{}] * N, [[]] * N,
                             [{}] * G, max_skew=skew, policy=policy)
        assert all(np.array_equal(x, y) for x, y in zip(a, b) if isinstance(x, np.ndarray)), it


def test_compiled_rules_against_the_strings():
    """The masks and sets compile_rules makes (the form Snapshot.node_bind takes) evaluated per (group, node) equal the
    string evaluation: untolerated hard taint, PreferNoSchedule count, required affinity and preferred raw."""
    rng = np.random.default_rng(0x90E3)
    for it in range(8):
        N, G = 200, 6
        labels, taints, rules = random_cluster(rng, N, G, int(rng.choice([0, 1, 3, 64])))
        r = compile_rules(labels, taints, rules)
        doms = r["rule_keys"]
        for g in range(G):
            terms = [t for t in r["node_terms"] if t[0] == g]

            def match(t, n):
                if not t[2]:
                    return False
                for k, words in t[2]:
                    d, D = int(doms[k][0][n]), doms[k][1]
                    b = D if d < 0 else d
                    if not int(words[b // 64]) >> (b % 64) & 1:
                        return False
                return True
            req = [t for t in terms if t[1] == 0]
            for n in range(N):
                tols = rules[g].get("tolerations", ())
                hard = int(r["taint_hard"][n]) & ~int(r["tolerate_hard"][g])
                assert bool(hard) == untolerated_hard(taints[n], tols), (it, g, n)
                soft = bin(int(r["taint_soft"][n]) & ~int(r["tolerate_soft"][g])).count("1")
                assert soft == intolerable_soft(taints[n], tols), (it, g, n)
                assert (not req or any(match(t, n) for t in req)) == required_ok(rules[g], labels[n]), (it, g, n)
                assert sum(t[1] for t in terms if t[1] and match(t, n)) == preferred_raw(rules[g], labels[n])


def test_struct_and_constant_mirrors(ks):
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    for name, v in (("KS_NODE_RULES_MAX_TAINTS", 64), ("KS_NODE_RULES_MAX_KEYS", 16),
                    ("KS_NODE_RULES_MAX_PREFERRED", 4096)):
        assert re.search(r"#define %s %du\b" % (name, v), hdr) and getattr(ks.capi, name) == v, name
    assert re.search(r"#define KS_NODE_RULES_MAX_WORDS \(1ull << 26\)", hdr)
    assert ks.capi.KS_NODE_RULES_MAX_WORDS == 1 << 26
    body = re.search(r"typedef struct ks_node_rules \{(.*?)\} ks_node_rules;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body)
    fields = re.findall(r"(\w+)(?:\[\w+\])?;", body)
    assert [f[0] for f in ks.capi.ks_node_rules._fields_] == fields
    # u32 + pad, 4 pointers, u32 + 16 u32 + pad, 16 pointers, u32 + pad, 3 pointers, u32 + pad, 3 pointers, 2 u32
    assert C.sizeof(ks.capi.ks_node_rules) == 312
    assert ks.capi.ks_node_rules.node_domain.offset == 112 and ks.capi.ks_node_rules.weight_taint.offset == 304
    assert "ks_node_bind" in ks.declared_symbols() and hasattr(ks.lib, "ks_node_bind")
    assert len(ks.lib.ks_node_bind.argtypes) == 15


def test_errors_without_a_device(ks):
    """A NULL scoring is refused before the snapshot is looked at; a NULL snapshot with a valid scoring is refused."""
    rc_, sel = np.zeros(1, np.int64), np.zeros(1, np.uint64)
    pods = ks.capi.ks_pods(1, rc_.ctypes.data, rc_.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
    grp, dom = np.zeros(1, np.int32), np.zeros(4, np.int32)
    idx = np.empty(1, np.int32)
    sp = ks.capi.ks_spread_multi(1, (C.c_uint32 * 4)(1), (C.c_void_p * 4)(dom.ctypes.data), None, None, None)
    aff = ks.capi.ks_pod_affinity()
    sc = ks.capi.ks_bind_scoring(None, None, None, 1, 2, 2)
    nr = ks.capi.ks_node_rules()
    assert ks.lib.ks_node_bind(None, C.byref(pods), grp.ctypes.data, 1, C.byref(sp), C.byref(aff), None, C.byref(nr),
                               4, idx.ctypes.data, None, None, None, None, None) == ks.capi.KS_ERR_INVALID
    assert "NULL scoring" in ks.lib.ks_last_error().decode()
    for rules in (None, C.byref(nr)):
        assert ks.lib.ks_node_bind(None, C.byref(pods), grp.ctypes.data, 1, C.byref(sp), C.byref(aff), C.byref(sc),
                                   rules, 4, idx.ctypes.data, None, None, None, None, None) == ks.capi.KS_ERR_INVALID
        assert "NULL scoring" not in ks.lib.ks_last_error().decode()


def test_rust_shim_mirror():
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    body = re.sub(r"/\*.*?\*/", "", re.search(r"typedef struct ks_node_rules \{(.*?)\} ks_node_rules;", hdr, re.S).group(1))
    fields = re.findall(r"(\w+)(?:\[\w+\])?;", body)
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    rs_body = re.search(r"pub struct ks_node_rules \{(.*?)\}", rs, re.S).group(1)
    assert re.findall(r"pub (\w+):", rs_body) == fields
    assert re.search(r"pub fn ks_node_bind\(", rs)
    assert re.search(r"pub const KS_NODE_RULES_MAX_KEYS: usize = 16;", rs)
