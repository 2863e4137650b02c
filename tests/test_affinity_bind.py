"""Inter-pod affinity when binding (ks_affinity_bind), CPU part: the per-term restatement of
tests/affinity_bind_oracle.py against the hand-derived GV-1 queues of tests/golden/gv1_affinity_bind.json; identities
I1 (no terms is ks_spread_bind), I2 (no terms and no spread is ks_gang_bind with singletons), I3 (hostname-style self
anti-affinity is a prefix of ks_place_replicas_spread's copy list) and I4 (anti-affinity is symmetric in its owner)
between the restatements; the C / ctypes / Rust mirrors; and the errors caught without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from affinity_bind_oracle import ANTI, AFFINITY, affinity_bind_packed
from gang_oracle import gang_bind_packed
from helpers import load_golden
from policy_oracle import Oracle
from spread_bind_oracle import spread_bind_packed
from spread_oracle import spread_packed
from test_replicas import random_cluster
from test_spread_bind import _queue, _random_keys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = (0, 1, 3, 4)


def _gv1(ks):
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        ac, am, lab = ctx.export_packed()[:3]
        rc, rm, sel = ctx.pack_pods(arena.pods(g["pods"]), len(g["pods"]))
    return [p["name"] for p in g["pods"]], ac, am, lab, rc, rm, sel


def test_gv1_affinity_bind_golden(ks):
    names, ac, am, lab, rc, rm, sel = _gv1(ks)
    want = load_golden("gv1_affinity_bind.json")
    N = len(ac)
    key_of = {"zone": (want["zone_domain"], want["n_zones"]), "host": (list(range(N)), N)}
    for c in want["cases"]:
        i = [names.index(p) for p in c["pods"]]
        keys = [key_of[k] for k in c["keys"]]
        ex = None if "existing" not in c else [np.array(e) for e in c["existing"]]

        def run(terms, skew):
            fc, fm = ac.copy(), am.copy()
            return affinity_bind_packed(fc, fm, ac, am, lab, rc[i], rm[i], sel[i], c["group"], c["n_groups"], keys,
                                        terms, c.get("existing_pods"), skew, None, ex)

        node, score, refused, counts = run(c["terms"], c.get("max_skew"))
        assert node.tolist() == c["node"] and score.tolist() == c["score"], c["_why"]
        assert refused.tolist() == c["refused"], c["_why"]
        if "spread_only" in c:  # neither constraint alone chooses the node both choose
            assert run([], c["max_skew"])[0].tolist() == c["spread_only"] != c["node"], c["_why"]
            assert run(c["terms"], None)[0].tolist() == c["anti_only"] != c["node"], c["_why"]


def _random_terms(rng, G, K, T):
    return [(int(rng.integers(0, G)), int(rng.integers(0, 2)), int(rng.integers(0, K)),
             sorted(set(rng.integers(0, G, int(rng.integers(0, 3))).tolist()))) for _ in range(T)]


@pytest.mark.parametrize("policy", POLICIES)
def test_no_terms_is_spread_bind(policy):
    """I1: with no terms the nodes, scores, spread refusals, counts and final free[] are ks_spread_bind's; no affinity
    refusal.  Also checks the restatement's spread half against spread_bind_packed on whole queues."""
    rng = np.random.default_rng(0xAF1 + policy)
    for it in range(80):
        fc, fm, ac, am, labels, rc, rm, sel, _ = random_cluster(rng, n_max=12)
        N = len(fc)
        K = int(rng.integers(1, 4))
        keys = _random_keys(rng, N, K)
        G = int(rng.integers(0, 4))
        P = int(rng.integers(1, 25))
        qc, qm, qs, group = _queue(rng, rc, rm, sel, G, P)
        skew = rng.integers(0, 3, (G, K))
        mind = rng.integers(0, 3, (G, K)) if it % 2 else None
        ex = [rng.integers(0, 3, (G, d)) for _, d in keys]
        sfc, sfm = fc.copy(), fm.copy()
        want = spread_bind_packed(sfc, sfm, ac, am, labels, qc, qm, qs, group, keys, skew, mind, ex, policy)
        afc, afm = fc.copy(), fm.copy()
        got = affinity_bind_packed(afc, afm, ac, am, labels, qc, qm, qs, group, G, keys, [], None, skew, mind, ex,
                                   policy)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), it
        assert np.array_equal(got[2][:, 0], want[2]) and not got[2][:, 1].any(), it
        assert all(np.array_equal(a, b) for a, b in zip(got[3], want[3])), it
        assert np.array_equal(afc, sfc) and np.array_equal(afm, sfm), it


@pytest.mark.parametrize("policy", POLICIES)
def test_no_terms_no_spread_is_gang_bind(orc, policy):
    """I2: no terms and max_skew None: ks_gang_bind with one singleton group per pod."""
    rng = np.random.default_rng(0xAF2 + policy)
    for it in range(60):
        fc, fm, ac, am, labels, rc, rm, sel, _ = random_cluster(rng)
        N = len(fc)
        keys = _random_keys(rng, N, int(rng.integers(1, 4)))
        G = int(rng.integers(0, 4))
        P = int(rng.integers(1, 20))
        qc, qm, qs, group = _queue(rng, rc, rm, sel, G, P)
        gfc, gfm = fc.copy(), fm.copy()
        want = gang_bind_packed(Oracle(orc), gfc, gfm, ac, am, labels, qc, qm, qs, np.arange(P + 1, dtype=np.uint64),
                                np.zeros(P, np.uint32), policy)
        afc, afm = fc.copy(), fm.copy()
        got = affinity_bind_packed(afc, afm, ac, am, labels, qc, qm, qs, group, G, keys, policy=policy)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), it
        assert not got[2].any() and np.array_equal(afc, gfc) and np.array_equal(afm, gfm), it


def _replica_prefix(node, score, dom):
    """ks_place_replicas_spread's copy list up to the first copy whose domain already holds one."""
    seen = set()
    for i, n in enumerate(node):
        if n < 0 or dom[n] in seen:
            return node[:i], score[:i]
        seen.add(dom[n])
    return node, score


@pytest.mark.parametrize("policy", POLICIES)
def test_self_anti_affinity_is_the_replica_prefix(policy):
    """I3: one group of R identical pods, anti-affine to itself on a key every node carries, no existing pods: the
    prefix of ks_place_replicas_spread's copy list (max_skew 1) up to the first copy in an occupied domain, then every
    later pod unbound."""
    rng = np.random.default_rng(0xAF3 + policy)
    for it in range(120):
        fc, fm, ac, am, labels, rc, rm, sel, R = random_cluster(rng, t_max=1, r_max=12)
        N, R = len(fc), int(R[0])
        D = int(rng.integers(1, N + 1)) if it % 2 else N
        dom = rng.integers(0, D, N) if it % 2 else np.arange(N)
        keys = [(dom, D)]
        want = spread_packed(fc, fm, ac, am, labels, rc, rm, sel, [R], dom, D, [1], [0], None, policy)
        wn, ws = _replica_prefix(want[1], want[2], dom)
        afc, afm = fc.copy(), fm.copy()
        got = affinity_bind_packed(afc, afm, ac, am, labels, np.repeat(rc, R), np.repeat(rm, R),
                                   np.repeat(sel, R, axis=0), np.zeros(R), 1, keys, [(0, ANTI, 0, [0])], policy=policy)
        assert np.array_equal(got[0][:len(wn)], wn) and np.array_equal(got[1][:len(ws)], ws), it
        assert (got[0][len(wn):] == -1).all(), it


@pytest.mark.parametrize("policy", POLICIES)
def test_anti_affinity_is_symmetric(policy):
    """I4: "g anti h on key k" and "h anti g on key k" bind the same queue the same way, with and without existing pods
    and other terms."""
    rng = np.random.default_rng(0xAF4 + policy)
    for it in range(80):
        fc, fm, ac, am, labels, rc, rm, sel, _ = random_cluster(rng, n_max=12)
        N = len(fc)
        K = int(rng.integers(1, 4))
        keys = _random_keys(rng, N, K)
        G = int(rng.integers(2, 5))
        P = int(rng.integers(1, 25))
        qc, qm, qs, group = _queue(rng, rc, rm, sel, G, P)
        g, h, k = int(rng.integers(0, G)), int(rng.integers(0, G)), int(rng.integers(0, K))
        others = _random_terms(rng, G, K, int(rng.integers(0, 3)))
        ex = (rng.integers(0, G, 3), rng.integers(0, N, 3)) if it % 2 else None
        runs = []
        for term in ((g, ANTI, k, [h]), (h, ANTI, k, [g])):
            f_c, f_m = fc.copy(), fm.copy()
            runs.append(affinity_bind_packed(f_c, f_m, ac, am, labels, qc, qm, qs, group, G, keys, others + [term], ex,
                                             policy=policy) + (f_c, f_m))
        for a, b in zip(runs[0], runs[1]):
            if isinstance(a, list):
                assert all(np.array_equal(x, y) for x, y in zip(a, b)), it
            else:
                assert np.array_equal(a, b), it


def test_affinity_rules_at_each_turn():
    """Random queues with both term kinds: every placed pod of a group with affinity terms lands where each term's key
    holds a pod of M_g (or by the first-pod rule), and no placed pod shares a domain with a pod its anti terms, or the
    anti terms of a bound pod, forbid."""
    rng = np.random.default_rng(0xAF5)
    for it in range(80):
        fc, fm, ac, am, labels, rc, rm, sel, _ = random_cluster(rng, n_max=12)
        N = len(fc)
        K = int(rng.integers(1, 3))
        keys = _random_keys(rng, N, K)
        G = int(rng.integers(1, 4))
        P = int(rng.integers(1, 25))
        qc, qm, qs, group = _queue(rng, rc, rm, sel, G, P)
        terms = _random_terms(rng, G, K, int(rng.integers(1, 4)))
        node, _, refused, _ = affinity_bind_packed(fc.copy(), fm.copy(), ac, am, labels, qc, qm, qs, group, G, keys,
                                                   terms)
        bound = []
        for p in range(P):
            g, n = int(group[p]), int(node[p])
            if n < 0 or g < 0:
                continue
            for o, kind, k, tg in terms:
                d = keys[k][0]
                for h, m in bound:
                    if kind == ANTI and d[n] >= 0 and d[n] == d[m] and ((o == g and h in tg) or (o == h and g in tg)):
                        pytest.fail(f"{it}: pod {p} anti-affinity broken")
            aff = [(k, tg) for o, kind, k, tg in terms if o == g and kind == AFFINITY]
            if aff:
                match = [m for h, m in bound if all(h in tg for _, tg in aff)]
                assert all(keys[k][0][n] >= 0 for k, _ in aff), it
                if any(keys[k][0][m] >= 0 for k, _ in aff for m in match):
                    assert all(any(keys[k][0][m] == keys[k][0][n] for m in match) for k, _ in aff), it
                else:
                    assert all(g in tg for _, tg in aff), it
            bound.append((g, n))


def test_struct_and_constant_mirrors(ks):
    """ks_pod_affinity and ksh_pod_affinity field by field, the constants and KSH_RECONCILE_AFFINITY_UNSATISFIED in the
    headers, the ctypes modules and the Rust shim; both calls declared, exported and bound in Rust."""
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    hhdr = open(os.path.join(ROOT, "include", "ksched_host.h")).read()
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    for name, value in (("KS_POD_AFFINITY", "0"), ("KS_POD_ANTI_AFFINITY", "1"), ("KS_AFFINITY_MAX_TERMS", "16384u"),
                        ("KS_AFFINITY_MAX_TARGETS", r"\(1ull << 22\)"), ("KS_AFFINITY_MAX_EXISTING", r"\(1ull << 24\)"),
                        ("KS_AFFINITY_MAX_UPDATES", r"\(1ull << 24\)")):
        assert re.search(r"#define %s %s\n" % (name, value), hdr), name
    capi = ks.capi
    assert (capi.KS_POD_AFFINITY, capi.KS_POD_ANTI_AFFINITY, capi.KS_AFFINITY_MAX_TERMS) == (0, 1, 16384)
    assert capi.KS_AFFINITY_MAX_TARGETS == 1 << 22 and capi.KS_AFFINITY_MAX_EXISTING == 1 << 24
    assert capi.KS_AFFINITY_MAX_UPDATES == 1 << 24
    assert re.search(r"pub const KS_AFFINITY_MAX_TERMS: u32 = 16384;", rs)
    assert re.search(r"pub const KS_AFFINITY_MAX_TARGETS: u64 = 1 << 22;", rs)
    assert re.search(r"pub const KS_AFFINITY_MAX_EXISTING: u64 = 1 << 24;", rs)
    assert re.search(r"pub const KS_AFFINITY_MAX_UPDATES: u64 = 1 << 24;", rs)
    assert re.search(r"pub const KS_POD_ANTI_AFFINITY: u8 = 1;", rs)
    assert re.search(r"#define KSH_RECONCILE_AFFINITY_UNSATISFIED 6\b", hhdr)
    assert ks.host.KSH_RECONCILE_AFFINITY_UNSATISFIED == 6
    assert re.search(r"pub const KSH_RECONCILE_AFFINITY_UNSATISFIED: c_int = 6;", rs)
    fields = ["n_terms", "owner", "kind", "key", "target_offset", "target", "n_existing", "existing_group"]
    for struct, last, py in (("ks_pod_affinity", "existing_node", capi.ks_pod_affinity),
                             ("ksh_pod_affinity", "existing_node_name", ks.host.ksh_pod_affinity)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), hdr + hhdr, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body)
        assert re.findall(r"(\w+);", body) == fields + [last], struct
        assert [f[0] for f in py._fields_] == fields + [last], struct
        assert C.sizeof(py) == 72, struct  # u32 (+ pad), five pointers, u64, two pointers
        rs_body = re.search(r"pub struct %s \{(.*?)\}" % struct, rs, re.S).group(1)
        assert re.findall(r"pub (\w+):", rs_body) == fields + [last], struct
    for fn in ("ks_affinity_bind", "ksh_reconcile_affinity"):
        assert fn in ks.declared_symbols() and hasattr(ks.lib, fn), fn
        assert re.search(r"pub fn %s\(" % fn, rs), fn
    assert len(ks.lib.ks_affinity_bind.argtypes) == 11 and len(ks.lib.ksh_reconcile_affinity.argtypes) == 18


def test_errors_without_a_device(ks):
    """A NULL snapshot is refused on the host; the object-level call is KS_ERR_RANGE for a key count outside [1, 4],
    KS_ERR_INVALID for a group outside [-1, n_groups) or NULL existing-pod arrays before it needs the device, and
    KS_ERR_NO_DEVICE on a packing-only context."""
    rc_, sel = np.zeros(1, np.int64), np.zeros(1, np.uint64)
    pods = ks.capi.ks_pods(1, rc_.ctypes.data, rc_.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
    grp, dom = np.zeros(1, np.int32), np.zeros(4, np.int32)
    idx = np.empty(1, np.int32)
    sp = ks.capi.ks_spread_multi(1, (C.c_uint32 * 4)(1), (C.c_void_p * 4)(dom.ctypes.data), None, None, None)
    aff = ks.capi.ks_pod_affinity()
    assert ks.lib.ks_affinity_bind(None, C.byref(pods), grp.ctypes.data, 1, C.byref(sp), C.byref(aff), 0,
                                   idx.ctypes.data, None, None, None) == ks.capi.KS_ERR_INVALID
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        p = arena.pods(g["pods"][:2])
        with pytest.raises(ks.KsError) as e:
            ctx.reconcile_affinity(p, 2, [0, -1], 1, ["zone"], [(0, ANTI, 0, [0])], [(0, "n0")])
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
        with pytest.raises(ks.KsError) as e:
            ctx.reconcile_affinity(p, 2, [0, 1], 1, ["zone"])
        assert e.value.code == ks.capi.KS_ERR_INVALID
        keys = (C.c_char_p * 5)(*[b"k"] * 5)
        st, nd = np.empty(2, np.int32), np.empty(2, np.int32)
        for k in (0, 5):
            assert ks.lib.ksh_reconcile_affinity(ctx._h, C.addressof(p), 2, grp.ctypes.data, 0, C.cast(keys, C.c_void_p),
                                                 k, None, None, None, None, None, 0, st.ctypes.data, nd.ctypes.data,
                                                 None, 0, None) == ks.capi.KS_ERR_RANGE
        bad = ks.host.ksh_pod_affinity(0, None, None, None, None, None, 1, None, None)  # E = 1, NULL arrays
        grp2 = np.zeros(2, np.int32)
        assert ks.lib.ksh_reconcile_affinity(ctx._h, C.addressof(p), 2, grp2.ctypes.data, 1, C.cast(keys, C.c_void_p), 1,
                                             None, None, None, None, C.byref(bad), 0, st.ctypes.data, nd.ctypes.data,
                                             None, 0, None) == ks.capi.KS_ERR_INVALID
