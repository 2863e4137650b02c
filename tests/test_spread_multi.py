"""Topology spread over several keys (ks_place_replicas_spread_multi), CPU part: the restatement of
tests/spread_multi_oracle.py against the single-key restatement (K = 1, a key passed twice, a one-domain second key);
the skew bound of every key after every copy; the blocked_domain cases; the hand-derived GV-1 plans of
tests/golden/gv1_spread_multi.json; the C / ctypes / Rust mirrors; and the errors caught without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from helpers import load_golden
from spread_multi_oracle import spread_multi_packed
from spread_oracle import spread_packed
from test_replicas import random_cluster

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = (0, 1, 3, 4)


def _random_key(rng, N, T):
    D = int(rng.integers(1, N + 2))
    dom = rng.integers(0, D, N)
    dom[rng.random(N) < 0.1] = -1
    return dom, D, rng.integers(1, 4, T), rng.integers(0, 4, T), rng.integers(0, 4, (T, D))


@pytest.mark.parametrize("policy", POLICIES)
def test_one_key_twice_and_a_one_domain_key(policy):
    """K = 1 is the single-key plan; the same key twice gives that plan with each row duplicated; a second key with one
    domain on every node changes nothing."""
    rng = np.random.default_rng(0x3C1 + policy)
    for it in range(200):
        fc, fm, ac, am, labels, rc, rm, sel, R = random_cluster(rng)
        N, T = len(fc), len(rc)
        dom, D, skew, mind, ex = _random_key(rng, N, T)
        want = spread_packed(fc, fm, ac, am, labels, rc, rm, sel, R, dom, D, skew, mind, ex, policy)
        got = spread_multi_packed(fc, fm, ac, am, labels, rc, rm, sel, R, [(dom, D)], skew[:, None], mind[:, None],
                                  [ex], policy)
        assert np.array_equal(got[0][:, 0], want[0]), it
        assert all(np.array_equal(a, b) for a, b in zip(got[1:4], want[1:4])), it
        assert np.array_equal(got[4][0], want[4]), it
        twice = spread_multi_packed(fc, fm, ac, am, labels, rc, rm, sel, R, [(dom, D), (dom, D)],
                                    np.stack([skew, skew], 1), np.stack([mind, mind], 1), [ex, ex], policy)
        assert np.array_equal(twice[0][:, 0], want[0]) and np.array_equal(twice[0][:, 1], want[0]), it
        assert all(np.array_equal(a, b) for a, b in zip(twice[1:4], want[1:4])), it
        one = spread_multi_packed(fc, fm, ac, am, labels, rc, rm, sel, R, [(dom, D), (np.zeros(N), 1)],
                                  np.stack([skew, np.ones(T, np.int64)], 1), None, [ex, np.zeros((T, 1))], policy)
        plain = spread_packed(fc, fm, ac, am, labels, rc, rm, sel, R, dom, D, skew, None, ex, policy)
        assert np.array_equal(one[0][:, 0], plain[0]), it
        assert all(np.array_equal(a, b) for a, b in zip(one[1:4], plain[1:4])), it


@pytest.mark.parametrize("policy", POLICIES)
def test_every_key_stays_within_its_skew(policy):
    """No existing pods: after every copy and for every key, max cnt_k - m_k <= max_skew (m_k over E_k)."""
    rng = np.random.default_rng(0x5E7 + policy)
    for it in range(150):
        fc, fm, ac, am, labels, rc, rm, sel, R = random_cluster(rng, r_max=30)
        N, T = len(fc), len(rc)
        keys = [(rng.integers(0, d, N), d) for d in (int(rng.integers(1, 5)), N)]
        skew = rng.integers(1, 3, (T, 2))
        rows, node, _, off, _ = spread_multi_packed(fc, fm, ac, am, labels, rc, rm, sel, R, keys, skew, policy=policy)
        for t in range(T):
            placed = node[int(off[t]):int(off[t + 1])]
            placed = placed[placed >= 0]
            elig = ((sel[t][None, :] & ~labels) == 0).all(axis=1)
            for k, (dom, D) in enumerate(keys):
                e = np.zeros(D, bool)
                e[dom[elig]] = True
                cnt = np.zeros(D, np.int64)
                for n in placed:
                    cnt[dom[n]] += 1
                    assert cnt.max() - cnt[e].min() <= skew[t, k], (it, t, k)


def _flat(N, cpu=4, mem=4):
    v = np.full(N, cpu, np.int64), np.full(N, mem, np.int64)
    return v[0], v[1], v[0], v[1], np.zeros((N, 1), np.uint64)


def test_blocked_domain_cases():
    """Every single-key case of test_spread.test_blocked_domain_cases with a hostname key beside it at an unbounded
    skew, then: zone admits but hostname refuses, a node lacking the second key, minDomains on one key only."""
    fc, fm, ac, am, lab = _flat(6)
    zone = np.array([0, 0, 1, 1, 2, 2])
    host = np.arange(6)

    def plan(R, dom=zone, D=3, skew=1, mind=None, ex=None, sel=0, f=fc, second=(host, 6), skew2=1 << 20, mind2=0,
             ex2=None):
        rows = spread_multi_packed(f, fm, ac, am, lab, [1], [1], np.array([[sel]], np.uint64), [R],
                                   [(dom, D), second], [[skew, skew2]], None if mind is None else [[mind[0], mind2]],
                                   None if ex is None and ex2 is None else
                                   [np.zeros((1, D)) if ex is None else ex,
                                    np.zeros((1, second[1])) if ex2 is None else ex2], 0)[0]
        return rows[0, 0], rows[0, 1]

    r, _ = plan(6)
    assert r["placed"] == 6 and r["blocked_domain"] == -1 and r["min_count"] == 2
    r, _ = plan(3, sel=1)
    assert r["placed"] == 0 and r["eligible_domains"] == 0 and r["blocked_domain"] == -1
    r, h = plan(3, dom=np.full(6, -1))
    assert r["placed"] == 0 and r["eligible_domains"] == 0 and h["eligible_domains"] == 0
    r, _ = plan(9, mind=[4])
    assert r["placed"] == 3 and r["min_count"] == 0 and r["blocked_domain"] == -1
    full = fc.copy()
    full[[2, 3]] = 0
    r, h = plan(9, f=full)
    # hostname's lowest admitted node is n0: it has room, but zone 0 is at max_skew
    assert r["placed"] == 2 and r["min_count"] == 0 and r["blocked_domain"] == 1 and h["blocked_domain"] == 0
    full[[0, 1]] = 0
    r, _ = plan(9, f=full)
    assert r["placed"] == 1 and r["blocked_domain"] == 0
    r, _ = plan(9, mind=[4], f=np.where(zone == 1, 0, fc))
    assert r["placed"] == 2 and r["blocked_domain"] == 1
    r, _ = plan(9, ex=np.array([[5, 0, 0]]))
    assert r["placed"] == 9 and r["blocked_domain"] == -1
    r, _ = plan(0)
    assert r["placed"] == 0 and r["blocked_domain"] == -1 and r["eligible_domains"] == 3
    # zone admits, hostname refuses: node 0 already holds a pod above m + 1 on hostname, so zone 0 has only node 1
    # left; node 1 full stops zone 0 through capacity and hostname together, and zone names it
    f = fc.copy()
    f[1] = 0
    r, h = plan(9, f=f, skew2=1, ex2=np.array([[2, 0, 0, 0, 0, 0]]))
    assert r["placed"] == 2 and r["blocked_domain"] == 0 and h["blocked_domain"] == 1
    # a node lacking the second key is neither counted nor chosen: n0..n4 take one copy each, then n4 (zone 2, whose
    # other node n5 lacks the key) takes the sixth
    r, h = plan(6, second=(np.array([0, 1, 2, 3, 4, -1]), 5), skew2=1)
    assert r["eligible_domains"] == 3 and h["eligible_domains"] == 5 and r["placed"] == 6 and h["min_count"] == 1
    # minDomains on the hostname key only: six eligible nodes < 7 holds its m at 0, one copy per node
    r, h = plan(9, skew=5, skew2=1, mind=[0], mind2=7)
    assert r["placed"] == 6 and h["min_count"] == 0 and r["min_count"] == 2 and h["blocked_domain"] == -1


def test_gv1_spread_multi_golden(ks):
    g = load_golden("gv1.json")
    want = load_golden("gv1_spread_multi.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        ac, am, lab = ctx.export_packed()[:3]
        rc, rm, sel = ctx.pack_pods(arena.pods(g["pods"]), len(g["pods"]))
    names = [p["name"] for p in g["pods"]]
    N = len(g["nodes"])
    keys = [(want["zone_domain"], want["n_zones"]), (list(range(N)), N)]
    for case in want["cases"]:
        i = names.index(case["spec"])
        rows, node, score, off, cnt = spread_multi_packed(ac, am, ac, am, lab, rc[i:i + 1], rm[i:i + 1], sel[i:i + 1],
                                                          [case["replicas"]], keys, [case["max_skew"]],
                                                          [case["min_domains"]], policy=0)
        assert node.tolist() == case["node"] and score.tolist() == case["score"], case["_why"]
        for k, row in enumerate(case["rows"]):
            assert {f: int(rows[f][0, k]) for f in row} == row, case["_why"]
        assert [c[0].tolist() for c in cnt] == case["counts"], case["_why"]
        if "zone_only_node" in case:  # the hostname skew changes the zone-only plan
            zone = spread_packed(ac, am, ac, am, lab, rc[i:i + 1], rm[i:i + 1], sel[i:i + 1], [case["replicas"]],
                                 want["zone_domain"], want["n_zones"], [case["max_skew"][0]], [case["min_domains"][0]])
            assert zone[1].tolist() == case["zone_only_node"] != case["node"], case["_why"]


def test_struct_mirrors(ks):
    """ks_spread_multi: the ctypes struct and the Rust shim list the header's fields; KS_SPREAD_MAX_KEYS everywhere."""
    hdr = open(os.path.join(ROOT, "include", "ksched.h")).read()
    rs = open(os.path.join(ROOT, "examples", "rust_shim", "ksched_sys.rs")).read()
    body = re.search(r"typedef struct ks_spread_multi \{(.*?)\} ks_spread_multi;", hdr, re.S).group(1)
    c_fields = re.findall(r"\b\**([a-z_]+)(?:\[[A-Z_]+\])?;", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert c_fields == [f[0] for f in ks.capi.ks_spread_multi._fields_]
    rbody = re.search(r"pub struct ks_spread_multi \{(.*?)\n\}", rs, re.S).group(1)
    assert re.findall(r"pub ([a-z_0-9]+):", rbody) == c_fields
    assert C.sizeof(ks.capi.ks_spread_multi) == 4 + 4 * 4 + 4 + 8 * 4 + 3 * 8
    assert ks.capi.KS_SPREAD_MAX_KEYS == 4 and "#define KS_SPREAD_MAX_KEYS 4u" in hdr
    assert re.search(r"pub const KS_SPREAD_MAX_KEYS: u32 = 4;", rs)
    for fn in ("ks_place_replicas_spread_multi", "ksh_place_replicas_spread_multi"):
        assert fn in ks.declared_symbols() and hasattr(ks.lib, fn), fn
        assert re.search(r"pub fn %s\(" % fn, rs), fn


def test_errors_without_a_device(ks):
    """A NULL snapshot is refused on the host; the object-level call on a packing-only context is KS_ERR_NO_DEVICE, and
    a key count outside [1, 4] is KS_ERR_RANGE before that."""
    out = (ks.capi.ks_spread_plan * 4)()
    rc_, sel = np.zeros(1, np.int64), np.zeros(1, np.uint64)
    pods = ks.capi.ks_pods(1, rc_.ctypes.data, rc_.ctypes.data, sel.ctypes.data, ks.KS_MEM_HOST)
    rep, skew, dom = np.ones(1, np.uint32), np.ones(2, np.uint32), np.zeros(4, np.int32)
    sp = ks.capi.ks_spread_multi(2, (C.c_uint32 * 4)(1, 1, 0, 0), (C.c_void_p * 4)(dom.ctypes.data, dom.ctypes.data),
                                 skew.ctypes.data, None, None)
    assert ks.lib.ks_place_replicas_spread_multi(None, C.byref(pods), rep.ctypes.data, C.byref(sp), 0, out, None, None,
                                                 None) == ks.capi.KS_ERR_INVALID
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    with ks.host.Context(ks.host.KSH_DEVICE_NONE) as ctx:
        ctx.set_nodes(arena.nodes(g["nodes"]), len(g["nodes"]))
        with pytest.raises(ks.KsError) as e:
            ctx.place_replicas_spread_multi(arena.pods(g["pods"][:2]), 2, [3, 1], ["zone", "host"], np.ones((2, 2)))
        assert e.value.code == ks.capi.KS_ERR_NO_DEVICE
        keys = (C.c_char_p * 5)(*[b"k"] * 5)
        ones = np.ones(10, np.uint32)
        p = arena.pods(g["pods"][:2])
        for k in (0, 5):
            assert ks.lib.ksh_place_replicas_spread_multi(ctx._h, C.addressof(p), 2, ones.ctypes.data, C.cast(keys, C.c_void_p),
                                                          k, ones.ctypes.data, None, None, None, 0, out, None, None,
                                                          None) == ks.capi.KS_ERR_RANGE
