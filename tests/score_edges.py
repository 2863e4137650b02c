"""Score parts of the bind calls at their edges: the cases of test_score_edges.py (CPU) and test_score_edges_gpu.py (H100),
the searches that find their hazard values, and mutants of the oracle arithmetic that each case must tell apart.

ks_profile_bind, ks_node_bind, ks_fit_bind and ks_gang_fit_bind pick a pod's node by a total of normalised parts
(include/ksched.h): PodTopologySpread pts from a GoRound-ed double sum, InterPodAffinity ipa from one double division,
TaintToleration tt and NodeAffinity na from integer divisions.  A kernel that rounds, divides or converts differently
agrees with the oracle almost everywhere; the cases here put a candidate where it does not.

A case is one queue on identical nodes whose pods request nothing, so the policy score is one constant over the nodes
and the parts alone pick the winner: the pod binds on a node whose part sits on a hazard, or where two decompositions of
the total tie.  Mutants are source patches of the oracle functions, live only inside `mutant(name)`; a case lists the
mutants it kills, and test_score_edges.py checks each claim on the CPU.

Regenerate the search fixture (about a minute) with `python tests/score_edges.py --regenerate`."""
import json
import math
import os
import sys
from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

import fit_bind_oracle
import node_bind_oracle
import oracle_mutants
import profile_bind_oracle
from affinity_bind_oracle import AFFINITY
from bind_edges import bind_slices, resource_maps
from fit_bind_oracle import final_free
from profile_bind_oracle import ANTI_PREFERRED, PREFERRED

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "score_edges.json")
MAX_EXISTING = 1 << 24              # KS_SPREAD_MAX_EXISTING
SEARCH_SC = MAX_EXISTING + 65_536   # soft counts an existing count plus a full queue can reach
SEARCH_SIZES = range(1, 257)
SHARED_BITMAP = 64 * 32             # PB_SH_WORDS * 32: domains below it are marked in the CTA's shared bitmap
ALLOC_C, ALLOC_M = 4000, 16 << 30   # every node; pods request 0, so the policy score is one constant

# ------------------------------------------------------------------------------------------------------------ mutants
_PACKED = (("profile_bind_oracle", "profile_bind_packed"), ("node_bind_oracle", "node_bind_packed"),
           ("fit_bind_oracle", "fit_bind_packed"))
_IPA = "ipa = int(100.0 * (float(int(iraw[n]) - lo) / float(hi - lo))) if hi > lo else 0"
_TERM = "score += float(sc[k][g][dom[k][n]]) * weight[k] + float(soft_skew[g][k] - 1)"
_PTS = (("profile_bind_oracle", "pts_scores"),)
_NORM = (("node_bind_oracle", "normalize"),)

# name -> (what a kernel would get wrong, the functions patched, [(oracle text, mutant text)])
MUTANTS = {
    "half-even": ("GoRound replaced by round-half-to-even (rint)", (("profile_bind_oracle", "go_round"),),
                  [("r = f + 1 if a - f >= 0.5 else f", "r = f + 1 if a - f > 0.5 or (a - f == 0.5 and f % 2) else f")]),
    "exact-raw": ("the PTS raw summed exactly and rounded once", _PTS,
                  [("score = 0.0", "score = Fraction(0)"),
                   (_TERM, "score += Fraction(int(sc[k][g][dom[k][n]])) * Fraction(weight[k]) + int(soft_skew[g][k] - 1)")]),
    "integer-ipa": ("ipa as (100 * (raw - min)) // (max - min) in integers", _PACKED,
                    [(_IPA, "ipa = 100 * (int(iraw[n]) - lo) // (hi - lo) if hi > lo else 0")]),
    "float32-counts": ("soft (and existing) counts read through float32", _PTS,
                       [("float(sc[k][g][dom[k][n]])", "float(np.float32(sc[k][g][dom[k][n]]))")]),
    "int32-skew": ("soft_skew read as int32, then minus 1", _PTS,
                   [("float(soft_skew[g][k] - 1)", "float((int(soft_skew[g][k]) + 2**31) % 2**32 - 2**31 - 1)")]),
    "no-empty-domain": ("size_k without the +1 for the empty value under soft_all_keys = 0", _PTS,
                        [("values[k].add(int(dom[k][n]))", "values[k].update([int(dom[k][n])] if dom[k][n] >= 0 else [])")]),
    "shared-bitmap-only": ("size_k without the domains at or above PB_SH_WORDS * 32 = 2048 (the global bitmap's)", _PTS,
                           [("values[k].add(int(dom[k][n]))",
                             "values[k].update([int(dom[k][n])] if dom[k][n] < SHARED_BITMAP else [])")]),
    "global-bitmap-only": ("size_k without the domains below 2048 (the CTA's shared bitmap's)", _PTS,
                           [("values[k].add(int(dom[k][n]))",
                             "values[k].update([int(dom[k][n])] if not 0 <= dom[k][n] < SHARED_BITMAP else [])")]),
    "logw-shifted": ("w_k read one entry off in the log table: log(size + 3)", _PTS,
                     [("math.log(float(len(values[k]) + 2))", "math.log(float(len(values[k]) + 3))")]),
    "ignored-domains": ("size_k counting the domains of ignored nodes", _PTS,
                        [("ignored.add(n)", "ignored.add(n); [values[k].add(int(dom[k][n])) for k in sigma if dom[k][n] >= 0]")]),
    "rounded-normalize": ("tt and na rounded instead of truncated", _NORM,
                          [("100 - 100 * v // mx if reverse else 100 * v // mx",
                            "100 - round(100 * v / mx) if reverse else round(100 * v / mx)")]),
    "complement-tt": ("tt as 100 * (max - t) / max, one truncation of the complement", _NORM,
                      [("100 - 100 * v // mx if reverse", "100 * (mx - v) // mx if reverse")]),
    "ties-high": ("ties in the total to the higher index", _PACKED,
                  [("if best is None or total > best[0]:", "if best is None or total >= best[0]:")]),
}

# Mistakes no reachable input tells apart from the header's arithmetic: the case list runs them and none may be killed.
NEUTRAL = {
    "float32-existing": ("existing counts read through float32 when the counters are loaded; every existing count is at "
                         "most KS_SPREAD_MAX_EXISTING = 2^24, which float32 holds exactly (counts above it arise only "
                         "from bindings, which float32-counts covers)",
                         _PACKED, [("np.asarray(existing[k], np.int64)", "np.asarray(existing[k], np.float32).astype(np.int64)")]),
    "uint32-skew": ("soft_skew - 1 in uint32 arithmetic, as the kernel computes it: a key scores only with soft_skew >= 1, "
                    "so the difference never wraps", _PTS,
                    [("float(soft_skew[g][k] - 1)", "float((int(soft_skew[g][k]) - 1) % 2**32)")]),
}


def mutant(name):
    """The oracle with one mutant's patches applied; restored on exit"""
    return oracle_mutants.mutant({**MUTANTS, **NEUTRAL}, name, Fraction=Fraction, np=np, SHARED_BITMAP=SHARED_BITMAP)


# ----------------------------------------------------------------------------------------------------------- searches
def search_exact_halves(sizes=SEARCH_SIZES, limit=SEARCH_SC):
    """Every (size, sc) with sc < limit whose double product sc * log(size + 2) is exactly k + 0.5: [size, sc, k,
    exact product below the half]"""
    sc = np.arange(limit, dtype=np.float64)
    out = []
    for size in sizes:
        w = math.log(size + 2)
        p = sc * w
        for i in np.flatnonzero(p - np.floor(p) == 0.5):
            k = int(math.floor(p[i]))
            out.append([size, int(i), k, Fraction(int(i)) * Fraction(w) < Fraction(2 * k + 1, 2)])
    return out


def search_truncating(b_max=200):
    """Every (a, b), 0 <= a <= b <= b_max, where (int64)(100.0 * (a / b)) differs from (100 * a) // b"""
    return [[a, b] for b in range(1, b_max + 1) for a in range(b + 1) if int(100.0 * (a / b)) != (100 * a) // b]


def truncating_at(b):
    """The smallest a with a truncating pair (a, b)"""
    return next(a for a in range(b + 1) if int(100.0 * (a / b)) != (100 * a) // b)


def regenerate():
    data = {"exact_halves": search_exact_halves(), "truncating": search_truncating(),
            "truncating_20000": [truncating_at(20_000), 20_000]}
    with open(GOLDEN, "w") as f:
        json.dump(data, f, indent=1)
        f.write("\n")


def fixture():
    with open(GOLDEN) as f:
        return json.load(f)


# -------------------------------------------------------------------------------------------------------------- cases
@dataclass
class Case:
    """One queue: N identical nodes with `lab` labels, pods (rc, rm, sel, group) over G groups and keys; kw are the
    oracle keywords (terms, existing_pods, existing, soft_skew, soft_all_keys, term_weight, hard_affinity_weight and the
    plugin weights), cluster the node labels, taints and group rules of ks_node_bind, gangs (offset, min_member) for
    ks_gang_fit_bind.  kills: the mutants the case tells apart; expect: (pod, parts word, value) the oracle must give."""
    name: str
    N: int
    group: np.ndarray
    G: int
    keys: list
    kw: dict = field(default_factory=dict)
    calls: tuple = ("profile", "node", "fit")
    cluster: tuple = None
    lab: np.ndarray = None
    sel: np.ndarray = None
    rc: np.ndarray = None
    kills: tuple = ()
    expect: tuple = ()
    gangs: tuple = None

    @property
    def P(self):
        return len(self.group)

    def nodes(self):
        """(ac, am, lab, fc, fm), fresh copies"""
        ac, am = np.full(self.N, ALLOC_C, np.int64), np.full(self.N, ALLOC_M, np.int64)
        lab = np.zeros((self.N, 1), np.uint64) if self.lab is None else self.lab
        return ac, am, lab, ac.copy(), am.copy()

    def queue(self):
        """(rc, rm, sel, group)"""
        W = 1 if self.lab is None else self.lab.shape[1]
        rc = np.zeros(self.P, np.int64) if self.rc is None else self.rc
        sel = np.zeros((self.P, W), np.uint64) if self.sel is None else self.sel
        return rc, np.zeros(self.P, np.int64), sel, self.group.astype(np.int32)

    def rules_cluster(self):
        if self.cluster is not None:
            return self.cluster
        return [{}] * self.N, [[]] * self.N, [{}] * self.G

    def res(self):
        """fit_bind_oracle's name maps: 1,000 pod slots per node, one per pod"""
        return resource_maps(np.full((1, self.N), 1000, np.int64), np.ones((self.P, 1), np.int64))


def oracle(case, call, policy):
    """The oracle's 7-tuple (node, score, parts, refused, counts, soft counts, free_r or None) and free_cpu, free_mem
    after the call; under `mutant` the patched functions run"""
    ac, am, lab, fc, fm = case.nodes()
    rc, rm, sel, group = case.queue()
    kw = dict(case.kw, policy=policy)
    if call == "profile":
        for k in ("weight_taint", "weight_node_affinity"):
            kw.pop(k, None)
        out = profile_bind_oracle.profile_bind_packed(fc, fm, ac, am, lab, rc, rm, sel, group, case.G, case.keys, **kw)
        return out + (None,), fc, fm
    nl, nt, gr = case.rules_cluster()
    if call == "node":
        out = node_bind_oracle.node_bind_packed(fc, fm, ac, am, lab, rc, rm, sel, group, case.G, case.keys, nl, nt, gr,
                                                **kw)
        return out + (None,), fc, fm
    alloc, bound, pod_res = case.res()
    if call == "fit":
        out = fit_bind_oracle.fit_bind_packed(fc, fm, ac, am, lab, rc, rm, sel, group, case.G, case.keys, nl, nt, gr,
                                              alloc, bound, pod_res, **kw)
        return out[:6] + (final_free(alloc, out[6], ["pods"]),), fc, fm
    import gang_fit_bind_oracle
    out = gang_fit_bind_oracle.gang_fit_bind_packed(fc, fm, ac, am, lab, rc, rm, sel, group, case.G, case.keys, nl, nt,
                                                    gr, alloc, bound, pod_res, *case.gangs, **kw)
    return out[:6] + (final_free(alloc, out[6], ["pods"]), out[7]), fc, fm


def device_args(case):
    """Snapshot keywords of the case: the oracle keywords renamed, rules compiled, resources as arrays"""
    kw = dict(case.kw)
    dev = dict(terms=kw.pop("terms", ()), existing_pods=kw.pop("existing_pods", None),
               existing=kw.pop("existing", None))
    wt, wn = kw.pop("weight_taint", 3), kw.pop("weight_node_affinity", 2)
    dev.update(kw)
    return dev, (wt, wn)


def outputs(out):
    """node, score and parts of an oracle result, for telling a mutant apart"""
    return out[0], out[1], out[2]


def differs(a, b):
    return any(not np.array_equal(x, y) for x, y in zip(outputs(a), outputs(b)))


def kills(case, name, calls=None, policies=(1, 3, 4)):
    """Whether mutant `name` changes the node, score or parts of some call and policy of the case"""
    for call in calls or case.calls:
        for policy in policies:
            want = oracle(case, call, policy)[0]
            with mutant(name):
                got = oracle(case, call, policy)[0]
            if differs(got, want):
                return True
    return False


# ---------------------------------------------------------------- helpers shared by the constructors
def _soft_existing(G, keys, entries):
    """existing counts [G, D_k] per key with entries {(g, k, d): count}"""
    ex = [np.zeros((G, D), np.uint32) for _, D in keys]
    for (g, k, d), c in entries.items():
        ex[k][g, d] = c
    return ex


def _pods_on(nodes_counts, g):
    """existing_pods (groups, nodes) with `c` pods of group g on node n for each (n, c)"""
    nodes = np.concatenate([np.full(c, n, np.int32) for n, c in nodes_counts]) if nodes_counts else np.zeros(0, np.int32)
    return np.full(len(nodes), g, np.int32), nodes


def _merge_pods(*ps):
    return np.concatenate([p[0] for p in ps]).astype(np.int32), np.concatenate([p[1] for p in ps]).astype(np.int32)


def _pts_raw(sc, w, c):
    """GoRound(sc * w + c) in double, as the header defines one key's raw"""
    return profile_bind_oracle.go_round(float(sc) * w + float(c))


# ---------------------------------------------------------------------------------------- PodTopologySpread cases
def half_case(size, sc, k, below):
    """An exact-half raw reached through an existing soft count: `size` nodes, one zone each (key 0, soft skew k + 1, so
    every raw carries the constant k), node 0's zone at soft count sc with sc * log(size + 2) = k + 0.5 exactly, the
    others at 0.  Node 0's raw is GoRound(2k + 0.5) = 2k + 1 and the maximum, the others' k the minimum, so node 0 has
    pts = 100 k / (2k + 1) = 49; a raw of 2k (an even floor under half-to-even, or the exact product below the half)
    gives 50.  A weight-1 preferred term towards an existing pod of group 1 on node 0 (hostname key 1) lifts node 0's
    ipa to 100, so the pods bind there and show pts in their parts."""
    N, G = size, 2
    keys = [(np.arange(N, dtype=np.int32), size), (np.arange(N, dtype=np.int32), N)]
    soft = np.zeros((G, 2), np.uint32)
    soft[0, 0] = k + 1
    kw = dict(soft_skew=soft, existing=_soft_existing(G, keys, {(0, 0, 0): sc}), existing_pods=_pods_on([(0, 1)], 1),
              terms=[(0, PREFERRED, 1, [1])], term_weight=[1])
    kills = ("half-even",) + (("exact-raw",) if below else ())
    return Case(f"half size={size} sc={sc}", N, np.zeros(2, np.int32), G, keys, kw, kills=kills,
                expect=((0, 1, 49),))


def _boosted_soft_case(name, N, keys, soft, entries, winner, soft_all=None, G=2, P=2):
    """A soft-spread queue of group 0 whose pods an IPA lift (a weight-1 preferred term towards a pod of group G - 1 on
    `winner`, over the last key, a hostname key) sends to `winner`"""
    kw = dict(soft_skew=soft, existing=_soft_existing(G, keys, entries), existing_pods=_pods_on([(winner, 1)], G - 1),
              terms=[(0, PREFERRED, len(keys) - 1, [G - 1])], term_weight=[1])
    if soft_all is not None:
        kw["soft_all_keys"] = np.asarray(soft_all, np.uint8)
    return Case(name, N, np.zeros(P, np.int32), G, keys, kw)


def cross_case():
    """A soft count that crosses 2^24 during the queue: two zones (w = log 4), zone 0 at 2^24 - 1, and four pods that all
    bind in it (the IPA lift), so the raws are read at 2^24 - 1, 2^24, 2^24 + 1 and 2^24 + 2.  The constant c is
    GoRound(2^24 * w): at 2^24 + 1, which float32 rounds to 2^24, the float32 raw is 2c and gives pts 50, the true raw
    is above it and gives 49."""
    w = math.log(4)
    c = _pts_raw(MAX_EXISTING, w, 0)
    keys = [(np.array([0, 1], np.int32), 2), (np.arange(2, dtype=np.int32), 2)]
    soft = np.zeros((2, 2), np.uint32)
    soft[0, 0] = c + 1
    case = _boosted_soft_case("count crosses 2^24", 2, keys, soft, {(0, 0, 0): MAX_EXISTING - 1}, 0, P=4)
    case.kills, case.expect = ("float32-counts",), ((2, 1, 49),)
    return case


def skew_case(s):
    """soft_skew = s (2^31 or 2^32 - 1) on a zone key of three zones at soft counts 5, 0, 0, the pods lifted to zone 0:
    every raw carries s - 1; read as int32 the constant turns negative and the normalisation changes"""
    keys = [(np.arange(3, dtype=np.int32), 3), (np.arange(3, dtype=np.int32), 3)]
    soft = np.zeros((2, 2), np.uint32)
    soft[0, 0] = s
    case = _boosted_soft_case(f"soft_skew={s}", 3, keys, soft, {(0, 0, 0): 5}, 0)
    case.kills = ("int32-skew",)
    return case


def empty_value_case():
    """soft_all_keys = 0 and a node without the zone key: size = 2 zones + 1 for the empty value (w = log 5).  Node 2
    lacks the key (raw 0, the minimum), zone 0 holds 40 pods (node 0, the maximum), node 1 in zone 1 at 0 wins by the
    lift.  With c = GoRound(40 log 5), node 1's pts is 100 - 100 c / (2c) = 50; without the +1 (w = log 4) node 0's
    raw drops and node 1 gets 49."""
    w = math.log(5)
    x = _pts_raw(40, w, 0)
    keys = [(np.array([0, 1, -1], np.int32), 2), (np.arange(3, dtype=np.int32), 3)]
    soft = np.zeros((2, 2), np.uint32)
    soft[0, 0] = x + 1
    case = _boosted_soft_case("empty value +1", 3, keys, soft, {(0, 0, 0): 40}, 1, soft_all=[0, 1])
    case.kills, case.expect = ("no-empty-domain",), ((0, 1, 50),)
    return case


def ignored_case():
    """soft_all_keys = 1, two soft keys; node 2 lacks key 1 and is ignored, so zone 2 of key 0 is not counted: size_0 =
    2 (w = log 4).  Zone 0 at 40 pods (node 0, the maximum and the winner), node 1 at 0 the minimum; with c =
    GoRound(40 log 4) node 0's pts is 100 c / (2c) = 50, and with the ignored zone counted (w = log 5) 49."""
    x = _pts_raw(40, math.log(4), 0)
    keys = [(np.array([0, 1, 2], np.int32), 3), (np.array([0, 0, -1], np.int32), 1), (np.arange(3, dtype=np.int32), 3)]
    soft = np.zeros((2, 3), np.uint32)
    soft[0, 0], soft[0, 1] = x + 1, 1
    case = _boosted_soft_case("ignored node's domain", 3, keys, soft, {(0, 0, 0): 40}, 0)
    case.kills, case.expect = ("ignored-domains",), ((0, 1, 50),)
    return case


def size_one_case(with_empty):
    """A one-domain zone key (size 1, w = log 3) beside a soft hostname key.  Nodes 0 and 1 share the zone at soft
    count 30, node 1's host is at 5; with_empty: node 2 lacks the zone under soft_all_keys = 0, so size is 2 (w = log 4),
    else node 2 sits in the zone too.  Node 0 wins by the lift; the zone's constant is the first in 1..399 at which
    dropping the empty value's +1 changes the outputs (the zone term then moves node 0 against node 2's raw)."""
    zone = [0, 0, -1] if with_empty else [0, 0, 0]
    keys = [(np.array(zone, np.int32), 1), (np.arange(3, dtype=np.int32), 3), (np.arange(3, dtype=np.int32), 3)]

    def build(c):
        soft = np.zeros((2, 3), np.uint32)
        soft[0, 0], soft[0, 1] = c + 1, 1
        return _boosted_soft_case(f"size 1{' and the empty value' if with_empty else ''} c={c}", 3, keys, soft,
                                  {(0, 0, 0): 30, (0, 1, 1): 5}, 0, soft_all=[0 if with_empty else 1, 1])
    if not with_empty:
        return build(0)
    case = next(c for c in map(build, range(1, 400)) if kills(c, "no-empty-domain", ("profile",), (4,)))
    case.kills = ("no-empty-domain",)
    return case


def _middle_raw(a, b, w, c):
    """pts of the candidate at soft count a when the others sit at 0 (raw c, the minimum) and b (the maximum)"""
    M, r = _pts_raw(b, w, c), _pts_raw(a, w, c)
    return 100 * (M + c - r) // M


def _tuned_constant(a, b, w, wrong, cs):
    """The first constant c of `cs` at which the middle candidate's pts differs under every weight of `wrong`"""
    return next(c for c in cs if all(_middle_raw(a, b, v, c) != _middle_raw(a, b, w, c) for v in wrong))


def hostname_case(N):
    """Every node a candidate on a hostname soft key, so size = N and w = logw[N], the last entry of the call's table
    [N + 2].  Host 0 (the winner, by the lift) at soft count 2^23, host N - 1 at 2^24 (the maximum), the rest at 0 (the
    minimum, raw c).  pts(0) = 100 (M + c - r) / M moves with w only through c: c is the first constant, from the one at
    which the pts sits on 60 under log(N + 2), at which log(N + 3) gives another pts."""
    w = math.log(N + 2)
    a, b = 1 << 23, 1 << 24
    M, r = _pts_raw(b, w, 0), _pts_raw(a, w, 0)
    c0 = (60 * M - 100 * (M - r)) // 40  # 100 (M - r + c) / (M + c) = 60
    c = _tuned_constant(a, b, w, [math.log(N + 3)], range(max(c0 - 2000, 0), c0 + 2000))
    keys = [(np.arange(N, dtype=np.int32), N), (np.arange(N, dtype=np.int32), N)]
    soft = np.zeros((2, 2), np.uint32)
    soft[0, 0] = c + 1
    case = _boosted_soft_case(f"hostname N={N}", N, keys, soft, {(0, 0, 0): a, (0, 0, N - 1): b}, 0)
    case.kills, case.expect = ("logw-shifted",), ((0, 1, _middle_raw(a, b, w, c)),)
    return case


BITMAP_ZONES = list(range(2040, 2056)) + list(range(4090, 4100))  # 8 candidate zones below 2048, 18 at or above


def bitmap_edge_case():
    """Zone domains on both sides of PB_SH_WORDS * 32 = 2048, where the CTA's shared bitmap ends: 8,200 nodes, two per
    zone (zone n // 2, so the key is not one node per domain and the walk counts size_k through the bitmaps), group 0's
    selector on the nodes of zones 2040-2055 and 4090-4099: size = 26, 8 of them below 2048.  Zone 2048 (nodes 4096 and
    4097) at soft count a wins by the lift on node 4096, zone 2047 at b is the maximum, the rest at 0 the minimum; a, b
    and the constant are the first at which the winner's pts changes when size_k misses either bitmap's domains or w is
    read one entry off."""
    N = 8200
    zone = (np.arange(N) // 2).astype(np.int32)
    size = len(BITMAP_ZONES)
    below = sum(z < SHARED_BITMAP for z in BITMAP_ZONES)
    w = math.log(size + 2)
    wrong = [math.log(size - below + 2), math.log(below + 2), math.log(size + 3)]
    a, b, c = next((a, b, c) for b in range(2, 40) for a in range(1, b) for c in range(0, 60)
                   if all(_middle_raw(a, b, v, c) != _middle_raw(a, b, w, c) for v in wrong))
    keys = [(zone, N // 2), (np.arange(N, dtype=np.int32), N)]
    soft = np.zeros((2, 2), np.uint32)
    soft[0, 0] = c + 1
    case = _boosted_soft_case("domains at 2047 / 2048", N, keys, soft, {(0, 0, 2048): a, (0, 0, 2047): b}, 4096)
    lab = np.zeros((N, 1), np.uint64)
    lab[np.isin(zone, BITMAP_ZONES), 0] = 1
    case.lab, case.sel = lab, np.ones((case.P, 1), np.uint64)
    case.kills = ("shared-bitmap-only", "global-bitmap-only", "logw-shifted")
    case.expect = ((0, 1, _middle_raw(a, b, w, c)),)
    return case


def ignored_all_case(mode):
    """soft_all_keys = 1 and candidates that lack the soft key: 'all' (every candidate ignored: pts 0 everywhere, the IPA
    lift decides), 'one' (one candidate not ignored: min = max = its raw), 'zero' (max 0: every soft count 0, pts 100)"""
    N = 5
    zone = {"all": [-1] * 5, "one": [-1, -1, 0, -1, -1], "zero": [0, 1, 2, 3, 4]}[mode]
    keys = [(np.array(zone, np.int32), 5), (np.arange(N, dtype=np.int32), N)]
    soft = np.zeros((2, 2), np.uint32)
    soft[0, 0] = 1
    return _boosted_soft_case(f"ignored {mode}", N, keys, soft, {}, 2, P=3)


# ------------------------------------------------------------------------------------------ InterPodAffinity cases
def ipa_case(a, b, variant="w1", N=3, where=None):
    """ipa at a truncating pair: candidate raws min, min + a and min + b, so the middle node's ipa is
    (int64)(100.0 * (a / b)), one below (100 a) // b.  A hostname soft spread (every other host at soft count 10) gives
    the middle node pts 100 and the others 0, so it wins.  Variants: 'w1' (weight-1 preferred term, existing pods of
    group 1), 'hard100' (group 1's required affinity towards group 0 at hard_affinity_weight 100), 'dup100' (two
    weight-100 duplicate terms), 'negative' (an anti-preferred term towards group 2: raws -b, a - b, 0).  N > 3: the
    three nodes at `where` = (min node, middle node, max node) among N, the others at raw 0 between the extremes
    (variant 'mixed': a preferred term towards group 1 and an anti-preferred one towards group 2, min = -1)."""
    lo, mid, hi = where if where is not None else (0, 1, 2)
    G = 3
    host = np.arange(N, dtype=np.int32)
    keys = [(host, N)]
    soft = np.zeros((G, 1), np.uint32)
    soft[0, 0] = 1
    ex = np.full((G, N), 0, np.uint32)
    ex[0, :] = 10
    ex[0, mid] = 0
    hard = 1
    if variant == "w1":
        pods, terms, tw = _pods_on([(mid, a), (hi, b)], 1), [(0, PREFERRED, 0, [1])], [1]
    elif variant == "hard100":
        pods, terms, tw, hard = _pods_on([(mid, a), (hi, b)], 1), [(1, AFFINITY, 0, [0])], [0], 100
    elif variant == "dup100":
        pods, terms, tw = _pods_on([(mid, a), (hi, b)], 1), [(0, PREFERRED, 0, [1])] * 2, [100, 100]
    elif variant == "negative":
        pods, terms, tw = _pods_on([(lo, b), (mid, b - a)], 2), [(0, ANTI_PREFERRED, 0, [2])], [1]
    else:  # mixed: min -1, middle a - 1, max b - 1, everything else 0
        pods = _merge_pods(_pods_on([(lo, 1)], 2), _pods_on([(mid, a - 1), (hi, b - 1)], 1))
        terms, tw = [(0, PREFERRED, 0, [1]), (0, ANTI_PREFERRED, 0, [2])], [1, 1]
    kw = dict(soft_skew=soft, existing=[ex], existing_pods=pods, terms=terms, term_weight=tw, hard_affinity_weight=hard)
    want = int(100.0 * (a / b))
    return Case(f"ipa {variant} ({a}, {b}) N={N}", N, np.zeros(2, np.int32), G, keys, kw, kills=("integer-ipa",),
                expect=((0, 2, want),))


def ipa_slice_cases(N, sms):
    """The extremes only in the first slice (nodes 0 and 1) or only in the last (nodes N - 1, N - 2), the middle node
    at the other end, at the (29, 50) pair"""
    return [ipa_case(29, 50, "mixed", N, where=(0, N - 1, 1)), ipa_case(29, 50, "mixed", N, where=(N - 1, 0, N - 2))]


# ------------------------------------------------------------------------------------------ TaintToleration cases
def taint_case(M):
    """Nodes 0..M, node i with i untolerated PreferNoSchedule taints (max = M); group g prefers node g at weight 100
    with NodeAffinity's plugin weight 100, so pod g binds on node g and shows tt = 100 - 100 g / M"""
    N, G = M + 1, M + 1
    labels = [{"n": str(i)} for i in range(N)]
    taints = [[{"key": f"t{j}", "value": "", "effect": "PreferNoSchedule"} for j in range(i)] for i in range(N)]
    rules = [{"preferred": [(100, [{"key": "n", "operator": "In", "values": [str(g)]}])]} for g in range(G)]
    keys = [(np.zeros(N, np.int32), 1)]
    kills = []
    if any(2 * (100 * g % M) >= M for g in range(N)):
        kills.append("rounded-normalize")
    if any(100 * g % M for g in range(N)):
        kills.append("complement-tt")
    return Case(f"taints max={M}", N, np.arange(G, dtype=np.int32), G, keys, dict(weight_node_affinity=100),
                calls=("node", "fit"), cluster=(labels, taints, rules), kills=tuple(kills),
                expect=tuple((g, 3, 100 - 100 * g // M) for g in range(N)))


# ------------------------------------------------------------------------------------------ NodeAffinity cases
NA_TERMS = 4096


def node_affinity_case():
    """Groups 0 and 1 share one rule class: 4,096 weight-100 preferred terms, term j matching the nodes whose match count
    exceeds j.  Node 2 matches all (raw 409,600, the cap) and carries one PreferNoSchedule taint (tt 0); node 1 matches
    2,069 terms (na = 100 * 206,900 / 409,600 = 50.51, truncated 50) and wins; node 3 matches 1,024 (na 25 exactly)."""
    matches = [0, 2069, NA_TERMS, 1024]
    N = len(matches)
    labels = [{"v": str(i)} for i in range(N)]
    terms = [(100, [{"key": "v", "operator": "In", "values": [str(i) for i in range(N) if matches[i] > j]}])
             for j in range(NA_TERMS)]
    rule = {"preferred": terms}
    taints = [[], [], [{"key": "spot", "value": "", "effect": "PreferNoSchedule"}], []]
    keys = [(np.zeros(N, np.int32), 1)]
    return Case("node affinity 4096 x 100", N, np.array([0, 1, 0], np.int32), 2, keys, {}, calls=("node", "fit"),
                cluster=(labels, taints, [rule, dict(rule)]), kills=("rounded-normalize",), expect=((0, 4, 50),))


# ---------------------------------------------------------------------------------------------------- total ties
def tie_nodes(N, sms):
    """Both sides of every edge between two walk slices, and the first and last node"""
    grid, chunk = bind_slices(N, sms)
    e = {0, N - 1}
    for s in range(1, grid):
        if s * chunk < N:
            e.update((s * chunk - 1, s * chunk))
    return np.array(sorted(e), np.int64)


def tie_case(N, sms):
    """Ties between two decompositions of the total at every slice edge: the candidates (one selector bit) are the edge
    nodes; on alternate edges the left or the right node is 'a' (soft count 0: pts 100, ipa 0) and the other 'b' (soft
    count 1 and an existing pod of the preferred target: pts 0, ipa 100), so both total 2 * 100.  Each binding lowers
    the bound node, and the queue walks the ties edge by edge; ties go to the lower index."""
    E = tie_nodes(N, sms)
    _, chunk = bind_slices(N, sms)
    b_nodes = [int(n) for n in E if (n // chunk) % 2 == 1]  # the left node on even edges, the right one on odd edges
    lab = np.zeros((N, 1), np.uint64)
    lab[E, 0] = 1
    keys = [(np.arange(N, dtype=np.int32), N)]
    soft = np.zeros((2, 1), np.uint32)
    soft[0, 0] = 1
    ex = np.zeros((2, N), np.uint32)
    ex[0, b_nodes] = 1
    kw = dict(soft_skew=soft, existing=[ex], existing_pods=_pods_on([(n, 1) for n in b_nodes], 1),
              terms=[(0, PREFERRED, 0, [1])], term_weight=[1])
    P = len(E)
    return Case(f"ties N={N} sms={sms}", N, np.zeros(P, np.int32), 2, keys, kw, lab=lab,
                sel=np.ones((P, 1), np.uint64), kills=("ties-high",))


def weight_case(ws, wa):
    """Plugin weights 0 and 100 on the (29, 50) IPA queue: weight_spread ws, weight_affinity wa.  With ws > 0 the
    middle node still wins by its pts and reports ipa 57 whatever wa is; with ws = 0 the max node (wa > 0) or node 0
    (both 0: every total ties) wins and no part sits on the hazard."""
    case = ipa_case(29, 50)
    case.kw.update(weight_spread=ws, weight_affinity=wa)
    case.name += f" weights {ws}/{wa}"
    if not ws:
        case.kills, case.expect = (), ((0, 2, 100 if wa else 0),)
    return case


# ------------------------------------------------------------------------------------------------------------- gangs
def gang_cases():
    """ks_gang_fit_bind over soft counts near 2^24 and large IPA counters: the cross_case queue, and the 20,000-pod IPA
    queue with a weight-100 anti-preferred self term (each bound pod of group 0 lowers its host's IPA raw by 200 for the
    next pod of group 0, one point of ipa), each cut into gangs of two with the middle gang unable to place (a pod of
    2^36 millicores).  The middle gang's first pod binds and changes the soft counts or the IPA counters; the rollback
    must undo that, or the last gang's parts differ (test_score_edges.py checks that they do)."""
    ipa = ipa_case(*truncating_pair_20000(), "w1")
    ipa.kw["terms"] = ipa.kw["terms"] + [(0, ANTI_PREFERRED, 0, [0])]
    ipa.kw["term_weight"] = ipa.kw["term_weight"] + [100]
    out = []
    for base in (cross_case(), ipa):
        P = 6
        base.group = np.zeros(P, np.int32)
        rc = np.zeros(P, np.int64)
        rc[3] = 1 << 36
        base.rc = rc
        base.gangs = (np.array([0, 2, 4, 6], np.uint64), np.array([2, 2, 2], np.uint32))
        base.name = "gang " + base.name
        base.calls = ("gang",)
        base.expect, base.kills = (), ()
        out.append(base)
    return out


def truncating_pair_20000():
    return tuple(fixture()["truncating_20000"])


# ------------------------------------------------------------------------------------------------------ case lists
def pts_cases():
    halves = [half_case(*h) for h in fixture()["exact_halves"]]
    return halves + [cross_case(), skew_case(1 << 31), skew_case((1 << 32) - 1), empty_value_case(), ignored_case(),
                     size_one_case(False), size_one_case(True), bitmap_edge_case()] + [ignored_all_case(m) for m in
                                                                                         ("all", "one", "zero")]


def ipa_cases():
    pairs = fixture()["truncating"]
    out = [ipa_case(a, b, v) for a, b in pairs for v in ("w1", "negative")]
    out += [ipa_case(29, 50, "hard100"), ipa_case(57, 100, "dup100"), ipa_case(*truncating_pair_20000(), "w1")]
    return out


def node_rule_cases():
    return [taint_case(M) for M in range(1, 65)] + [node_affinity_case()]


def weight_cases():
    return [weight_case(ws, wa) for ws, wa in ((0, 100), (100, 0), (100, 100), (0, 0))]


def cpu_cases():
    """Every case whose mutant claims test_score_edges.py checks on the CPU: all but the shapes that need the SM count,
    and the tie queue at N = 129 on 132 SMs"""
    return pts_cases() + ipa_cases() + node_rule_cases() + weight_cases() + [tie_case(129, 132)]


if __name__ == "__main__":
    if "--regenerate" in sys.argv:
        regenerate()
