"""Preemption and drain under the full filter at their edges: the cases of test_fit_edges.py (CPU) and
test_fit_edges_gpu.py (H100), a model of the node-chunk grid both scans launch, and mutants of the two restatements
(fit_preempt_oracle.py, fit_drain_oracle.py) that each case must tell apart.

ks_fit_preempt (k_fit_preempt_scan) and ks_fit_drain_check (k_fit_drain_scan) split the nodes across gridDim.y when the
pods give fewer than two CTAs per SM: each CTA carries its counts and its best key over `tiles_per_chunk` tiles of
TILE_N nodes, and the chunks merge in ascending order.  The geometry cases reach chunks of several tiles with a short
last chunk, four chunks over ten tiles, and one chunk over every tile, with candidates on both sides of each edge.  The
other families sit on one hazard each: the 128-bit victim key (ks_internal.cuh, preempt_key), the boundaries of the
reprieve walk, and the scalar-resource and pod-count edges of both calls.

A case is a dict the restatement takes (fit_preempt_oracle.cluster_inputs plus the string-level objects, or
fit_drain_oracle.cluster) and the mutants it claims to kill; test_fit_edges.py checks every claim on the CPU."""
import os
import re
from dataclasses import dataclass, field

import numpy as np

import fit_drain_oracle as fdo
import fit_preempt_oracle as fpo
import oracle_mutants

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kube-scheduler-rs-reference_b200",
                    "csrc")
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1


def source_constant(fname, name):
    """An integer `constexpr` of the CUDA sources; one definition must exist, or the model would drift silently"""
    with open(os.path.join(CSRC, fname)) as f:
        found = re.findall(rf"constexpr\s+\w+\s+{name}\s*=\s*(\d+)u?\s*;", f.read())
    assert len(found) == 1, f"{name} in {fname}: {found}"
    return int(found[0])


TILE_N = source_constant("ks_internal.cuh", "TILE_N")
DIRECT_THREADS = source_constant("ks_internal.cuh", "DIRECT_THREADS")
FIT_PREEMPT_PODS_PER_WARP = source_constant("ks_launch.h", "FIT_PREEMPT_PODS_PER_WARP")
FIT_DRAIN_PODS_PER_WARP = source_constant("ks_launch.h", "FIT_DRAIN_PODS_PER_WARP")


# ---------------------------------------------------------------------------------------------------- grid model
@dataclass(frozen=True)
class Grid:
    """direct_grid_ppw's launch (ks_direct.cu): pod_ctas x n_chunks CTAs, chunk c scanning tiles [c * tiles_per_chunk,
    min((c + 1) * tiles_per_chunk, n_tiles)) of N nodes"""
    pod_ctas: int
    n_chunks: int
    tiles_per_chunk: int
    n_tiles: int
    N: int

    def chunks(self):
        """(first, last) real node of each chunk"""
        span = self.tiles_per_chunk * TILE_N
        return [(c * span, min((c + 1) * span, self.N) - 1) for c in range(self.n_chunks)]

    def chunk_of(self, n):
        return n // (self.tiles_per_chunk * TILE_N)

    @property
    def uneven(self):
        """The last chunk holds fewer tiles than the others"""
        return self.n_tiles - (self.n_chunks - 1) * self.tiles_per_chunk < self.tiles_per_chunk


def direct_grid(ppw, P, N, sms):
    """direct_grid_ppw(ppw, P, Npad, sms): node chunks across gridDim.y when the pods alone give fewer than two CTAs per
    SM, then the chunk count recomputed from the tiles per chunk"""
    assert N > 0
    pods_per_cta = (DIRECT_THREADS // 32) * ppw
    n_tiles = -(-N // TILE_N)
    want = 2 * sms
    pod_ctas = -(-P // pods_per_cta)
    n_chunks = min(n_tiles, -(-want // pod_ctas)) if pod_ctas < want else 1
    tpc = -(-n_tiles // n_chunks)
    return Grid(pod_ctas, -(-n_tiles // tpc), tpc, n_tiles, N)


def preempt_grid(P, N, sms):
    return direct_grid(FIT_PREEMPT_PODS_PER_WARP, P, N, sms)


def drain_grid(D, N, sms):
    """The grid of a drain round (and of the refusal pass) with D candidates running"""
    return direct_grid(FIT_DRAIN_PODS_PER_WARP, D, N, sms)


# ------------------------------------------------------------------------------------------------------- mutants
_WALK = (("fit_preempt_oracle", "fit_preempt_packed"),)
_FITS = (("fit_preempt_oracle", "fits_state"),)
_REQ = (("fit_bind_oracle", "fits_request"),)
_DRAIN = (("fit_drain_oracle", "fit_drain"),)


def _order(fields):
    """The candidate comparison with the key (vmax, vsum, vcnt, node) read as `fields` of k (the row still reports the
    real fields)"""
    best = fields.replace("k[", "best[0][")
    return "if best is None or k < best[0]:", f"if best is None or ({fields},) < ({best},):"


# name -> (what a kernel would get wrong, the functions patched, [(restatement text, mutant text)])
MUTANTS = {
    "zero-left-cpu": ("a reprieve that leaves exactly 0 cpu refused (rc >= avail)", _FITS,
                      [("if rc > c or rm > m:", "if rc >= c or rm > m:")]),
    "zero-left-mem": ("a reprieve that leaves exactly 0 memory refused", _FITS,
                      [("if rc > c or rm > m:", "if rc > c or rm >= m:")]),
    "zero-left-scalar": ("a scalar request that leaves exactly 0 refused", _REQ,
                         [("if q > alloc.get(name, 0) - requested.get(name, 0):",
                           "if q >= alloc.get(name, 0) - requested.get(name, 0):")]),
    "zero-left-pods": ("the last pod slot refused (pods + 1 >= allocatable)", _REQ,
                       [("if n_pods + 1 > alloc.get(\"pods\", 0):", "if n_pods + 1 >= alloc.get(\"pods\", 0):")]),
    "lower-set-inclusive": ("bound pods at the pod's own priority in the lower set", _WALK,
                            [("if bound[b][3] < pi", "if bound[b][3] <= pi")]),
    "ties-high-bound": ("equal priorities walked from the higher bound index", _WALK,
                        [("key=lambda b: (-bound[b][3], b)", "key=lambda b: (-bound[b][3], -b)")]),
    "evict-keeps-pod-count": ("an eviction that does not free one pod of the pods count",
                              (("fit_preempt_oracle", "evicted"),),
                              [("usage.pods[n] - len(removed))", "usage.pods[n])")]),
    "max-victims-exclusive": ("a plan of exactly max_victims victims refused", _WALK,
                              [("if len(vic) > max_victims:", "if len(vic) >= max_victims:")]),
    "key-count-first": ("the key orders the victim count before the priority sum", _WALK,
                        [_order("k[0], k[2], k[1], k[3]")]),
    "key-no-count": ("the victim count left out of the key", _WALK, [_order("k[0], k[1], k[3]")]),
    "key-sum-high-bits": ("the priority sum's low 8 bits dropped from the key", _WALK,
                          [_order("k[0], k[1] >> 8, k[2], k[3]")]),
    "key-node-high": ("node ties to the higher index", _WALK, [_order("k[0], k[1], k[2], -k[3]")]),
    "no-zero-skip": ("a zero request checked against a negative free amount", _REQ + _DRAIN,
                     [("if name in CPU_MEM or name == \"pods\" or q == 0:", "if name in CPU_MEM or name == \"pods\":"),
                      ("if name in CPU_MEM or q == 0 or", "if name in CPU_MEM or")]),
    "drain-keeps-pod-count": ("the drain overlay does not charge the pod count", _DRAIN,
                              [("st[3] += 1", "pass")]),
    "drain-keeps-scalar": ("the drain overlay does not charge the scalar resources", _DRAIN,
                           [("st[2][name] = st[2].get(name, 0) + q", "pass")]),
    "drain-taint-first": ("a destination that fails a resource and a taint counted as taint", _DRAIN + (
        ("fit_drain_oracle", "Cluster.node_stage"),),
        [("stage = np.where((stage > 0) & lack, 1, stage)", "stage = np.where((stage == PASS) & lack, 1, stage)"),
         ("    if self.alloc is not None and fits_request(d[\"pod_res\"][p], self.alloc[n], req, pods):\n"
          "        return 1\n    return int(self.rule_stage(int(d[\"group\"][p]))[n])",
          "    st = int(self.rule_stage(int(d[\"group\"][p]))[n])\n"
          "    if st == PASS and self.alloc is not None and fits_request(d[\"pod_res\"][p], self.alloc[n], req, pods):\n"
          "        return 1\n    return st")]),
    "drain-ties-high": ("the drain argmax ties to the higher node index", _DRAIN,
                        [("best = int(np.argmax(sc))", "best = len(sc) - 1 - int(np.argmax(sc[::-1]))")]),
}

# Mistakes no reachable input tells apart from the restatement: the case list runs them and none may be killed.
NEUTRAL = {
    "key-sum-int64-wrap": ("the priority sum wrapped at 2^40 before it is packed: at most 128 victims of terms below 2^32 "
                           "keep it below 2^39, so the wrap never happens", _WALK,
                           [_order("k[0], k[1] % (1 << 40), k[2], k[3]")]),
}


def mutant(name):
    """The restatements with one mutant's patches applied; restored on exit"""
    return oracle_mutants.mutant({**MUTANTS, **NEUTRAL}, name)


# --------------------------------------------------------------------------------------------------------- cases
MVS = (1, 3, 128)
RUNS = tuple((policy, flags) for policy in (0, 1, 3, 4) for flags in (0, 1))


@dataclass
class Case:
    """One cluster for one call ("preempt" or "drain"): d as the restatement takes it, kills the mutants it tells
    apart, mvs the max_victims it runs at (preempt), runs the (policy, flags) pairs (drain), family and geometry the
    shape it was built for (geometry: (kind, sms))."""
    name: str
    call: str
    d: dict
    kills: tuple = ()
    mvs: tuple = MVS
    runs: tuple = RUNS
    family: str = ""
    geometry: tuple = None
    notes: dict = field(default_factory=dict)


def run(case, arg):
    """The restatement's outputs at one max_victims (preempt) or one (policy, flags) pair (drain)"""
    d = case.d
    if case.call == "preempt":
        return fpo.run(d, arg)
    policy, flags = arg
    return fdo.fit_drain(d, d["node_idx"], d["offset"], policy, flags == 1)


def args_of(case):
    return case.mvs if case.call == "preempt" else case.runs


def differs(a, b):
    """Any output array differs: every row field, victim slot and unresolvable count, or placed, node, score and the
    refusal words"""
    if isinstance(a[0], np.ndarray) and a[0].dtype.names:
        if any(not np.array_equal(a[0][f], b[0][f]) for f in a[0].dtype.names):
            return True
        a, b = a[1:], b[1:]
    return any(not np.array_equal(x, y) for x, y in zip(a, b))


def kills(case, name):
    """Whether mutant `name` changes some output of the case at some max_victims or (policy, flags)"""
    for arg in args_of(case):
        want = run(case, arg)
        with mutant(name):
            got = run(case, arg)
        if differs(got, want):
            return True
    return False


# ------------------------------------------------------------------------------------------------ preempt builders
def _node(cpu=4000, mem=1 << 30, labels=None, taints=None, alloc=None):
    return dict(cpu=cpu, mem=mem, labels=labels or {}, taints=taints or [], alloc=alloc or {"pods": 110})


def _pod(cpu=0, mem=0, prio=100, sel=None, group=-1, res=None):
    return dict(cpu=cpu, mem=mem, selector=sel or {}, priority=prio, group=group, res=res or {})


def preempt_inputs(nodes, bound, pods, rules=(), names=None):
    """cluster_inputs with the string-level objects, for nodes (_node), bound (node, cpu, mem, priority, res) and pods
    (_pod)"""
    alloc = [n["alloc"] for n in nodes]
    d = fpo.cluster_inputs([n["cpu"] for n in nodes], [n["mem"] for n in nodes], [n["labels"] for n in nodes],
                           [n["taints"] for n in nodes], alloc, bound, pods, names)
    d.update(node_labels=[n["labels"] for n in nodes], node_taints=[n["taints"] for n in nodes],
             group_rules=list(rules), alloc=alloc, bound=list(bound), pod_res=[p["res"] for p in pods], G=len(rules))
    return d


def _preempt(name, family, nodes, bound, pods, kills, rules=(), names=None, mvs=MVS, **notes):
    return Case(name, "preempt", preempt_inputs(nodes, bound, pods, rules, names), tuple(kills), mvs, family=family,
                notes=notes)


GEOMETRY = ("a", "b", "c")


def geometry_shape(kind, sms):
    """(P, N) of a geometry family: (a) 8 pods over 2 sms + 1 tiles, chunks of 2 tiles and a last one of 1; (b) pods
    for half as many CTAs as SMs over 10 tiles, 4 chunks of 3, 3, 3 and 1 tiles; (c) pods for two CTAs per SM, one
    chunk over all 10 tiles of N = 10,000"""
    per_cta = (DIRECT_THREADS // 32) * FIT_PREEMPT_PODS_PER_WARP
    if kind == "a":
        return per_cta, 2 * sms * TILE_N + 1
    if kind == "b":
        return per_cta * -(-sms // 2), 9 * TILE_N + 5
    return per_cta * 2 * sms, 10_000


def tile_pairs(N):
    """(t, left, right) for every tile boundary t: the last node of tile t - 1 and the first of tile t"""
    return [(t, t * TILE_N - 1, t * TILE_N) for t in range(1, -(-N // TILE_N))]


def geometry_case(kind, sms):
    """Candidates on both sides of every tile boundary (so on both sides of every chunk edge) and on nodes 0 and N - 1;
    every other node lacks the pods' selector labels, so it is unresolvable and the unresolvable sums cross every chunk
    and the padding.  Each candidate is full (4,000 cpu) with one bound pod of priority q: 0 on the left of a boundary,
    -1 on the right of an odd one (else 0), -1 on N - 1, and -7 on the left of the 'star' boundary, the last node of a
    chunk that has candidates in earlier tiles.  Pods (4,000 cpu) come in four families: all candidates at priority 10
    (the star wins after a carry over the chunk's tiles) and at 0 (only q < 0 are candidates); one boundary pair at 10
    (an even pair ties on every key field but the node, an odd one's right node is better) and at 0 (the lower set is
    strictly below: an even pair has no candidate)."""
    P, N = geometry_shape(kind, sms)
    g = preempt_grid(P, N, sms)
    pairs = tile_pairs(N)
    star = g.tiles_per_chunk * (g.n_chunks // 2) if g.n_chunks > 1 else len(pairs) // 2 + 1
    if star > len(pairs):
        star = len(pairs)
    nodes = [_node() for _ in range(N)]
    q = {0: 0, N - 1: -1}
    nodes[0]["labels"] = {"c": "1", "e": "first"}
    nodes[N - 1]["labels"] = {"c": "1", "e": "last"}
    for t, left, right in pairs:
        nodes[left]["labels"] = {"c": "1", "e": str(t)}
        nodes[right]["labels"] = {"c": "1", "e": str(t)}
        q[left] = -7 if t == star else 0
        q[right] = -1 if t % 2 else 0
    bound = [(n, 4000, 0, q[n], {}) for n in sorted(q)]
    pods = []
    for p in range(P):
        fam, i = p % 4, p // 4
        t = 1 + (i * 37) % len(pairs)
        sel = {"c": "1"} if fam in (0, 3) else {"e": str(t)}
        pods.append(_pod(cpu=4000, prio=10 if fam in (0, 1) else 0, sel=sel))
    case = _preempt(f"geometry {kind} sms={sms} P={P} N={N}", "geometry", nodes, bound, pods,
                    ("key-node-high", "lower-set-inclusive"), names=["pods"], star=star)
    case.geometry = (kind, sms)
    return case


def key_cases():
    """Identical pods on nodes whose lower sets tie on every key field but one"""
    out = []
    # vmax 10 on both, sums 2^32 + 15 and 2^32 + 14: equal above the low 8 bits; node 1 wins by the sum alone
    nodes = [_node(cpu=2000), _node(cpu=2000)]
    bound = [(0, 1000, 0, 10, {}), (0, 1000, 0, 5, {}), (1, 1000, 0, 10, {}), (1, 1000, 0, 4, {})]
    out.append(_preempt("key: sum's low 8 bits", "key", nodes, bound, [_pod(cpu=2000)], ["key-sum-high-bits"],
                        names=["pods"], pair=(0, 1)))
    # equal vmax and sum (an INT32_MIN victim adds 0), node 0 two victims, node 1 one: node 1 wins by the count
    bound = [(0, 1000, 0, 10, {}), (0, 1000, 0, INT32_MIN, {}), (1, 2000, 0, 10, {})]
    out.append(_preempt("key: count only", "key", nodes, bound, [_pod(cpu=2000)], ["key-no-count"], names=["pods"],
                        pair=(0, 1)))
    # node 0: 2 victims, sum 2^32 + 19; node 1: 3 victims, sum 2^31 + 10 - the sum decides before the count
    bound = [(0, 1000, 0, 10, {}), (0, 1000, 0, 9, {}), (1, 1000, 0, 10, {}), (1, 500, 0, INT32_MIN, {}),
             (1, 500, 0, INT32_MIN, {})]
    out.append(_preempt("key: sum before count", "key", nodes, bound, [_pod(cpu=2000)], ["key-count-first"],
                        names=["pods"], pair=(0, 1)))
    # the same plan on nodes 1023 and 1024, on either side of a chunk edge (3 tiles, 8 pods: one tile per chunk), and
    # on nodes 2047, 2048 and N - 1 = 3071 at a worse victim priority
    N = 3 * TILE_N
    nodes = [_node() for _ in range(N)]
    cand = {1023: 0, 1024: 0, 2047: 1, 2048: 1, N - 1: 1}
    for n in cand:
        nodes[n]["labels"] = {"c": "1"}
    bound = [(n, 4000, 0, pr, {}) for n, pr in cand.items()]
    pods = [_pod(cpu=4000, sel={"c": "1"}, prio=p) for p in (10, 1, 2, 0)] * 2
    out.append(_preempt("key: node ties across a chunk edge", "key", nodes, bound, pods, ["key-node-high"],
                        names=["pods"], pair=(1023, 1024)))
    # 128 victims at 2^31 - 2 (sum 2^39 - 256) against 127 of them and one at 2^31 - 3 (sum one lower), for a pod at
    # INT32_MAX; only max_victims 128 holds either plan
    nodes = [_node(cpu=12800), _node(cpu=12800)]
    bound = [(0, 100, 0, INT32_MAX - 1, {}) for _ in range(128)]
    bound += [(1, 100, 0, INT32_MAX - 1, {}) for _ in range(127)] + [(1, 100, 0, INT32_MAX - 2, {})]
    out.append(_preempt("key: sum near 2^39", "key", nodes, bound, [_pod(cpu=12800, prio=INT32_MAX)],
                        ["max-victims-exclusive"], names=["pods"], mvs=(1, 3, 127, 128), pair=(0, 1)))
    return out


def walk_cases():
    """One small node set on each side of each boundary of the reprieve walk"""
    out = []
    # a bound pod at the pod's own priority is not in the lower set: node 0 holds only one, node 1 one below and one at
    nodes = [_node(cpu=2000, labels={"n": "0"}), _node(cpu=2000, labels={"n": "1"})]
    bound = [(0, 2000, 0, 50, {}), (1, 1000, 0, 49, {}), (1, 1000, 0, 50, {})]
    pods = [_pod(cpu=1000, prio=50, sel={"n": "0"}), _pod(cpu=2000, prio=50, sel={"n": "1"}),
            _pod(cpu=1000, prio=51, sel={"n": "0"})]
    out.append(_preempt("walk: bound pod at the pod's priority", "walk", nodes, bound, pods, ["lower-set-inclusive"],
                        names=["pods"]))
    # equal priorities walk in bound-index order: node 0's two priority-5 pods sit at bound indices 1 (2,000 cpu) and
    # 3 (1,000 cpu) between node 1's pods; the first one visited is reprieved
    nodes = [_node(cpu=3000), _node(cpu=1000)]
    bound = [(1, 500, 0, 0, {}), (0, 2000, 0, 5, {}), (1, 500, 0, 0, {}), (0, 1000, 0, 5, {})]
    pods = [_pod(cpu=1000, prio=6)]
    out.append(_preempt("walk: equal priorities in bound order", "walk", nodes, bound, pods, ["ties-high-bound"],
                        names=["pods"]))
    # the reprieve of the priority-5 pod leaves exactly 0 in one dimension; the priority-4 pod is the victim
    X = "example.com/x"
    zero = [
        ("cpu", _node(cpu=3000), [(0, 1000, 0, 5, {}), (0, 2000, 0, 4, {})], _pod(cpu=2000), ["zero-left-cpu"]),
        ("memory", _node(mem=3000), [(0, 0, 1000, 5, {}), (0, 0, 2000, 4, {})], _pod(mem=2000), ["zero-left-mem"]),
        ("a scalar resource", _node(alloc={"pods": 110, X: 3}), [(0, 0, 0, 5, {X: 1}), (0, 0, 0, 4, {X: 2})],
         _pod(res={X: 2}), ["zero-left-scalar"]),
        ("pods", _node(alloc={"pods": 2}), [(0, 0, 0, 5, {}), (0, 0, 0, 4, {})], _pod(),
         ["zero-left-pods", "evict-keeps-pod-count"]),
    ]
    for what, node, bound, pod, k in zero:
        names = ["pods", X] if X in node["alloc"] else ["pods"]
        out.append(_preempt(f"walk: reprieve leaves 0 {what}", "walk", [node], bound, [pod], k, names=names,
                            zero=what))
    # exactly max_victims victims is a plan, one more is none: 3 needed, at max_victims 2 and 3
    bound = [(0, 1000, 0, pr, {}) for pr in (1, 2, 3)]
    out.append(_preempt("walk: max_victims = needed, needed - 1", "walk", [_node(cpu=3000)], bound, [_pod(cpu=3000)],
                        ["max-victims-exclusive"], names=["pods"], mvs=(2, 3)))
    # the int32 ends: a pod at INT32_MAX over bound pods at INT32_MAX and INT32_MAX - 1; pods at INT32_MIN (no lower set,
    # even over a bound pod at INT32_MIN) and INT32_MIN + 1 (its victim at INT32_MIN: key hi 0)
    nodes = [_node(cpu=2000, labels={"n": "0"}), _node(cpu=1000, labels={"n": "1"})]
    bound = [(0, 1000, 0, INT32_MAX, {}), (0, 1000, 0, INT32_MAX - 1, {}), (1, 1000, 0, INT32_MIN, {})]
    pods = [_pod(cpu=1000, prio=INT32_MAX, sel={"n": "0"}), _pod(cpu=1000, prio=INT32_MIN, sel={"n": "1"}),
            _pod(cpu=1000, prio=INT32_MIN + 1, sel={"n": "1"}), _pod(cpu=1000, prio=INT32_MIN)]
    out.append(_preempt("walk: priorities INT32_MIN and INT32_MAX", "walk", nodes, bound, pods,
                        ["lower-set-inclusive"], names=["pods"]))
    return out


R8 = ["pods"] + [f"example.com/r{i}" for i in range(1, 8)]


def preempt_scalar_cases():
    """Zero requests on negative free amounts, and a non-contiguous request mask at R = 8"""
    out = []
    X, Y = "example.com/x", "example.com/y"
    # node 0 must evict its priority-0 pod; x's free amount is -2 on both nodes (a priority-1000 pod holds 3 of 1).
    # Pod 0 asks 0 of x (and of y, which no node has) and preempts on node 0; pod 1 fits node 1 as it is.
    nodes = [_node(labels={"n": "0"}, alloc={"pods": 110, X: 1}), _node(labels={"n": "1"}, alloc={"pods": 110, X: 1})]
    bound = [(0, 2000, 0, 1000, {X: 3}), (0, 2000, 0, 0, {}), (1, 1000, 0, 1000, {X: 3})]
    pods = [_pod(cpu=2000, prio=500, sel={"n": "0"}, res={X: 0, Y: 0}),
            _pod(cpu=2000, prio=500, sel={"n": "1"}, res={X: 0})]
    out.append(_preempt("scalar: zero request, negative free", "scalar", nodes, bound, pods, ["no-zero-skip"],
                        names=["pods", X, Y]))
    # R = 8, the pod requests r2, r5 and r7 (mask 0b10100101 with pods) and 0 of the rest, which are negative on every
    # node; node n frees what the pod lacks only by evicting; node 2's reprieve leaves 0 of r5
    r = {nm: i for i, nm in enumerate(R8)}
    neg = {R8[i]: 0 for i in (1, 3, 4, 6)}
    hold = {R8[i]: 2 for i in (1, 3, 4, 6)}  # a priority-1000 pod on each node holds 2 of each of those
    nodes = [_node(alloc={"pods": 110, **neg, R8[2]: 1, R8[5]: 2, R8[7]: 1}) for _ in range(3)]
    bound = []
    for n in range(3):
        bound.append((n, 0, 0, 1000, dict(hold)))
    bound += [(0, 0, 0, 3, {R8[5]: 2}), (0, 0, 0, 2, {R8[7]: 1}),           # node 0: both must go
              (1, 0, 0, 3, {R8[2]: 1}), (1, 0, 0, 1, {R8[5]: 1}),           # node 1: r2 and r5 short
              (2, 0, 0, 4, {R8[5]: 1}), (2, 0, 0, 3, {R8[5]: 1}), (2, 0, 0, 2, {R8[7]: 1})]
    pod = _pod(prio=10, res={R8[2]: 1, R8[5]: 1, R8[7]: 1, **{R8[i]: 0 for i in (1, 3, 4, 6)}})
    assert sorted(r[nm] for nm, q in pod["res"].items() if q) == [2, 5, 7]
    out.append(_preempt("scalar: R = 8, requests r2, r5, r7", "scalar", nodes, bound, [pod, dict(pod, priority=4)],
                        ["no-zero-skip", "zero-left-scalar"], names=R8))
    return out


# -------------------------------------------------------------------------------------------------- drain builders
def _dnode(cpu=8000, mem=8 << 30, labels=None, taints=None, alloc=None):
    return dict(cpu=cpu, mem=mem, labels=labels or {"zone": "a"}, taints=taints or [], alloc=alloc or {"pods": 110})


def _dpod(cpu=1000, mem=1 << 20, group=-1, res=None, sel=None):
    return dict(cpu=cpu, mem=mem, selector=sel or {}, group=group, res=res or {})


def _drain(name, family, nodes, bound, cands, kills, rules=(), names=None, runs=RUNS, **notes):
    d = fdo.cluster(nodes, bound, cands, names)
    d["group_rules"] = list(rules)
    return Case(name, "drain", d, tuple(kills), runs=runs, family=family, notes=notes)


TAINT = {"key": "example.com/t", "value": "", "effect": "NoSchedule"}
TOLERATE = {"key": "example.com/t", "operator": "Exists", "effect": "NoSchedule"}
ZONE_A = {"required": [[{"key": "zone", "operator": "In", "values": ["a"]}]]}


def drain_cases():
    out = []
    X = "example.com/x"
    # Candidate 0 drains node 0: pod 0 (tolerates the taint, 2 of x) has one destination, node 1 (tainted, x = 2),
    # which it leaves at exactly 0 of x; pod 1 (no toleration, zone a required, 1 of x) then fails node 1 on x first
    # (word 1, not 2), node 2 on x (0), node 3 on the taint, node 4 on its zone, node 5 on cpu: refused [1, 2, 1, 1].
    # Candidate 1 drains node 5 (with exclusion node 0 is no destination of candidate 0 either way, and node 5 none of
    # candidate 0).
    nodes = [_dnode(alloc={"pods": 110}), _dnode(taints=[TAINT], alloc={"pods": 110, X: 2}),
             _dnode(alloc={"pods": 110}), _dnode(taints=[TAINT], alloc={"pods": 110, X: 1}),
             _dnode(labels={"zone": "c"}, alloc={"pods": 110, X: 1}), _dnode(cpu=500, alloc={"pods": 110})]
    cands = [(0, [_dpod(group=0, res={X: 2}), _dpod(group=1, res={X: 1})]), (5, [_dpod(cpu=100)])]
    out.append(_drain("drain: x to 0, then refusal word 1", "scalar", nodes, [], cands,
                      ["drain-taint-first", "drain-keeps-scalar"], rules=[{"tolerations": [TOLERATE]}, ZONE_A],
                      names=["pods", X], want_refused=[1, 2, 1, 1]))
    # The pod count to exactly 0: node 1 (2 of 4 pod slots taken) is the only destination with room for 2,000 cpu;
    # the candidate's second pod takes its last slot in the overlay, and the third finds none (word 1 on node 1, word 0
    # elsewhere)
    nodes = [_dnode(), _dnode(alloc={"pods": 4}), _dnode(cpu=1000), _dnode(cpu=1000)]
    bound = [(1, 0, 0, {}), (1, 0, 0, {})]
    out.append(_drain("drain: pods to 0, then refusal word 1", "scalar", nodes, bound,
                      [(0, [_dpod(cpu=2000) for _ in range(3)])], ["drain-keeps-pod-count", "zero-left-pods"],
                      names=["pods"]))
    # A zero request of x on a destination whose x is -2 (a pod there holds 3 of 1): node 1 is the only one with room
    nodes = [_dnode(), _dnode(alloc={"pods": 110, X: 1}), _dnode(cpu=500), _dnode(cpu=500, alloc={"pods": 110, X: 5})]
    bound = [(1, 0, 0, {X: 3})]
    out.append(_drain("drain: zero request, negative free", "scalar", nodes, bound,
                      [(0, [_dpod(cpu=4000, res={X: 0})]), (3, [_dpod(cpu=4000, res={X: 0})])], ["no-zero-skip"],
                      names=["pods", X]))
    # R = 8 with requests r2, r5 and r7 and the other columns negative; the overlay leaves r5 at exactly 0 on node 1
    neg = {R8[i]: 0 for i in (1, 3, 4, 6)}
    hold = {R8[i]: 1 for i in (1, 3, 4, 6)}
    nodes = [_dnode(alloc={"pods": 110, **neg}), _dnode(alloc={"pods": 110, **neg, R8[2]: 3, R8[5]: 2, R8[7]: 3}),
             _dnode(alloc={"pods": 110, **neg, R8[2]: 3, R8[5]: 1, R8[7]: 3}), _dnode(alloc={"pods": 110, **neg})]
    bound = [(n, 0, 0, dict(hold)) for n in range(4)]
    pod = _dpod(cpu=0, mem=0, res={R8[2]: 1, R8[5]: 1, R8[7]: 1, **{R8[i]: 0 for i in (1, 3, 4, 6)}})
    out.append(_drain("drain: R = 8, requests r2, r5, r7", "scalar", nodes, bound, [(0, [dict(pod) for _ in range(4)])],
                      ["no-zero-skip", "drain-keeps-scalar", "zero-left-scalar"], names=R8))
    # Ties: identical destinations, every pick the lowest index the overlay leaves level
    nodes = [_dnode() for _ in range(6)]
    out.append(_drain("drain: ties to the lower index", "tie", nodes, [],
                      [(0, [_dpod(cpu=0, mem=0) for _ in range(3)]), (5, [_dpod(cpu=8000)] * 2)],
                      ["drain-ties-high"], names=["pods"]))
    return out


def drain_geometry_case(sms, D=6):
    """ks_fit_drain_check on the grid of geometry (a): D candidates over 2 sms + 1 tiles, chunks of 2 tiles and a short
    last one.  x (one unit) exists only on the nodes on both sides of every tile boundary and on N - 1; every pod asks 1
    of x and no cpu or memory, so every score ties and each pick is the lowest-index node with x left in the candidate's
    overlay.  Candidate 0 has more pods than x nodes and stops (refusal word 1 counts every node); the others drain a few
    pods from x nodes, so exclusion moves the picks."""
    _, N = geometry_shape("a", sms)
    X = "example.com/x"
    nodes = [_dnode(labels={}) for _ in range(N)]
    xs = sorted({N - 1} | {n for _, l, r in tile_pairs(N) for n in (l, r)})
    for n in xs:
        nodes[n]["alloc"] = {"pods": 110, X: 1}
    pod = _dpod(cpu=0, mem=0, res={X: 1})
    cands = [(0, [dict(pod) for _ in range(len(xs) + 1)])]
    cands += [(xs[(7 * i) % len(xs)], [dict(pod) for _ in range(3 + i)]) for i in range(1, D)]
    case = _drain(f"drain geometry sms={sms} N={N}", "geometry", nodes, [], cands, ["drain-ties-high",
                  "drain-keeps-scalar"], names=["pods", X], runs=((0, 0), (0, 1)), xs=xs)
    case.geometry = ("a", sms)
    return case


# ----------------------------------------------------------------------------------------------------- case lists
def cpu_cases():
    """Every case whose claims test_fit_edges.py checks without an SM count"""
    return key_cases() + walk_cases() + preempt_scalar_cases() + drain_cases()
