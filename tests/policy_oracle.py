"""CPU restatement of the score policies the oracle library does not have, for the tests: KS_SCORE_MOST_ALLOCATED (3,
bin-packing) and KS_SCORE_LEAST_BALANCED (4, upstream's default resource scoring), as include/ksched.h defines them.

The oracle library scores LEFTOVER and LEAST_ALLOCATED only, so this module adds the two on top of it: which cells are
feasible (and the mask and counts) still come from orc_run_packed's cell codes, and the scores from the definitions
below (`SCORE`: Python integers, `SCORES`: numpy).  `Oracle(orc)` has orc's run_packed / stream_bind_packed /
commit_claims / free_reduce and accepts policies 3 and 4, so the existing restatements (gang_oracle, drain_oracle,
replicas_oracle.sequential_packed) run under them unchanged.  The replica plans restate the library's two algorithms:
`prefix_fill_packed` (policy 3: nodes filled whole, one after another, in order of copy 0's score descending, node
ascending) and `heap_packed` (policy 4: one copy at a time, with a heap instead of one full select per copy).

LEAST_BALANCED's balanced term is defined in IEEE double arithmetic: each operand is converted with float() (round to
nearest even, as CUDA's __ll2double_rn) before one true division, and every later step is one rounded double operation.
Python's `u / A` on two ints rounds the exact quotient once instead, which differs above 2^53: the helpers below never
use it."""
import heapq

import numpy as np

from replicas_oracle import PLAN_DTYPE, _row, _specs, node_copies

MOST_ALLOCATED = 3
LEAST_BALANCED = 4


# ---- KS_SCORE_MOST_ALLOCATED ----
def term(f, a, q):
    """One resource, Python integers: clamp(A - (f - q), 0, A) * 100 / A, 0 for A <= 0."""
    if a <= 0:
        return 0
    return min(max(a - (f - q), 0), a) * 100 // a


def most_score(fc, fm, ac, am, rc, rm):
    return (term(int(fc), int(ac), int(rc)) + term(int(fm), int(am), int(rm))) // 2


def most_scores(fc, fm, ac, am, rc, rm):
    """The same on int64 arrays (broadcasting); inside the limits of ksched.h nothing overflows."""
    def t(f, a, q):
        pos = a > 0
        u = np.clip(a - (f - q), 0, np.where(pos, a, 0))
        return np.where(pos, (u * 100) // np.where(pos, a, 1), 0)
    return (t(fc, ac, rc) + t(fm, am, rm)) // 2


# ---- KS_SCORE_LEAST_BALANCED ----
def least(fc, fm, ac, am, rc, rm):
    """KS_SCORE_LEAST_ALLOCATED on Python ints: truncating divisions, as the C expression."""
    def t(f, q, a):
        if a <= 0:
            return 0
        x = (f - q) * 100
        return abs(x) // a * (1 if x >= 0 else -1)
    s = t(int(fc), int(rc), int(ac)) + t(int(fm), int(rm), int(am))
    return abs(s) // 2 * (1 if s >= 0 else -1)


def balanced(fc, fm, ac, am, rc, rm):
    """The balanced term on Python ints and floats, one rounded double operation per step."""
    fc, fm, ac, am, rc, rm = (int(v) for v in (fc, fm, ac, am, rc, rm))
    if ac <= 0 or am <= 0:
        return 100
    uc = min(max(ac - (fc - rc), 0), ac)
    um = min(max(am - (fm - rm), 0), am)
    xc = float(uc) / float(ac)
    xm = float(um) / float(am)
    sd = abs(xc - xm) / 2.0
    return int((1.0 - sd) * 100.0)  # int() truncates toward zero; the value is >= 50


def balanced_score(fc, fm, ac, am, rc, rm):
    return least(fc, fm, ac, am, rc, rm) + balanced(fc, fm, ac, am, rc, rm)


def balanced_scores(fc, fm, ac, am, rc, rm):
    """The same on int64 arrays (broadcasting).  numpy's int64 -> float64 cast rounds to nearest even and its float64
    operations are single IEEE operations, so this is bit for bit the scalar form; inside the limits of ksched.h nothing
    overflows."""
    fc, fm, ac, am, rc, rm = np.broadcast_arrays(*(np.asarray(v, np.int64) for v in (fc, fm, ac, am, rc, rm)))

    def pct(f, q, a):  # truncating (f - q) * 100 / a, 0 for a <= 0
        pos = a > 0
        x = (f - q) * 100
        d = np.where(pos, a, 1)
        return np.where(pos, np.sign(x) * (np.abs(x) // d), 0)

    s = pct(fc, rc, ac) + pct(fm, rm, am)
    lst = np.sign(s) * (np.abs(s) // 2)
    both = (ac > 0) & (am > 0)
    a_c, a_m = np.where(ac > 0, ac, 1), np.where(am > 0, am, 1)
    uc = np.clip(ac - (fc - rc), 0, np.maximum(ac, 0))
    um = np.clip(am - (fm - rm), 0, np.maximum(am, 0))
    with np.errstate(all="ignore"):
        xc = uc.astype(np.float64) / a_c.astype(np.float64)
        xm = um.astype(np.float64) / a_m.astype(np.float64)
        sd = np.abs(xc - xm) / 2.0
        bal = ((1.0 - sd) * 100.0).astype(np.int64)  # truncation toward zero
    return lst + np.where(both, bal, 100)


SCORE = {MOST_ALLOCATED: most_score, LEAST_BALANCED: balanced_score}
SCORES = {MOST_ALLOCATED: most_scores, LEAST_BALANCED: balanced_scores}


# ---- LEAST_BALANCED's bit-parallel walk bound (ks_bitpar.cu, DESIGN.md 5j), restated for the bound tests ----
def node_bound(fc, fm, ac, am):
    """b(n) = least_alloc_bound(n) + bal(n), unclamped."""
    b = least(fc, fm, ac, am, 0, 0)
    if ac <= 0 or am <= 0:
        return b + 100
    d = abs(term(fc, ac, 0) - term(fm, am, 0))
    return b + 100 - (max(d - 1, 0) // 2)


def slack(q, m):
    """min(100, ceil(q * 100 / m)) for q >= 0, m > 0."""
    x = q * 100
    return min(100, x // m + (1 if x % m else 0))


def pod_slack(rc, rm, amax_c, amax_m, amin_c, amin_m):
    """D - E: every feasible cell of the pod scores <= b(n) - (D - E).  amax = max allocatable (INT64_MAX when some node
    has none), amin = smallest positive allocatable (INT64_MAX when none)."""
    dl = ((rc * 100) // amax_c + (rm * 100) // amax_m) // 2
    e = (max(slack(rc, amin_c), slack(rm, amin_m)) + 1) // 2
    return dl - e


# ---- the bit-parallel walk of both policies (bound_walk in ks_bitpar.cu, DESIGN.md 5i / 5j), restated ----
I64_MAX = (1 << 63) - 1
LB_UNBOUNDED = 1 << 62  # LEAST_BALANCED's stored bound above 200
TILE, FIRST_WINDOW, WINDOW = 256, 8, 32


def most_bound(fc, fm, ac, am):
    """MOST_ALLOCATED's b(n) = term(f_c, A_c, 0) + term(f_m, A_m, 0), in [0, 200]."""
    return term(int(fc), int(ac), 0) + term(int(fm), int(am), 0)


def most_slack(rc, rm, amin_c, amin_m):
    """MOST_ALLOCATED's D: every feasible cell of a pod with requests >= 0 scores <= (b(n) + D) // 2."""
    return slack(rc, amin_c) + slack(rm, amin_m)


def stored_bound(policy, fc, fm, ac, am):
    """The bound the walk's order stores for a node: MOST_ALLOCATED's b(n); LEAST_BALANCED's b(n) as k_balanced_order
    stores it, LB_UNBOUNDED above 200 and 0 below 0."""
    if policy == MOST_ALLOCATED:
        return most_bound(fc, fm, ac, am)
    b = node_bound(int(fc), int(fm), int(ac), int(am))
    return LB_UNBOUNDED if b > 200 else max(b, 0)


def walk_limit(policy, top, d):
    """The highest score a feasible cell in a slot of bound `top' can have: (top + D) / 2 or top - D (C division)."""
    if policy == MOST_ALLOCATED:
        x = top + d
        return abs(x) // 2 * (1 if x >= 0 else -1)
    return top - d


def walk_packed(oracle, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, policy, margin=0):
    """k_most_alloc / k_least_balanced's control flow, not only its result: nodes in descending stored bound (ties to
    the lower index), tiles of 256 slots in windows of 8 then 32 tiles, the exit test `best > limit(top) + margin' in
    front of each window (from the second on) and in front of each tile with a feasible slot, no exit for a negative
    request, an immediate -1 for a pod that fits nowhere by rank or selector.  margin shifts the exit limit (-1: an exit
    one step too early) so that a test can show its cases would catch that.  Feasibility comes from the oracle's cell
    codes.  Returns (node, score, scored, exit): per pod the tiles it scored and the tile in front of which it stopped
    (-1: it walked to the end)."""
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    rc, rm = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
    N, P = fc.shape[0], rc.shape[0]
    lab = np.ascontiguousarray(labels, np.uint64).reshape(N, -1)
    sel = np.ascontiguousarray(sel, np.uint64).reshape(P, -1)
    codes = oracle.orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, 0, want_mask=False, want_codes=True)[4]
    bound = np.array([stored_bound(policy, *v) for v in zip(fc, fm, ac, am)], np.int64)
    order = np.lexsort((np.arange(N), -bound))
    top = bound[order]
    n_tiles = (N + TILE - 1) // TILE
    amax_c = I64_MAX if (ac <= 0).any() else int(ac.max())  # k_node_bound: a node with A <= 0 gives no slack
    amax_m = I64_MAX if (am <= 0).any() else int(am.max())
    amin_c = int(ac[ac > 0].min()) if (ac > 0).any() else I64_MAX
    amin_m = int(am[am > 0].min()) if (am > 0).any() else I64_MAX
    live = np.bitwise_or.reduce(lab, axis=0) if N else np.zeros(lab.shape[1], np.uint64)
    score = SCORES[policy]
    idx, sc = np.full(P, -1, np.int32), np.zeros(P, np.int64)
    scored, exits = [], np.full(P, -1, np.int64)
    for p in range(P):
        q_c, q_m = int(rc[p]), int(rm[p])
        seen = []
        scored.append(seen)
        if N == 0 or q_c > fc.max() or q_m > fm.max() or (sel[p] & ~live).any():
            continue  # dead: k_pod_ranks' rank is N, or a required pair no node carries
        bounded = q_c >= 0 and q_m >= 0
        if not bounded:
            d = 0
        elif policy == MOST_ALLOCATED:
            d = most_slack(q_c, q_m, amin_c, amin_m)
        else:
            d = pod_slack(q_c, q_m, amax_c, amax_m, amin_c, amin_m)
        feas = codes[p][order] == 0
        best, bidx = 0, -1

        def stop(k):
            return bounded and bidx >= 0 and best > walk_limit(policy, int(top[k * TILE]), d) + margin

        k0, win = 0, FIRST_WINDOW
        while exits[p] < 0 and k0 < n_tiles:
            if k0 > 0 and stop(k0):
                exits[p] = k0
                break
            for k in range(k0, min(k0 + win, n_tiles)):
                f = np.nonzero(feas[k * TILE:(k + 1) * TILE])[0] + k * TILE
                if not len(f):
                    continue
                if stop(k):
                    exits[p] = k
                    break
                seen.append(k)
                n = order[f]
                s = score(fc[n], fm[n], ac[n], am[n], q_c, q_m)
                j = np.lexsort((n, -s))[0]
                if bidx < 0 or s[j] > best or (s[j] == best and n[j] < bidx):
                    best, bidx = int(s[j]), int(n[j])
            k0 += win
            win = WINDOW
        idx[p], sc[p] = bidx, best if bidx >= 0 else 0
    return idx, sc, scored, exits


# ---- clusters that put the winner exactly at an exit of the walk ----
# Per policy, three node profiles as (share of cpu, share of memory) in percent, on allocatables of 100 and 100 MiB so
# that every share is exact, for zero-request pods (D = 0, the bound is attained): X, Y with X one bound above Y and
# the same score, and Y' one score below X.  MOST_ALLOCATED: b = 2k + 1 and 2k both score k.  LEAST_BALANCED: shares
# 40 / 41 give b = 159 and score 158 (|P_c - P_m| = 1: bal = 100, balanced = trunc(99.5)); equal shares 42 score
# their bound 158.  `before' nodes bound above X, `after' nodes below Y and Y'.
EDGE_PROFILES = {
    MOST_ALLOCATED: dict(x=(61, 60), y=(60, 60), y_low=(60, 59), before=(100, 100), after=(0, 0)),
    LEAST_BALANCED: dict(x=(40, 41), y=(42, 42), y_low=(43, 43), before=(0, 0), after=(100, 100)),
}
EDGE_A_CPU, EDGE_A_MEM = 100, 100 << 20
EDGE_BIT = 1 << 5  # the label every pod requires: X, Y and the nodes after them carry it, the nodes before do not
# boundary -> (tile of X, tile of Y, number of tiles; Y sits at the first slot of its tile unless both share one).
# "inside one tile" has no exit test between X and Y: the tie is the tile merge's; tiles 0/1 and 20/21 are exits inside
# a window, 7/8 (also a column-block edge), 39/40 and 71/72 the exits in front of a window.
EDGES = {"inside one tile": (3, 3, 6), "tile 0/1": (0, 1, 3), "tile 7/8": (7, 8, 10), "tile 20/21": (20, 21, 24),
         "tile 39/40": (39, 40, 42), "tile 71/72": (71, 72, 74), "last tile": (76, 77, 78)}


def exit_tie_cluster(policy, edge, mirror=False, seed=0):
    """A packed cluster (fc, fm, ac, am, labels, rc, rm, sel) in which X lies in front of the boundary `edge' and Y
    right after it in bound order, Y at a lower node index than X.  Tie (mirror False): Y scores as X and the limit of
    its tile, so Y must win.  Mirror: Y scores one lower, the walk stops in front of Y's tile and X wins.  Two
    zero-request pods require EDGE_BIT, the second also a pair on the second label word.  Returns the cluster and the
    node indices of X and Y."""
    tx, ty, n_tiles = EDGES[edge]
    prof = EDGE_PROFILES[policy]
    sx = ty * TILE - 1 if tx != ty else tx * TILE + 100  # slots in bound order
    N = (n_tiles - 1) * TILE + 37  # the last tile is a partial one
    rng = np.random.default_rng(seed)
    shares = [prof["before"]] * sx + [prof["x"], prof["y_low"] if mirror else prof["y"]]
    shares += [prof["after"]] * (N - len(shares))
    perm = rng.permutation(N)  # slot -> node index, Y below X
    if perm[sx + 1] > perm[sx]:
        perm[sx], perm[sx + 1] = perm[sx + 1], perm[sx]
    u = np.zeros((N, 2), np.int64)
    u[perm] = np.array(shares, np.int64)
    ac, am = np.full(N, EDGE_A_CPU, np.int64), np.full(N, EDGE_A_MEM, np.int64)
    fc, fm = ac - u[:, 0], am - (u[:, 1] << 20)
    lab = np.zeros((N, 2), np.uint64)
    lab[:, 1] = rng.integers(0, 1 << 16, N).astype(np.uint64)
    lab[perm[sx:], 0] = EDGE_BIT
    lab[perm[sx:], 1] |= np.uint64(1)
    sel = np.array([[EDGE_BIT, 0], [EDGE_BIT, 1]], np.uint64)
    z = np.zeros(2, np.int64)
    return (fc, fm, ac, am, lab, z, z.copy(), sel), int(perm[sx]), int(perm[sx + 1])


class Oracle:
    """orc with policies 3 and 4 added to run_packed and stream_bind_packed."""

    def __init__(self, orc):
        self.orc = orc

    def __getattr__(self, name):
        return getattr(self.orc, name)

    def run_packed(self, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, policy=0,
                   want_mask=True, want_codes=False, nthreads=0):
        if policy not in SCORES:
            return self.orc.run_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, policy,
                                       want_mask, want_codes, nthreads)
        _, _, cnt, mask, codes = self.orc.run_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem,
                                                     sel, 0, want_mask, True, nthreads)
        fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
        ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
        rc, rm = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
        P = rc.shape[0]
        idx = np.full(P, -1, np.int32)
        sc = np.zeros(P, np.int64)
        INF = np.iinfo(np.int64).min
        for p0 in range(0, P, 512):  # bounded memory for large P
            p1 = min(P, p0 + 512)
            if not fc.shape[0]:
                break
            s = SCORES[policy](fc[None, :], fm[None, :], ac[None, :], am[None, :], rc[p0:p1, None], rm[p0:p1, None])
            s = np.where(codes[p0:p1] == 0, s, INF)
            best = s.argmax(axis=1)  # first maximum: ties to the lowest node index
            bs = s[np.arange(p1 - p0), best]
            ok = bs != INF
            idx[p0:p1][ok] = best[ok]
            sc[p0:p1][ok] = bs[ok]
        return idx, sc, cnt, mask, codes if want_codes else None

    def stream_bind_packed(self, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, policy=0):
        """orc_stream_bind_packed's round loop: select the pending pods, commit the claims per node in arrival order,
        losers retry; in place on free_cpu / free_mem."""
        if policy not in SCORES:
            return self.orc.stream_bind_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel,
                                               policy)
        P = len(req_cpu)
        rc, rm = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
        sel = np.ascontiguousarray(sel, np.uint64).reshape(P, -1)
        idx = np.full(P, -1, np.int32)
        sc = np.zeros(P, np.int64)
        pending = np.arange(P)
        rounds = 0
        while len(pending) and rounds <= P + 1:
            i, s = self.run_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, rc[pending], rm[pending],
                                   sel[pending], policy, want_mask=False)[:2]
            acc = self.orc.commit_claims(free_cpu, free_mem, i, rc[pending], rm[pending])
            won = (i >= 0) & (acc != 0)
            idx[pending[won]], sc[pending[won]] = i[won], s[won]
            pending = pending[(i >= 0) & (acc == 0)]
            rounds += 1
        return idx, sc, rounds


def topk_packed(oracle, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, k, policy):
    """ks_select_topk's rows under policy 3 or 4: feasible nodes by score descending, node ascending."""
    from topk_oracle import _ranked
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    rc, rm = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
    codes = oracle.orc.run_packed(fc, fm, ac, am, labels, rc, rm, sel, 0, want_mask=False, want_codes=True)[4]
    rows = []
    for p in range(len(rc)):
        n = np.nonzero(codes[p] == 0)[0]
        rows.append((n, SCORES[policy](fc[n], fm[n], ac[n], am[n], rc[p], rm[p])))
    return _ranked(rows, k)


def _plan_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, replicas, place):
    """The plan's rows, copy lists and offsets, spec by spec: place(fc, fm, ac, am, rc, rm, R, c, feas) returns spec t's
    copies in placement order as (nodes, scores), given every node's copy count c (-1: no limit) and the nodes that
    hold at least one.  Returns (rows, node, score, offset) as replicas_oracle.merge_packed does."""
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    N, T = fc.shape[0], len(req_cpu)
    labels, sel = _specs(labels, sel, N, T)
    offset = np.zeros(T + 1, np.uint64)
    np.cumsum(np.asarray(replicas, np.uint64), out=offset[1:])
    rows = np.zeros(T, PLAN_DTYPE)
    node = np.full(int(offset[-1]), -1, np.int32)
    sc = np.zeros(int(offset[-1]), np.int64)
    for t in range(T):
        rc, rm, R, o = int(req_cpu[t]), int(req_mem[t]), int(replicas[t]), int(offset[t])
        c, cap = node_copies(fc, fm, labels, rc, rm, sel[t])
        feas = np.nonzero(c != 0)[0]
        n_of, s_of = place(fc, fm, ac, am, rc, rm, R, c, feas)
        r = len(n_of)
        node[o:o + r], sc[o:o + r] = n_of, s_of
        rows[t] = _row(cap, len(feas), node[o:o + r], int(sc[o + r - 1]) if r else 0)
    return rows, node, sc, offset


def prefix_fill_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, replicas):
    """Replica placement under policy 3 without one select per copy: s_n(j) is non-decreasing in j, so the node being
    filled never loses to one not yet touched; nodes take up to c_n copies each, in order of s_n(0) descending, node
    ascending."""
    def place(fc, fm, ac, am, rc, rm, R, c, feas):
        s0 = most_scores(fc[feas], fm[feas], ac[feas], am[feas], rc, rm)
        order = feas[np.lexsort((feas, -s0))]
        cn = np.where(c[order] < 0, R, np.minimum(c[order], R))
        take = np.clip(R - (np.cumsum(cn) - cn), 0, cn)  # each node in turn takes what it holds of what is left
        n_of = np.repeat(order, take)
        j = np.arange(int(take.sum()), dtype=np.int64) - np.repeat(np.cumsum(take) - take, take)
        return n_of, most_scores(fc[n_of] - j * rc, fm[n_of] - j * rm, ac[n_of], am[n_of], rc, rm)
    return _plan_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, replicas, place)


def heap_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, replicas):
    """Replica placement under policy 4, one copy at a time: a heap of (-s_n(j), n) over the nodes that hold another
    copy; the popped node takes the copy and goes back with s_n(j + 1) while j + 1 < min(c_n, R).  Ties pop the lower
    node index, as the argmax."""
    def place(fc, fm, ac, am, rc, rm, R, c, feas):
        k = np.where(c < 0, R, np.minimum(c, R))
        s0 = balanced_scores(fc[feas], fm[feas], ac[feas], am[feas], rc, rm)
        heap = [(-int(s), int(n)) for s, n in zip(s0, feas) if k[n] > 0]
        heapq.heapify(heap)
        placed = np.zeros(fc.shape[0], np.int64)
        n_of, s_of = [], []
        while len(n_of) < R and heap:
            s, n = heapq.heappop(heap)
            n_of.append(n)
            s_of.append(-s)
            j = placed[n] = placed[n] + 1
            if j < k[n]:
                heapq.heappush(heap, (-balanced_score(fc[n] - j * rc, fm[n] - j * rm, ac[n], am[n], rc, rm), n))
        return np.array(n_of, np.int32), np.array(s_of, np.int64)
    return _plan_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, replicas, place)


PLAN = {MOST_ALLOCATED: prefix_fill_packed, LEAST_BALANCED: heap_packed}


# ---- LEAST_BALANCED: cells whose (1 - std) * 100 lies within a few ulps of an integer ----
def _chain(uc, ac, um, am, fma=False, recip=False):
    from fractions import Fraction
    if recip:
        xc, xm = float(uc) * (1.0 / float(ac)), float(um) * (1.0 / float(am))
    else:
        xc, xm = float(uc) / float(ac), float(um) / float(am)
    sd = abs(xc - xm) / 2.0
    v = float(Fraction(100) - Fraction(100) * Fraction(sd)) if fma else (1.0 - sd) * 100.0
    return int(v)


def hazard_cells(seed, n):
    """Cells (fc, fm, ac, am, rc, rm) whose exact shares differ by 2k/100, so the exact (1 - std) * 100 is the integer
    100 - k and the double evaluation lands a few ulps to either side.  Kept: the cells where contracting the last two
    steps to an FMA or dividing by a reciprocal would change the truncated result, and as many where neither would.
    Returns the arrays and the number of distinguishing cells."""
    rng = np.random.default_rng(seed)
    hit, calm = [], []
    while len(hit) < n // 2 or len(calm) < n - n // 2:
        ac, am = 50 * int(rng.integers(1, 1 << 29)), 50 * int(rng.integers(1, 1 << 49))
        i = int(rng.integers(0, 51))
        k = int(rng.integers(0, i + 1))
        uc, um = ac // 50 * i, am // 50 * (i - k)
        if rng.random() < 0.5:  # the larger share on either resource
            uc, um = ac // 50 * (i - k), am // 50 * i
        fc, fm = ac - uc, am - um  # u = A - (f - q) with q = 0: free = A - u
        q_c = int(rng.integers(0, 1 << 20)) if rng.random() < 0.3 else 0
        fc += q_c  # the same u with a request: f - q unchanged
        b = _chain(uc, ac, um, am)
        distinct = b != _chain(uc, ac, um, am, fma=True) or b != _chain(uc, ac, um, am, recip=True)
        (hit if distinct else calm).append((fc, fm, ac, am, q_c, 0))
    cells = hit[:n // 2] + calm[:n - n // 2]
    return tuple(np.array(c, np.int64) for c in zip(*cells)), len(hit[:n // 2])


def walk_extreme_clusters(policy, seed=0):
    """(name, cluster) at the walk's length extremes, ~20 000 nodes (79 tiles: every window) and 160 pods:
      "last tiles only"    the selector of most pods is carried only by the 300 nodes of lowest bound: every window;
      "free above alloc"   15 % of the nodes, scattered, hold free above allocatable (LEAST_BALANCED stores them 2^62);
      "alloc <= 0"         10 % of the allocatables are 0 or negative (no LEAST_ALLOCATED slack: amax = INT64_MAX);
      "one alloc of 1"     one node has allocatables of 1: D saturates and MOST_ALLOCATED's walks are exhaustive;
      "equal allocatables" every node has the same allocatables, the tightest D."""
    rng = np.random.default_rng(seed)
    N, P = 79 * TILE - 40, 160

    def base():
        ac = rng.choice([4000, 8000, 16000, 32000, 96000], N).astype(np.int64)
        am = rng.choice([4, 16, 64, 384], N).astype(np.int64) << 30
        fc, fm = ac * rng.integers(0, 65, N) // 64, am * rng.integers(0, 65, N) // 64
        lab = rng.integers(0, 1 << 8, (N, 1)).astype(np.uint64)
        rc = rng.choice([0, 1, 100, 250, 1000, 4000], P).astype(np.int64)
        rm = rng.choice([0, 1, 1 << 27, 1 << 30, 1 << 32], P).astype(np.int64)
        sel = np.where(rng.random((P, 1)) < 0.3, np.uint64(1) << rng.integers(0, 8, (P, 1)).astype(np.uint64), 0)
        return fc, fm, ac, am, lab, rc, rm, sel.astype(np.uint64)

    fc, fm, ac, am, lab, rc, rm, sel = base()
    low = np.argsort([-stored_bound(policy, *v) for v in zip(fc, fm, ac, am)], kind="stable")[-300:]
    lab[low, 0] |= np.uint64(1 << 9)
    sel[:P - 20, 0] = 1 << 9  # the last 20 pods keep a random selector: they stop early
    yield "last tiles only", (fc, fm, ac, am, lab, rc, rm, sel)
    fc, fm, ac, am, lab, rc, rm, sel = base()
    over = rng.random(N) < 0.15
    fc[over], fm[over] = ac[over] * rng.integers(2, 5, int(over.sum())), am[over] * 3 + 7
    yield "free above alloc", (fc, fm, ac, am, lab, rc, rm, sel)
    fc, fm, ac, am, lab, rc, rm, sel = base()
    ac[rng.random(N) < 0.1] = 0
    am[rng.random(N) < 0.05] = -(1 << 20)
    yield "alloc <= 0", (fc, fm, ac, am, lab, rc, rm, sel)
    fc, fm, ac, am, lab, rc, rm, sel = base()
    n = int(rng.integers(0, N))
    ac[n], am[n], fc[n], fm[n] = 1, 1, 1, 1
    yield "one alloc of 1", (fc, fm, ac, am, lab, rc, rm, sel)
    fc, fm, ac, am, lab, rc, rm, sel = base()
    ac[:], am[:] = 16000, 64 << 30
    fc, fm = ac * rng.integers(0, 1001, N) // 1000, am * rng.integers(0, 1001, N) // 1000
    yield "equal allocatables", (fc, fm, ac, am, lab, rc, rm, sel)
