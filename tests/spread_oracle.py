"""CPU restatement of topology-spread replica placement (ks_place_replicas_spread, include/ksched.h; DESIGN.md 5k).

spread_packed places one copy at a time in numpy over a private per-node copy count: c_n from
replicas_oracle.node_copies, s_n(j) from replicas_oracle.copy_scores (policies 0 and 1) or policy_oracle.SCORES (3 and
4), and the domain rule restated from the header's definition.  It returns (rows, node, score, offset, counts) as
Snapshot.place_replicas_spread does."""
import numpy as np

from policy_oracle import SCORES
from replicas_oracle import _specs, copy_scores, node_copies

INT64_MIN = np.iinfo(np.int64).min
SPREAD_PLAN_DTYPE = np.dtype([("placed", np.uint32), ("nodes", np.uint32), ("max_per_node", np.uint32),
                              ("eligible_domains", np.uint32), ("min_count", np.uint32), ("blocked_domain", np.int32),
                              ("last_score", np.int64)])


def scores_at(fc, fm, ac, am, rc, rm, j, policy):
    """s_n(j) on arrays: the spec's score on node n with j copies already bound there."""
    if policy in (0, 1):
        return copy_scores(fc, fm, ac, am, rc, rm, j, policy)
    return SCORES[policy](fc - j * rc, fm - j * rm, ac, am, rc, rm)


def spread_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, replicas, node_domain,
                  n_domains, max_skew, min_domains=None, existing=None, policy=0):
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    N, T, D = fc.shape[0], len(req_cpu), int(n_domains)
    labels, sel = _specs(labels, sel, N, T)
    dom = np.asarray(node_domain, np.int64).reshape(N)
    ex = np.zeros((T, D), np.int64) if existing is None else np.asarray(existing, np.int64).reshape(T, D)
    offset = np.zeros(T + 1, np.uint64)
    np.cumsum(np.asarray(replicas, np.uint64), out=offset[1:])
    rows = np.zeros(T, SPREAD_PLAN_DTYPE)
    node = np.full(int(offset[-1]), -1, np.int32)
    score = np.zeros(int(offset[-1]), np.int64)
    counts = np.zeros((T, D), np.uint32)
    for t in range(T):
        rc, rm, R, o, skew = int(req_cpu[t]), int(req_mem[t]), int(replicas[t]), int(offset[t]), int(max_skew[t])
        mind = 0 if min_domains is None else int(min_domains[t])
        c, _ = node_copies(fc, fm, labels, rc, rm, sel[t])
        k = np.where(c < 0, R, np.minimum(c, R))
        # 1. eligible nodes and domains: a domain, and the selector matches; resource fit plays no part
        eligible = (dom >= 0) & ((sel[t][None, :] & ~labels) == 0).all(axis=1)
        in_e = np.zeros(D, bool)
        in_e[dom[eligible]] = True
        ne = int(in_e.sum())
        # 2. counts, 3. the global minimum (0 under minDomains when fewer domains are eligible)
        cnt = ex[t].copy()
        forced = ne < mind
        m = 0 if ne == 0 or forced else int(cnt[in_e].min())
        j = np.zeros(N, np.int64)
        cur = np.where(k > 0, scores_at(fc, fm, ac, am, rc, rm, np.zeros(N, np.int64), policy), INT64_MIN)
        dn = np.where(dom >= 0, dom, 0)
        r = 0
        while ne and r < R:  # 4. one copy at a time
            admitted = in_e & (cnt + 1 - m <= skew)
            cand = eligible & (j < k) & admitted[dn]
            if not cand.any():
                break
            s = np.where(cand, cur, INT64_MIN)
            n = int(s.argmax())  # first maximum: ties to the lower node index
            node[o + r], score[o + r] = n, s[n]
            j[n] += 1
            cnt[dom[n]] += 1
            if j[n] < k[n]:
                cur[n] = scores_at(fc[n:n + 1], fm[n:n + 1], ac[n:n + 1], am[n:n + 1], rc, rm, j[n:n + 1], policy)[0]
            if not forced:
                m = int(cnt[in_e].min())
            r += 1
        # 5. the row
        row = rows[t]
        row["placed"], row["eligible_domains"], row["min_count"], row["blocked_domain"] = r, ne, m, -1
        if r:
            row["nodes"], row["max_per_node"], row["last_score"] = int((j > 0).sum()), int(j.max()), score[o + r - 1]
        if r < R:
            admitted = in_e & (cnt + 1 - m <= skew)
            room = np.zeros(D, bool)
            room[dom[eligible & (j < k)]] = True
            blocked = np.nonzero(admitted & ~room)[0]
            if len(blocked):
                row["blocked_domain"] = blocked[0]
        counts[t] = cnt
    return rows, node, score, offset, counts
