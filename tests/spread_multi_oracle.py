"""CPU restatement of topology-spread replica placement over several keys (ks_place_replicas_spread_multi,
include/ksched.h; DESIGN.md 5l).

spread_multi_packed places one copy at a time in numpy, exactly as the header defines it: c_n from
replicas_oracle.node_copies, s_n(j) from spread_oracle.scores_at, and every key's skew rule at once.  It returns (rows
[T, K], node, score, offset, counts) as Snapshot.place_replicas_spread_multi does, counts a list of K arrays [T, D_k]."""
import numpy as np

from replicas_oracle import _specs, node_copies
from spread_oracle import INT64_MIN, SPREAD_PLAN_DTYPE, scores_at


def spread_multi_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, replicas, keys,
                        max_skew, min_domains=None, existing=None, policy=0):
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    N, T, K = fc.shape[0], len(req_cpu), len(keys)
    labels, sel = _specs(labels, sel, N, T)
    dom = [np.asarray(d, np.int64).reshape(N) for d, _ in keys]
    D = [int(n) for _, n in keys]
    skew = np.asarray(max_skew, np.int64).reshape(T, K)
    mind = np.zeros((T, K), np.int64) if min_domains is None else np.asarray(min_domains, np.int64).reshape(T, K)
    ex = [np.zeros((T, d), np.int64) if existing is None else np.asarray(existing[k], np.int64).reshape(T, d)
          for k, d in enumerate(D)]
    offset = np.zeros(T + 1, np.uint64)
    np.cumsum(np.asarray(replicas, np.uint64), out=offset[1:])
    rows = np.zeros((T, K), SPREAD_PLAN_DTYPE)
    node = np.full(int(offset[-1]), -1, np.int32)
    score = np.zeros(int(offset[-1]), np.int64)
    counts = [np.zeros((T, d), np.uint32) for d in D]
    has_all = np.ones(N, bool)
    for d in dom:
        has_all &= d >= 0
    dn = [np.where(d >= 0, d, 0) for d in dom]
    for t in range(T):
        rc, rm, R, o = int(req_cpu[t]), int(req_mem[t]), int(replicas[t]), int(offset[t])
        c, _ = node_copies(fc, fm, labels, rc, rm, sel[t])
        k_n = np.where(c < 0, R, np.minimum(c, R))
        # 1. eligible: every key, and the selector matches; resource fit plays no part
        eligible = has_all & ((sel[t][None, :] & ~labels) == 0).all(axis=1)
        in_e = []
        for k in range(K):
            e = np.zeros(D[k], bool)
            e[dom[k][eligible]] = True
            in_e.append(e)
        ne = [int(e.sum()) for e in in_e]
        # 2. counts, 3. each key's minimum (0 under minDomains)
        cnt = [ex[k][t].copy() for k in range(K)]
        forced = [ne[k] < int(mind[t, k]) for k in range(K)]
        m = [0 if ne[k] == 0 or forced[k] else int(cnt[k][in_e[k]].min()) for k in range(K)]

        def admits(k):  # key k's rule, per node (its domain's count within max_skew of m_k)
            return (cnt[k] + 1 - m[k] <= skew[t, k])[dn[k]]

        j = np.zeros(N, np.int64)
        cur = np.where(k_n > 0, scores_at(fc, fm, ac, am, rc, rm, np.zeros(N, np.int64), policy), INT64_MIN)
        r = 0
        while eligible.any() and r < R:  # 4. one copy at a time
            cand = eligible & (j < k_n)
            for k in range(K):
                cand &= admits(k)
            if not cand.any():
                break
            s = np.where(cand, cur, INT64_MIN)
            n = int(s.argmax())  # first maximum: ties to the lower node index
            node[o + r], score[o + r] = n, s[n]
            j[n] += 1
            for k in range(K):
                cnt[k][dom[k][n]] += 1
            if j[n] < k_n[n]:
                cur[n] = scores_at(fc[n:n + 1], fm[n:n + 1], ac[n:n + 1], am[n:n + 1], rc, rm, j[n:n + 1], policy)[0]
            for k in range(K):
                if not forced[k]:
                    m[k] = int(cnt[k][in_e[k]].min())
            r += 1
        # 5. the rows
        room = eligible & (j < k_n)
        ok = [admits(k) for k in range(K)]
        for k in range(K):
            row = rows[t, k]
            row["placed"], row["eligible_domains"], row["min_count"], row["blocked_domain"] = r, ne[k], m[k], -1
            if r:
                row["nodes"], row["max_per_node"], row["last_score"] = int((j > 0).sum()), int(j.max()), score[o + r - 1]
            if r < R:
                others = room.copy()
                for k2 in range(K):
                    if k2 != k:
                        others &= ok[k2]
                has_room = np.zeros(D[k], bool)
                has_room[dom[k][others]] = True
                own = in_e[k] & (cnt[k] + 1 - m[k] <= skew[t, k])
                blocked = np.nonzero(own & ~has_room)[0]
                if len(blocked):
                    row["blocked_domain"] = blocked[0]
            counts[k][t] = cnt[k]
    return rows, node, score, offset, counts
