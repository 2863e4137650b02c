"""CPU restatement of ks_select_topk's ranked lists for the tests, built on the oracle's own entry points: which cells are
feasible comes from the cell codes of orc_run_packed / orc_run_faithful, and the scores from the oracle's score
definitions (the faithful form calls orc_score_cell per feasible cell; the packed form restates orc_run_packed's int64
expressions in numpy, and the tests check its entry 0 against orc_run_packed's argmax).  Rows are ranked by score
descending, ties to the lower node index; slots past the feasible count hold node -1 and score 0."""
import numpy as np


def _ranked(rows, k):
    """rows[p] = (feasible node indices ascending, their scores) -> (node_idx [P,k], score [P,k], feasible_cnt [P])."""
    P = len(rows)
    idx = np.full((P, k), -1, np.int32)
    score = np.zeros((P, k), np.int64)
    cnt = np.zeros(P, np.uint32)
    for p, (n, s) in enumerate(rows):
        cnt[p] = len(n)
        order = np.lexsort((n, -s))[:k]  # primary key: score descending; then node index ascending
        idx[p, :len(order)] = n[order]
        score[p, :len(order)] = s[order]
    return idx, score, cnt


def packed_scores(policy, fc, fm, ac, am, rc, rm):
    """Scores of feasible cells (one pod, nodes given by the arrays) as orc_run_packed computes them.  Inside the limits
    of ksched.h nothing overflows int64, and on a feasible cell free - req >= 0, so floor division is C's division."""
    if policy == 0:  # ORC_SCORE_LEFTOVER
        return (fc - rc) * np.int64(1 << 22) + (fm - rm)
    pc = np.where(ac > 0, ((fc - rc) * 100) // np.where(ac > 0, ac, 1), 0)
    pm = np.where(am > 0, ((fm - rm) * 100) // np.where(am > 0, am, 1), 0)
    return (pc + pm) // 2


def topk_packed(orc, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, k, policy=0):
    """Packed form (cpu millicores, memory bytes, label words); free_* after the bound-pod subtraction."""
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    rc, rm = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
    codes = orc.run_packed(fc, fm, ac, am, labels, rc, rm, sel, policy=policy, want_mask=False, want_codes=True)[4]
    rows = []
    for p in range(len(rc)):
        n = np.nonzero(codes[p] == 0)[0]  # ORC_CELL_OK
        rows.append((n, packed_scores(policy, fc[n], fm[n], ac[n], am[n], rc[p], rm[p])))
    return _ranked(rows, k)


def topk_faithful(orc, cluster, pods, n_pods, k, policy=0):
    """Object form on an orc.Cluster: feasibility from orc_check_node_validity, every score from orc_score_cell."""
    codes = cluster.run(pods, n_pods, policy=policy, want_mask=False, want_codes=True)[4]
    rows = []
    for p in range(n_pods):
        n = np.nonzero(codes[p] == 0)[0]
        s = np.empty(len(n), np.int64)
        for j, node in enumerate(n):
            rc, s[j] = cluster.score(policy, pods, p, int(node))
            assert rc == 0, rc
        rows.append((n, s))
    return _ranked(rows, k)
