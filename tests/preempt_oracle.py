"""CPU restatement of ks_preempt (include/ksched.h, DESIGN.md 5d) for the tests, built on the oracle's own entry points:
which cells are feasible and which fail on resources comes from the cell codes of orc_run_packed, and whether a pod's
selector matches a node from the same call with every request at its lowest legal value (every node then fits, so code
2 is exactly a selector miss).  Lower sets, the reprieve walk and the node choice follow the definition, vectorised over
the nodes of one pod: visit order is priority descending, ties to the lower bound index, so a node's lower set is a
suffix of its visit list."""
import numpy as np

INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1
LOW_CPU, LOW_MEM = -(1 << 36), -(1 << 55)  # KS_MAX_CPU_MILLI / KS_MAX_MEM_BYTES, negated
ROW_DTYPE = np.dtype([("node_idx", np.int32), ("n_victims", np.uint32), ("candidates", np.uint32),
                      ("feasible_cnt", np.uint32), ("max_victim_priority", np.int32), ("reserved", np.uint32),
                      ("victim_priority_sum", np.int64)])


def _visit_order(bound_node, bound_prio):
    """Bound pods sorted by node, then in each node's visit order; the sort keys; segment starts per node."""
    B = len(bound_node)
    node = np.asarray(bound_node, np.int64)
    prio = np.asarray(bound_prio, np.int64)
    order = np.lexsort((np.arange(B), -prio, node))  # node, priority descending, bound index ascending
    key = node[order] * (1 << 33) + (INT32_MAX - prio[order])
    return order, key


def preempt_packed(orc, free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, priority,
                   bound_node, bound_cpu, bound_mem, bound_prio, max_victims):
    """rows (ROW_DTYPE [P]) and victims (int32 [P, max_victims], bound indices, -1 past n_victims)."""
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    rc, rm = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
    P, N = len(rc), len(fc)
    rows = np.zeros(P, ROW_DTYPE)
    rows["node_idx"] = -1
    rows["max_victim_priority"] = INT32_MIN
    victims = np.full((P, max_victims), -1, np.int32)
    if P == 0:
        return rows, victims
    if N == 0:
        return rows, victims
    codes = orc.run_packed(fc, fm, alloc_cpu, alloc_mem, labels, rc, rm, sel, want_mask=False, want_codes=True)[4]
    low = orc.run_packed(fc, fm, alloc_cpu, alloc_mem, labels, np.full(P, LOW_CPU, np.int64), np.full(P, LOW_MEM, np.int64),
                         sel, want_mask=False, want_codes=True)[4]
    assert not (low == 1).any()  # the lowest legal request fits every node
    order, key = _visit_order(bound_node, bound_prio)
    s_cpu = np.asarray(bound_cpu, np.int64)[order]
    s_mem = np.asarray(bound_mem, np.int64)[order]
    s_prio = np.asarray(bound_prio, np.int64)[order]
    c_cpu = np.concatenate([[0], np.cumsum(s_cpu)])  # int64 wraps, but every difference used below fits int64
    c_mem = np.concatenate([[0], np.cumsum(s_mem)])
    seg_end = np.searchsorted(key, (np.arange(N, dtype=np.int64) + 1) * (1 << 33), side="left")
    rows["feasible_cnt"] = (codes == 0).sum(axis=1)
    for p in range(P):
        if rows["feasible_cnt"][p] > 0:
            continue  # already fits somewhere: no plan, no candidates
        pi = int(priority[p])
        nodes = np.nonzero((codes[p] == 1) & (low[p] == 0))[0]  # fails on resources alone
        if len(nodes) == 0:
            continue
        end = seg_end[nodes]
        q = np.searchsorted(key, nodes * (1 << 33) + (INT32_MAX - pi), side="right")  # lower set = [q, end)
        ac = fc[nodes] + (c_cpu[end] - c_cpu[q])
        am = fm[nodes] + (c_mem[end] - c_mem[q])
        ok = (q < end) & (rc[p] <= ac) & (rm[p] <= am)
        nodes, q, end, ac, am = nodes[ok], q[ok], end[ok], ac[ok], am[ok]
        K = len(nodes)
        if K == 0:
            continue
        vcnt = np.zeros(K, np.int64)
        vsum = np.zeros(K, np.int64)
        vmax = np.full(K, INT32_MIN, np.int64)
        alive = np.ones(K, bool)
        vic = np.full((K, max_victims), -1, np.int64)
        for k in range(int((end - q).max())):
            j = q + k
            act = alive & (j < end)
            if not act.any():
                break
            jj = np.where(act, j, 0)
            bc, bm = s_cpu[jj], s_mem[jj]
            keep = act & (rc[p] <= ac - bc) & (rm[p] <= am - bm)  # reprieved
            ac = np.where(keep, ac - bc, ac)
            am = np.where(keep, am - bm, am)
            evict = act & ~keep
            alive &= ~(evict & (vcnt == max_victims))  # one victim more than the cap
            evict &= alive
            vmax = np.where(evict & (vcnt == 0), s_prio[jj], vmax)
            vsum = np.where(evict, vsum + s_prio[jj] + (1 << 31), vsum)
            rows_e = np.nonzero(evict)[0]
            vic[rows_e, vcnt[rows_e]] = order[jj[rows_e]]
            vcnt = np.where(evict, vcnt + 1, vcnt)
        assert (vcnt[alive] > 0).all()
        if not alive.any():
            continue
        a = np.nonzero(alive)[0]
        best = a[np.lexsort((nodes[a], vcnt[a], vsum[a], vmax[a]))[0]]
        rows["candidates"][p] = len(a)
        rows["node_idx"][p] = nodes[best]
        rows["n_victims"][p] = vcnt[best]
        rows["max_victim_priority"][p] = vmax[best]
        rows["victim_priority_sum"][p] = vsum[best]
        victims[p] = vic[best]
    return rows, victims


def crowded(ks, n_pods, n_nodes, seed, n_keys=8, per_node=6, prio_levels=(0, 100, 1000), pod_levels=(0, 100, 1000, 5000)):
    """A synth cluster whose nodes are over-full: per_node bound pods per node, each taking 17-30% of its node, so that a
    pod fits only on the few light nodes (one in 997, pods of 1-4%) and elsewhere evicting lower-priority pods makes
    room.  prio_levels / pod_levels = None draws priorities from the whole int32 range.
    Returns (ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp)."""
    cl = ks.synth.make(n_pods, n_nodes, seed, n_keys=n_keys, bound_per_node=0)
    ac, am, lab, _, _, _, rc, rm, sel = cl.packed()
    rng = np.random.default_rng(seed)
    bn = np.repeat(np.arange(n_nodes, dtype=np.int32), per_node)
    rng.shuffle(bn)
    share = np.where(bn % 997 == 5, rng.integers(1, 5, len(bn)), rng.integers(17, 31, len(bn)))
    bc = ac[bn] * share // 100
    bm = am[bn] // 100 * share

    def draw(levels, n):
        if levels is None:
            return rng.integers(INT32_MIN, INT32_MAX, n, endpoint=True, dtype=np.int64).astype(np.int32)
        return rng.choice(np.array(levels, np.int32), n)

    return ac, am, lab, bn, bc, bm, draw(prio_levels, len(bn)), rc, rm, sel, draw(pod_levels, n_pods)
