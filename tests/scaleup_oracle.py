"""CPU restatement of the scale-up estimate (ks_scaleup_estimate, include/ksched.h; DESIGN.md 5g).  The cell codes and
the per-pod reasons come from the oracle's run_packed with the templates as the nodes (capacity F as the free values),
as tests/explain_oracle.py does; the order and the first-fit packing are done in Python integers."""
import numpy as np

from explain_oracle import _counts

SCALEUP_OPTION_DTYPE = np.dtype([("nodes", np.uint32), ("placed", np.uint32), ("eligible", np.uint32),
                                 ("utilization", np.int32), ("used_cpu", np.int64), ("used_mem", np.int64)])


def pack_template(rc, rm, elig, ac, am, fc, fm, max_nodes):
    """First fit of the eligible pods (indices, any order) into new nodes of one template.  Returns (row, {pod: ordinal})."""
    ac, am, fc, fm = int(ac), int(am), int(fc), int(fm)
    order = sorted((int(p) for p in elig), key=lambda p: (-(int(rc[p]) * am + int(rm[p]) * ac), p))
    rem_c = np.zeros(max(int(max_nodes), 1), np.int64)
    rem_m = np.zeros(max(int(max_nodes), 1), np.int64)
    nodes, where = 0, {}
    used_c = used_m = 0
    for p in order:
        c, m = int(rc[p]), int(rm[p])
        hit = np.nonzero((rem_c[:nodes] >= c) & (rem_m[:nodes] >= m))[0]
        if len(hit):
            o = int(hit[0])
        elif nodes < int(max_nodes):
            o = nodes
            nodes += 1
            rem_c[o], rem_m[o] = fc, fm
        else:
            continue  # not placed; a later, smaller pod may still fit
        rem_c[o] -= c
        rem_m[o] -= m
        where[p] = o
        used_c += c
        used_m += m
    util = (used_c * 100 // (nodes * ac) + used_m * 100 // (nodes * am)) // 2 if nodes else 0
    return (nodes, len(where), len(order), util, used_c, used_m), where


def best_template(rows):
    """Most pods placed, then the highest utilization, then the fewest nodes, then the lowest index; -1 if none places."""
    cand = [t for t in range(len(rows)) if rows["placed"][t] > 0]
    if not cand:
        return -1
    return min(cand, key=lambda t: (-int(rows["placed"][t]), -int(rows["utilization"][t]), int(rows["nodes"][t]), t))


def scaleup_packed(orc, alloc_cpu, alloc_mem, free_cpu, free_mem, labels, max_nodes, req_cpu, req_mem, sel, which=None):
    """Returns (rows[T] as SCALEUP_OPTION_DTYPE, best, node int32 [T, P], reasons uint32 [P, 4]).  which: the templates
    to pack (default all); the others keep a zero row and -1 nodes, and best is picked over the packed ones."""
    ac, am = np.asarray(alloc_cpu, np.int64), np.asarray(alloc_mem, np.int64)
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    rc, rm = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
    T, P = len(ac), len(rc)
    rows = np.zeros(T, SCALEUP_OPTION_DTYPE)
    node = np.full((T, P), -1, np.int32)
    if T == 0 or P == 0:
        return rows, -1, node, np.zeros((P, 4), np.uint32)
    labels = np.ascontiguousarray(labels, np.uint64).reshape(T, -1)
    sel = np.ascontiguousarray(sel, np.uint64).reshape(P, -1)
    codes = orc.run_packed(fc, fm, ac, am, labels, rc, rm, sel, want_mask=False, want_codes=True)[4]  # [P, T]
    reasons = _counts(codes, rc[:, None] > fc[None, :], rm[:, None] > fm[None, :])
    for t in range(T) if which is None else which:
        row, where = pack_template(rc, rm, np.nonzero(codes[:, t] == 0)[0], ac[t], am[t], fc[t], fm[t], max_nodes[t])
        rows[t] = row
        for p, o in where.items():
            node[t, p] = o
    return rows, best_template(rows), node, reasons


def packed_from_specs(template_specs, max_nodes, overhead_specs, pod_specs):
    """Test-side packing of object specs for the host-layer tests (quantities written as '<n>m' and plain bytes): one
    label bit per distinct (key, value) pair over templates and selectors.  Returns the arguments of scaleup_packed."""
    def cpu(q):
        return int(q[:-1]) if q.endswith("m") else int(q) * 1000

    def req(spec):
        cs = [c for c in spec.get("containers", []) if c]
        return sum(cpu(c["cpu"]) for c in cs if "cpu" in c), sum(int(c["memory"]) for c in cs if "memory" in c)
    pairs = {}
    for s in template_specs:
        for kv in (s.get("labels") or {}).items():
            pairs.setdefault(kv, len(pairs))
    for s in pod_specs:
        for kv in (s.get("selector") or {}).items():
            pairs.setdefault(kv, len(pairs))
    W = 1
    while len(pairs) > 64 * W:
        W *= 2
    T, P = len(template_specs), len(pod_specs)
    lab, sel = np.zeros((T, W), np.uint64), np.zeros((P, W), np.uint64)
    for rows, specs, field in ((lab, template_specs, "labels"), (sel, pod_specs, "selector")):
        for i, s in enumerate(specs):
            for kv in (s.get(field) or {}).items():
                b = pairs[kv]
                rows[i, b // 64] |= np.uint64(1) << np.uint64(b % 64)
    ac = np.array([cpu(s["allocatable"]["cpu"]) for s in template_specs], np.int64)
    am = np.array([int(s["allocatable"]["memory"]) for s in template_specs], np.int64)
    fc, fm = ac.copy(), am.copy()
    names = [s["name"] for s in template_specs]
    for s in overhead_specs:
        c, m = req(s)
        fc[names.index(s["node_name"])] -= c
        fm[names.index(s["node_name"])] -= m
    rq = np.array([req(s) for s in pod_specs], np.int64).reshape(P, 2)
    return ac, am, fc, fm, lab, np.asarray(max_nodes, np.uint32), rq[:, 0].copy(), rq[:, 1].copy(), sel
