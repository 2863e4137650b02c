"""CPU restatement of preemption under the full filter (ks_fit_preempt, include/ksched.h; DESIGN.md 5t).

Over string-level objects, as upstream's DefaultPreemption sees them: a node is unresolvable when the pod's selector
misses its labels, one of its NoSchedule / NoExecute taints is not tolerated (node_bind_oracle.untolerated_hard) or the
group's required node affinity fails (node_bind_oracle.required_ok); resources are name maps checked with
fit_bind_oracle.fits_request, which includes the pod count.  Each eligible node's lower set is walked in plain Python:
the pods with priority strictly below the pod's, in priority-descending order, ties to the lower bound index; a pod
stays when the pending pod still fits with it back on the node, otherwise it is a victim.  The compiled masks, domain
sets and arrays the device takes are never read here.

Inputs: free_cpu / free_mem [N] (allocatable minus the bound pods), labels [N, W] and sel [P, W] packed label bits,
req_cpu / req_mem / priority / group [P]; node_labels [N] and node_taints [N] (label maps and taint dicts),
group_rules[g] as node_bind_oracle takes them; alloc None (no resource is checked: the C call's NULL res) or [N] maps
{name: int} including "pods"; bound a list of (node, cpu, mem, priority, {name: int}); pod_res [P] maps."""
import numpy as np

from fit_bind_oracle import NodeUsage, fits_request
from node_bind_oracle import required_ok, untolerated_hard
from preempt_oracle import INT32_MIN, ROW_DTYPE


def resolvable_nodes(labels, sel_p, node_labels, node_taints, rule):
    """bool [N]: the nodes where no eviction is needed to pass the selector, taints and required node affinity."""
    sel_ok = ((np.asarray(sel_p, np.uint64)[None, :] & ~np.asarray(labels, np.uint64)) == 0).all(axis=1)
    tols = rule.get("tolerations", ())
    return np.array([bool(sel_ok[n]) and not untolerated_hard(node_taints[n], tols) and required_ok(rule, node_labels[n])
                     for n in range(len(sel_ok))], bool)


def evicted(fc, fm, usage, bound, n, removed):
    """Node n with the bound pods `removed` taken off it: (free cpu, free memory, requested map, pod count)."""
    req = dict(usage.req[n])
    for b in removed:
        for name, q in bound[b][4].items():
            req[name] = req.get(name, 0) - q
    return (int(fc[n]) + sum(bound[b][1] for b in removed), int(fm[n]) + sum(bound[b][2] for b in removed), req,
            usage.pods[n] - len(removed))


def put_back(state, b):
    """state with bound pod b (a bound-list row) back on the node"""
    c, m, req, pods = state
    req = dict(req)
    for name, q in b[4].items():
        req[name] = req.get(name, 0) + q
    return c - b[1], m - b[2], req, pods + 1


def fits_state(state, alloc, rc, rm, res, n):
    """A pod of requests rc, rm and res (a map) fits node n in `state`: cpu and memory without a zero skip, then
    (alloc not None) fits_request over the names and the pod count."""
    c, m, req, pods = state
    if rc > c or rm > m:
        return False
    return alloc is None or not fits_request(res, alloc[n], req, pods)


def fits_with(fc, fm, usage, alloc, bound, rc, rm, res, n, removed):
    """fits_state of node n with the bound pods `removed` taken off it"""
    return fits_state(evicted(fc, fm, usage, bound, n, removed), alloc, rc, rm, res, n)


def fit_preempt_packed(free_cpu, free_mem, labels, req_cpu, req_mem, sel, priority, group, node_labels, node_taints,
                       group_rules, alloc, bound, pod_res, max_victims):
    """rows (ROW_DTYPE [P]), victims (int32 [P, max_victims]) and unresolvable (uint32 [P]) as Snapshot.fit_preempt."""
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    N, P = len(fc), len(req_cpu)
    labels = np.asarray(labels, np.uint64).reshape(N, -1)
    sel = np.asarray(sel, np.uint64).reshape(P, -1)
    rows = np.zeros(P, ROW_DTYPE)
    rows["node_idx"] = -1
    rows["max_victim_priority"] = INT32_MIN
    victims = np.full((P, max_victims), -1, np.int32)
    unres = np.zeros(P, np.uint32)
    usage = NodeUsage(N, [(b[0], b[4]) for b in bound])
    on = [[] for _ in range(N)]
    for i, b in enumerate(bound):
        on[b[0]].append(i)
    cache = {}
    for p in range(P):
        g, pi, rc, rm = int(group[p]), int(priority[p]), int(req_cpu[p]), int(req_mem[p])
        rule = group_rules[g] if g >= 0 else {}
        key = (g, sel[p].tobytes())
        if key not in cache:
            cache[key] = resolvable_nodes(labels, sel[p], node_labels, node_taints, rule)
        res = cache[key]
        unres[p] = int((~res).sum())

        def fits(n, removed):
            return fits_with(fc, fm, usage, alloc, bound, rc, rm, pod_res[p], n, removed)

        best, ncand, feasible = None, 0, 0
        for n in np.nonzero(res)[0].tolist():
            if fits(n, ()):
                feasible += 1
                continue
            lower = sorted((b for b in on[n] if bound[b][3] < pi), key=lambda b: (-bound[b][3], b))
            if not lower:
                continue
            state = evicted(fc, fm, usage, bound, n, lower)
            if not fits_state(state, alloc, rc, rm, pod_res[p], n):
                continue
            vic = []
            for b in lower:
                back = put_back(state, bound[b])
                if fits_state(back, alloc, rc, rm, pod_res[p], n):
                    state = back  # reprieved
                else:
                    vic.append(b)
            assert vic  # with none, p would fit n as it is
            if len(vic) > max_victims:
                continue
            ncand += 1
            k = (bound[vic[0]][3], sum(bound[b][3] + (1 << 31) for b in vic), len(vic), n)
            if best is None or k < best[0]:
                best = (k, vic)
        rows["feasible_cnt"][p] = feasible
        if feasible or best is None:
            continue
        (vmax, vsum, vcnt, n), vic = best
        rows["candidates"][p] = ncand
        rows["node_idx"][p] = n
        rows["n_victims"][p] = vcnt
        rows["max_victim_priority"][p] = vmax
        rows["victim_priority_sum"][p] = vsum
        victims[p, :vcnt] = vic
    return rows, victims, unres


def bound_requests(bound, names):
    """bound_req int64 [B, R] of the bound list's maps for the batch's resource names ("pods" is 1)."""
    return np.array([[1 if r == "pods" else b[4].get(r, 0) for r in names] for b in bound],
                    np.int64).reshape(len(bound), len(names))


def pack_labels(node_labels, selectors):
    """labels uint64 [N, W] and sel [P, W]: one bit per (key, value) pair a node carries or a selector names."""
    pairs = sorted({kv for m in list(node_labels) + list(selectors) for kv in m.items()})
    W = next(w for w in (1, 2, 4, 8) if 64 * w >= max(len(pairs), 1))
    bit = {kv: i for i, kv in enumerate(pairs)}

    def pack(maps):
        out = np.zeros((len(maps), W), np.uint64)
        for i, m in enumerate(maps):
            for kv in m.items():
                out[i, bit[kv] // 64] |= np.uint64(1 << (bit[kv] % 64))
        return out
    return pack(node_labels), pack(selectors)


def cluster_inputs(node_cpu, node_mem, node_labels, node_taints, alloc, bound, pods, names=None):
    """Everything the restatement and Snapshot.fit_preempt take for one cluster.  pods: a list of dicts with cpu, mem,
    selector, priority, group and res; bound as fit_preempt_packed takes it.  Returns a dict: the packed node and pod
    arrays, the bound list's columns, free_cpu / free_mem, and (alloc given) names, node_free, pod_req and bound_req."""
    from fit_bind_oracle import compile_resources
    N = len(node_cpu)
    labels, sel = pack_labels(node_labels, [p["selector"] for p in pods])
    d = dict(ac=np.asarray(node_cpu, np.int64), am=np.asarray(node_mem, np.int64), labels=labels, sel=sel,
             rc=np.array([p["cpu"] for p in pods], np.int64).reshape(len(pods)),
             rm=np.array([p["mem"] for p in pods], np.int64).reshape(len(pods)),
             prio=np.array([p["priority"] for p in pods], np.int32).reshape(len(pods)),
             group=np.array([p["group"] for p in pods], np.int32).reshape(len(pods)),
             bn=np.array([b[0] for b in bound], np.int32).reshape(len(bound)),
             bc=np.array([b[1] for b in bound], np.int64).reshape(len(bound)),
             bm=np.array([b[2] for b in bound], np.int64).reshape(len(bound)),
             bp=np.array([b[3] for b in bound], np.int32).reshape(len(bound)))
    d["fc"], d["fm"] = d["ac"].copy(), d["am"].copy()
    np.subtract.at(d["fc"], d["bn"], d["bc"])
    np.subtract.at(d["fm"], d["bn"], d["bm"])
    if alloc is not None:
        names, node_free, pod_req = compile_resources(alloc, [(b[0], b[4]) for b in bound], [p["res"] for p in pods],
                                                      names)
        d.update(names=names, node_free=node_free.reshape(len(names), N), pod_req=pod_req,
                 bound_req=bound_requests(bound, names))
    return d


def golden_case(case):
    """cluster_inputs of one case of tests/golden/gv1_fit_preempt.json, with its string-level objects and rules."""
    nodes, pod = case["nodes"], dict(case["pod"])
    pod["group"] = 0 if pod["rule"] is not None else -1
    group_rules = [pod["rule"]] if pod["rule"] is not None else []
    bound = [(b[0], b[1], b[2], b[3], b[4]) for b in case["bound"]]
    alloc = [n["alloc"] for n in nodes]
    d = cluster_inputs([n["cpu"] for n in nodes], [n["mem"] for n in nodes], [n["labels"] for n in nodes],
                       [n["taints"] for n in nodes], alloc, bound, [pod], case.get("names"))
    d.update(node_labels=[n["labels"] for n in nodes], node_taints=[n["taints"] for n in nodes], group_rules=group_rules,
             alloc=alloc, bound=bound, pod_res=[pod["res"]], G=len(group_rules))
    return d


def fits_after(d, p, n, removed):
    """fits_with for pod p of cluster_inputs d on node n with the bound pods `removed` evicted"""
    return fits_with(d["fc"], d["fm"], NodeUsage(len(d["fc"]), [(b[0], b[4]) for b in d["bound"]]), d["alloc"],
                     d["bound"], int(d["rc"][p]), int(d["rm"][p]), d["pod_res"][p], n, removed)


def run(d, max_victims, with_res=True):
    """fit_preempt_packed over cluster_inputs (plus node_labels, node_taints, group_rules, alloc, bound, pod_res)."""
    return fit_preempt_packed(d["fc"], d["fm"], d["labels"], d["rc"], d["rm"], d["sel"], d["prio"], d["group"],
                              d["node_labels"], d["node_taints"], d["group_rules"], d["alloc"] if with_res else None,
                              d["bound"], d["pod_res"], max_victims)


TOL_POOL = [
    {"key": "nvidia.com/gpu", "operator": "Exists", "effect": "NoSchedule"},
    {"key": "dedicated", "operator": "Equal", "value": "db", "effect": ""},
    {"key": "", "operator": "Exists", "effect": ""},
]
REQ_POOL = [
    {"key": "zone", "operator": "In", "values": ["a", "b"]},
    {"key": "zone", "operator": "NotIn", "values": ["c"]},
    {"key": "gpu", "operator": "Exists"},
    {"key": "gen", "operator": "Gt", "values": ["2"]},
]


def random_cluster(rng, N, P, G, per_node=4, R=3, full_range=False):
    """A crowded random cluster over every filter: zone / gen / disk labels, NoSchedule and NoExecute taints (a GPU
    pool on about 1 node in 5), G group rules with tolerations and required terms, nodes at their pod limit, GPUs (R >= 2) and
    R - 2 further extended resources (some over-committed), bound pods holding 20-45% of a node each, and pending
    pods of 1-4 times that.  Priorities from {0, 100, 1000, 5000}, or with full_range the whole int32 range.  Returns
    cluster_inputs with the string-level objects, as golden_case does."""
    zones = ["a", "b", "c"]
    node_labels, node_taints, alloc = [], [], []
    extra = [f"example.com/r{i}" for i in range(max(0, R - 2))]
    for n in range(N):
        lab = {"zone": zones[int(rng.integers(0, 3))]}
        if rng.random() < 0.7:
            lab["gen"] = str(int(rng.integers(1, 5)))
        if rng.random() < 0.5:
            lab["disk"] = "ssd"
        gpu = rng.random() < 0.2
        taints = []
        if gpu:
            lab["gpu"] = "h100"
            taints.append({"key": "nvidia.com/gpu", "value": "present", "effect": "NoSchedule"})
        if rng.random() < 0.1:
            taints.append({"key": "dedicated", "value": "db", "effect": "NoExecute"})
        a = {"pods": int(rng.integers(1, per_node + 3))}
        if gpu:
            a["nvidia.com/gpu"] = 8
        for r in extra:
            if rng.random() < 0.6:
                a[r] = int(rng.integers(0, 6))
        node_labels.append(lab)
        node_taints.append(taints)
        alloc.append(a)
    ac = rng.integers(24000, 64000, N) * 4
    am = rng.integers(1 << 20, 1 << 30, N) * 8

    def prio():
        return int(rng.integers(-(1 << 31), (1 << 31) - 1, endpoint=True)) if full_range else \
            int(rng.choice([0, 100, 1000, 5000]))
    bound = []
    for n in range(N):
        for _ in range(int(rng.integers(per_node // 2, per_node + 1))):
            share = int(rng.integers(20, 46))
            res = {}
            if R >= 2 and "nvidia.com/gpu" in alloc[n] and rng.random() < 0.7:
                res["nvidia.com/gpu"] = int(rng.integers(1, 5))
            for r in extra:
                if rng.random() < 0.3:
                    res[r] = int(rng.integers(1, 4))
            bound.append((n, int(ac[n]) * share // 100, int(am[n]) // 100 * share, prio(), res))
    rules = []
    for g in range(G):
        r = {"tolerations": [TOL_POOL[int(i)] for i in rng.choice(len(TOL_POOL), int(rng.integers(0, 3)), replace=False)]}
        if rng.random() < 0.5:
            r["required"] = [[REQ_POOL[int(i)] for i in rng.choice(len(REQ_POOL), int(rng.integers(1, 3)), replace=False)]
                             for _ in range(int(rng.integers(1, 3)))]
        rules.append(r)
    pods = []
    mean_c, mean_m = int(ac.mean()), int(am.mean())
    for p in range(P):
        res = {}
        if R >= 2 and rng.random() < 0.3:  # only the batch's resources: the call sees no other
            res["nvidia.com/gpu"] = int(rng.integers(1, 9))
        for r in extra:
            if rng.random() < 0.2:
                res[r] = int(rng.integers(1, 4))
        sel = {}
        if rng.random() < 0.2:
            sel["disk"] = "ssd"
        pods.append(dict(cpu=mean_c * int(rng.integers(40, 130)) // 100, mem=mean_m // 100 * int(rng.integers(10, 60)),
                         selector=sel, priority=prio(), group=int(rng.integers(-1, G)), res=res))
    names = (["pods", "nvidia.com/gpu"] + extra)[:R] if R else None
    d = cluster_inputs(ac, am, node_labels, node_taints, alloc if R else None, bound, pods, names)
    d.update(node_labels=node_labels, node_taints=node_taints, group_rules=rules, alloc=alloc if R else None,
             bound=bound, pod_res=[p["res"] for p in pods], G=G)
    return d
