"""CPU restatement of the scale-up estimate under the full filter (ks_fit_scaleup_estimate, include/ksched.h; DESIGN.md
5v).

Over string-level objects, as cluster-autoscaler's binpacking estimator sees a template node: pod p is eligible for
template t when it passes, in ks_fit_bind's order, cpu and memory against the template's capacity (no zero skip) and
its selector against the template's labels, then fit_bind_oracle.fits_request against the template's allocatable by
name with its DaemonSet pods as the node's pods (the pod count and every requested name, upstream's zero skip), then
node_bind_oracle.untolerated_hard and node_bind_oracle.required_ok.  The eligible pods go, largest cpu/memory key first
(ties to the lower pod index), to the first open node of the template on which they pass the same resource filters
against what that node's pods already take, else to a new node while fewer than max_nodes are open.  The best template
is scaleup_oracle.best_template's.  The compiled rule words, label bits and resource columns the device takes are
never read here; to_arrays() builds them for the device tests from the same objects.

A problem is a dict: templates, a list of {ac, am (allocatable cpu / memory), fc, fm (capacity after the DaemonSet
pods), labels (map), taints (taint dicts), alloc ({name: int}, "pods" included), ds (a list of {name: int}: the DaemonSet
pods' requests), max_nodes}; pods, a list of {cpu, mem, selector (map), group, res ({name: int})}; group_rules, a list
of node_bind_oracle rule dicts; names, the resource names in device column order ("pods" first)."""
import numpy as np

from fit_bind_oracle import CPU_MEM, NodeUsage, fits_request
from fit_drain_oracle import pack_labels
from node_bind_oracle import compile_rules, required_ok, untolerated_hard
from scaleup_oracle import SCALEUP_OPTION_DTYPE, best_template

ELIGIBLE = 4


def sel_ok(selector, labels):
    return all(labels.get(k) == v for k, v in selector.items())


def stage(q, tp, rules, with_rules=True, with_res=True):
    """Pod q's refusal stage on an empty node of template tp: 0 cpu, memory or selector, 1 a resource, 2 a taint, 3 node
    affinity, ELIGIBLE."""
    if q["cpu"] > tp["fc"] or q["mem"] > tp["fm"] or not sel_ok(q["selector"], tp["labels"]):
        return 0
    if with_res:
        ds = NodeUsage(1, [(0, r) for r in tp["ds"]])
        if fits_request(q["res"], tp["alloc"], ds.req[0], ds.pods[0]):
            return 1
    if with_rules:
        rule = rules[q["group"]] if q["group"] >= 0 else {}
        if untolerated_hard(tp["taints"], rule.get("tolerations", ())):
            return 2
        if not required_ok(rule, tp["labels"]):
            return 3
    return ELIGIBLE


def fit_scaleup(d, with_rules=True, with_res=True, which=None):
    """(rows [T], best, node [T, P], refused [P, 4], used [T, R]) as Snapshot.fit_scaleup_estimate gives them for the
    arrays to_arrays(d) builds (rules and res NULL when with_rules / with_res is False).  which: the templates to pack
    (default all); the others keep a zero row and -1 nodes, and best is picked over the packed ones."""
    tps, pods, rules, names = d["templates"], d["pods"], d["group_rules"], d["names"] if with_res else []
    T, P = len(tps), len(pods)
    rows = np.zeros(T, SCALEUP_OPTION_DTYPE)
    node = np.full((T, P), -1, np.int32)
    refused = np.zeros((P, 4), np.uint32)
    used = np.zeros((T, len(names)), np.int64)
    st = np.array([[stage(q, tp, rules, with_rules, with_res) for tp in tps] for q in pods], np.int64).reshape(P, T)
    for s in range(4):
        refused[:, s] = (st == s).sum(axis=1)
    for t in range(T) if which is None else which:
        tp = tps[t]
        ac, am = int(tp["ac"]), int(tp["am"])
        elig = [p for p in range(P) if st[p, t] == ELIGIBLE]
        order = sorted(elig, key=lambda p: (-(pods[p]["cpu"] * am + pods[p]["mem"] * ac), p))
        open_ = []  # per node: [cpu left, memory left, NodeUsage of its pods (DaemonSet pods first)]
        placed = uc = um = 0
        for p in order:
            q = pods[p]
            o = next((i for i, (c, m, u) in enumerate(open_) if q["cpu"] <= c and q["mem"] <= m and
                      (not with_res or not fits_request(q["res"], tp["alloc"], u.req[0], u.pods[0]))), -1)
            if o < 0:
                if len(open_) >= int(tp["max_nodes"]):
                    continue  # not placed; a later, smaller pod may still fit
                open_.append([int(tp["fc"]), int(tp["fm"]), NodeUsage(1, [(0, r) for r in tp["ds"]])])
                o = len(open_) - 1
            open_[o][0] -= q["cpu"]
            open_[o][1] -= q["mem"]
            open_[o][2].add(0, q["res"])
            node[t, p] = o
            placed += 1
            uc += q["cpu"]
            um += q["mem"]
            for r, name in enumerate(names):
                used[t, r] += 1 if name == "pods" else q["res"].get(name, 0)
        n = len(open_)
        util = (uc * 100 // (n * ac) + um * 100 // (n * am)) // 2 if n else 0
        rows[t] = (n, placed, len(elig), util, uc, um)
    return rows, best_template(rows), node, refused, used


def to_arrays(d):
    """The arguments of Snapshot.fit_scaleup_estimate for problem d: a dict with alloc_cpu, alloc_mem, free_cpu,
    free_mem, labels, max_nodes, req_cpu, req_mem, sel, group, n_groups, rules (node_bind_oracle.compile_rules over the
    templates), node_free [R, T] (allocatable minus the DaemonSet pods; "pods" minus their number) and pod_req [P, R]."""
    tps, pods, names = d["templates"], d["pods"], d["names"]
    T, P = len(tps), len(pods)
    labels, sel = pack_labels([tp["labels"] for tp in tps], [q["selector"] for q in pods])
    node_free = np.array([[tp["alloc"].get(n, 0) - (len(tp["ds"]) if n == "pods" else
                                                     sum(r.get(n, 0) for r in tp["ds"])) for tp in tps]
                          for n in names], np.int64).reshape(len(names), T)
    pod_req = np.array([[1 if n == "pods" else q["res"].get(n, 0) for n in names] for q in pods],
                       np.int64).reshape(P, len(names))
    return dict(alloc_cpu=np.array([tp["ac"] for tp in tps], np.int64), alloc_mem=np.array([tp["am"] for tp in tps], np.int64),
                free_cpu=np.array([tp["fc"] for tp in tps], np.int64), free_mem=np.array([tp["fm"] for tp in tps], np.int64),
                labels=labels, max_nodes=np.array([tp["max_nodes"] for tp in tps], np.uint32),
                req_cpu=np.array([q["cpu"] for q in pods], np.int64), req_mem=np.array([q["mem"] for q in pods], np.int64),
                sel=sel, group=np.array([q["group"] for q in pods], np.int32), n_groups=len(d["group_rules"]),
                rules=compile_rules([tp["labels"] for tp in tps], [tp["taints"] for tp in tps], d["group_rules"]),
                node_free=node_free, pod_req=pod_req)


def batch_names(pods):
    """"pods", then every other name the pods request with a non-zero quantity, in order of first request"""
    names = ["pods"]
    for q in pods:
        for n, v in q["res"].items():
            if n not in CPU_MEM and n != "pods" and v and n not in names:
                names.append(n)
    return names


def template(cpu, mem, labels=None, taints=(), alloc=None, ds=(), max_nodes=1024):
    """A template of cpu millicores and mem bytes allocatable; ds: (cpu, mem, {name: int}) of its DaemonSet pods."""
    return dict(ac=cpu, am=mem, fc=cpu - sum(c for c, _, _ in ds), fm=mem - sum(m for _, m, _ in ds),
                labels=dict(labels or {}), taints=list(taints), alloc=dict(alloc or {"pods": 110}),
                ds=[dict(r) for _, _, r in ds], max_nodes=max_nodes)


def pod(cpu, mem, group=-1, selector=None, res=None):
    return dict(cpu=cpu, mem=mem, group=group, selector=dict(selector or {}), res=dict(res or {}))


def problem(templates, pods, group_rules=(), names=None):
    return dict(templates=list(templates), pods=list(pods), group_rules=list(group_rules),
                names=list(names) if names is not None else batch_names(pods))


GPU_TAINT = {"key": "nvidia.com/gpu", "value": "present", "effect": "NoSchedule"}
TOL_GPU = {"key": "nvidia.com/gpu", "operator": "Exists", "effect": "NoSchedule"}


def random_problem(rng, T, P, G=4, gpu_every=4, extra=1, max_nodes=(0, 40), ds_max=3):
    """T templates (a tainted 8-GPU group about one in gpu_every, instance-type / zone / gen labels, 32-110 pods,
    further extended resources, 0 to ds_max DaemonSet pods) and P pods of G groups: GPU groups tolerate the taint and
    request 1-8 GPUs, others carry required In / NotIn / Gt terms, selectors now and then."""
    types, zones = ["m5", "c5", "r5", "p4"], ["a", "b", "c"]
    ext = [f"example.com/r{i}" for i in range(extra)]
    tps = []
    for t in range(T):
        gpu = t % gpu_every == 0
        lab = {"node.kubernetes.io/instance-type": "p4" if gpu else types[int(rng.integers(0, 3))],
               "zone": zones[int(rng.integers(0, 3))]}
        if rng.random() < 0.7:
            lab["gen"] = str(int(rng.integers(1, 6)))
        alloc = {"pods": int(rng.integers(2, 111))}
        if gpu:
            alloc["nvidia.com/gpu"] = 8
        for r in ext:
            if rng.random() < 0.6:
                alloc[r] = int(rng.integers(0, 9))
        cpu, mem = int(rng.integers(4, 97)) * 1000, int(rng.integers(8, 385)) << 30
        ds = [(int(rng.integers(0, 500)), int(rng.integers(0, 1 << 28)),
               {r: 1 for r in ext if rng.random() < 0.2}) for _ in range(int(rng.integers(0, ds_max + 1)))]
        tps.append(template(cpu, mem, lab, [GPU_TAINT] if gpu else [], alloc, ds,
                            int(rng.integers(max_nodes[0], max_nodes[1] + 1))))
    rules = []
    for g in range(G):
        r = {"tolerations": [TOL_GPU] if g % 2 == 0 else []}
        if g % 3 == 1:
            r["required"] = [[{"key": "zone", "operator": "In", "values": ["a", "b"]}],
                             [{"key": "gen", "operator": "Gt", "values": ["3"]}]]
        if g % 3 == 2:
            r["required"] = [[{"key": "node.kubernetes.io/instance-type", "operator": "NotIn", "values": ["r5"]}]]
        rules.append(r)
    pods = []
    for _ in range(P):
        g = int(rng.integers(-1, G))
        res = {}
        if g >= 0 and g % 2 == 0 and rng.random() < 0.5:
            res["nvidia.com/gpu"] = int(rng.integers(1, 9))
        for r in ext:
            if rng.random() < 0.2:
                res[r] = int(rng.integers(1, 4))
        sel = {"zone": zones[int(rng.integers(0, 3))]} if rng.random() < 0.1 else {}
        pods.append(pod(int(rng.integers(1, 80)) * 100, int(rng.integers(1, 64)) << 27, g, sel, res))
    return problem(tps, pods, rules)


def golden_problem(case):
    """The problem of one case of tests/golden/gv1_fit_scaleup.json"""
    tps = [template(t["cpu"], t["mem"], t["labels"], t["taints"], t["alloc"], [tuple(x) for x in t["ds"]], t["max_nodes"])
           for t in case["templates"]]
    pods = [pod(q["cpu"], q["mem"], q["group"], q["selector"], q["res"]) for q in case["pods"] for _ in range(q["repeat"])]
    return problem(tps, pods, case["group_rules"])
