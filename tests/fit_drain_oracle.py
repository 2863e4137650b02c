"""CPU restatement of the drain simulation under the full filter (ks_fit_drain_check, include/ksched.h; DESIGN.md 5u).

Over string-level objects, as upstream's removal simulation sees them: for each candidate, a private copy of every
node's free cpu and memory and of what its pods request by name; its pods in order, each to the destination with the
best score among those that pass, in ks_fit_bind's order, cpu and memory (no zero skip) and the selector, then
fit_bind_oracle.fits_request (the pod count and every requested name, upstream's zero skip), then
node_bind_oracle.untolerated_hard and node_bind_oracle.required_ok; the move is then charged to the copy.  The first pod
with no destination stops the candidate, and the four refusal words count its destinations by the first filter each
fails.  The scores are ks_select's, written out below (policy_oracle's MOST_ALLOCATED and LEAST_BALANCED); the argmax
takes the highest score, ties to the lower node index.  The compiled masks, rule words and resource columns the device
takes are never read here: the name maps are evaluated node by node, once per group and once per name, and the
argmax runs over those values.

Inputs (a dict, as cluster() builds it): fc / fm [N] free cpu and memory, ac / am [N] allocatable, labels [N, W] and
sel [P, W] packed label bits, rc / rm / group [P]; node_labels [N] and node_taints [N] (label maps and taint dicts),
group_rules[g] as node_bind_oracle takes them; alloc None (no resource is checked: the C call's NULL res) or [N] maps
{name: int} including "pods"; bound a list of (node, {name: int}) of the pods on the nodes; pod_res [P] maps."""
import numpy as np

from fit_bind_oracle import CPU_MEM, NodeUsage, compile_resources, fits_request
from node_bind_oracle import required_ok, untolerated_hard
from policy_oracle import SCORE, least

PASS = 4  # stage of a node that passes every filter


def score(policy, fc, fm, ac, am, rc, rm):
    """ks_select's score of one node for one pod, on Python integers (LEFTOVER: the free pair after the pod, packed
    cpu * 2^22 + memory)."""
    if policy == 0:
        return (int(fc) - int(rc)) * (1 << 22) + (int(fm) - int(rm))
    if policy == 1:
        return least(fc, fm, ac, am, rc, rm)
    return SCORE[policy](fc, fm, ac, am, rc, rm)


def scores(policy, fc, fm, ac, am, rc, rm):
    """score() on int64 arrays (the same integers: inside the limits of ksched.h nothing overflows)"""
    if policy == 0:
        return (fc - rc) * (1 << 22) + (fm - rm)
    if policy == 1:
        def pct(f, a):
            pos = a > 0
            x = (f * 100)
            return np.where(pos, np.sign(x) * (np.abs(x) // np.where(pos, a, 1)), 0)
        s = pct(fc - rc, ac) + pct(fm - rm, am)
        return np.sign(s) * (np.abs(s) // 2)
    from policy_oracle import SCORES
    return SCORES[policy](fc, fm, ac, am, rc, rm)


class Cluster:
    """The string-level objects of one call, with each filter evaluated per node from the maps: rule_stage(g) [N] is 2
    (untolerated hard taint), 3 (required node affinity fails) or PASS, per group; free_of(name) [N] is what
    fits_request compares a request of `name` against (allocatable minus what the node's pods request; for "pods" the
    pods left under the limit)."""

    def __init__(self, d, with_rules=True, with_res=True):
        self.d = d
        self.N = len(d["fc"])
        self.alloc = d["alloc"] if with_res else None
        self.with_rules = with_rules
        self.usage = NodeUsage(self.N, d["bound"])
        self._stage, self._free = {}, {}

    def rule_of(self, g):
        return self.d["group_rules"][g] if g >= 0 and self.with_rules else {}

    def rule_stage(self, g):
        if g not in self._stage:
            rule = self.rule_of(g)
            tols = rule.get("tolerations", ())
            st = np.full(self.N, PASS, np.int8)
            if self.with_rules:
                for n in range(self.N):
                    if untolerated_hard(self.d["node_taints"][n], tols):
                        st[n] = 2
                    elif not required_ok(rule, self.d["node_labels"][n]):
                        st[n] = 3
            self._stage[g] = st
        return self._stage[g]

    def free_of(self, name):
        if name not in self._free:
            u = self.usage
            self._free[name] = np.array([self.alloc[n].get("pods", 0) - u.pods[n] if name == "pods" else
                                         self.alloc[n].get(name, 0) - u.req[n].get(name, 0) for n in range(self.N)],
                                        np.int64)
        return self._free[name]

    def node_stage(self, p, n, c, m, req, pods):
        """The stage of node n for pod p with the node's state (free cpu, free memory, requested map, pod count): 0
        cpu, memory or selector, 1 a resource (fits_request), 2 a taint, 3 node affinity, PASS."""
        d = self.d
        if d["rc"][p] > c or d["rm"][p] > m or ((d["sel"][p] & ~d["labels"][n]) != 0).any():
            return 0
        if self.alloc is not None and fits_request(d["pod_res"][p], self.alloc[n], req, pods):
            return 1
        return int(self.rule_stage(int(d["group"][p]))[n])


def fit_drain(d, node_idx, offset, policy=0, exclude=False, with_rules=True, with_res=True):
    """(placed[D], node_idx[P], score[P], refused[D, 4]) as Snapshot.fit_drain_check gives them for cluster d."""
    cl = Cluster(d, with_rules, with_res)
    fc, fm, ac, am = (np.asarray(d[k], np.int64) for k in ("fc", "fm", "ac", "am"))
    labels, sel = d["labels"], d["sel"]
    N, P, D = cl.N, len(d["rc"]), len(node_idx)
    node_idx = np.asarray(node_idx, np.int64)
    placed = np.zeros(D, np.uint32)
    idx = np.full(P, -1, np.int32)
    out = np.zeros(P, np.int64)
    refused = np.zeros((D, 4), np.uint32)
    sel_ok = {}
    for c in range(D):
        gone = np.zeros(N, bool)
        gone[node_idx if exclude else node_idx[c]] = True
        over = {}  # the candidate's moves: node -> [free cpu, free memory, requested map, pod count]
        for p in range(int(offset[c]), int(offset[c + 1])):
            rc, rm, g = int(d["rc"][p]), int(d["rm"][p]), int(d["group"][p])
            key = sel[p].tobytes()
            if key not in sel_ok:
                sel_ok[key] = ((sel[p][None, :] & ~labels) == 0).all(axis=1)
            # the nodes the candidate has not touched, from the per-node values
            stage = np.where((rc <= fc) & (rm <= fm) & sel_ok[key], cl.rule_stage(g), 0)
            if cl.alloc is not None:
                lack = np.zeros(N, bool)
                for name, q in list(d["pod_res"][p].items()) + [("pods", 1)]:
                    if name in CPU_MEM or q == 0 or (name == "pods" and q != 1):
                        continue
                    lack |= q > cl.free_of(name)
                stage = np.where((stage > 0) & lack, 1, stage)
            stage[gone] = -1
            for n, (c_, m_, req, pods) in over.items():  # the nodes it has: their private state
                stage[n] = cl.node_stage(p, n, c_, m_, req, pods)
            ok = np.flatnonzero(stage == PASS)
            if len(ok) == 0:
                refused[c] = [int((stage == s).sum()) for s in range(4)]
                break
            f_c = fc[ok].copy()
            f_m = fm[ok].copy()
            for i, n in enumerate(ok.tolist()):
                if n in over:
                    f_c[i], f_m[i] = over[n][0], over[n][1]
            sc = scores(policy, f_c, f_m, ac[ok], am[ok], rc, rm)
            best = int(np.argmax(sc))  # the first maximum: ties to the lower node index
            n = int(ok[best])
            idx[p], out[p] = n, int(sc[best])
            if n not in over:
                over[n] = [int(fc[n]), int(fm[n]), dict(cl.usage.req[n]), cl.usage.pods[n]]
            st = over[n]
            st[0] -= rc
            st[1] -= rm
            st[3] += 1
            for name, q in d["pod_res"][p].items():
                if name not in CPU_MEM:
                    st[2][name] = st[2].get(name, 0) + q
            placed[c] += 1
    return placed, idx, out, refused


def destinations(d, node_idx, c, exclude):
    """The destination count of candidate c"""
    gone = set(np.asarray(node_idx).tolist()) if exclude else {int(node_idx[c])}
    return len(d["fc"]) - len(gone)


def replay_ok(d, node_idx, offset, c, idx, with_rules=True, with_res=True):
    """D4: candidate c's moves applied one at a time to a copy of the cluster - free cpu and memory reduced by the
    requests, the node's requested map and pod count raised - each pod passing the full filter at its turn."""
    cl = Cluster(d, with_rules, with_res)
    state = {}
    for p in range(int(offset[c]), int(offset[c + 1])):
        n = int(idx[p])
        if n < 0 or n == int(node_idx[c]):
            return False
        st = state.setdefault(n, [int(d["fc"][n]), int(d["fm"][n]), dict(cl.usage.req[n]), cl.usage.pods[n]])
        if cl.node_stage(p, n, *st) != PASS:
            return False
        st[0] -= int(d["rc"][p])
        st[1] -= int(d["rm"][p])
        st[3] += 1
        for name, q in d["pod_res"][p].items():
            if name not in CPU_MEM:
                st[2][name] = st[2].get(name, 0) + q
    return True


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


def cluster(nodes, bound, cands, names=None, bind_drained=True):
    """Everything the restatement and Snapshot.fit_drain_check take for one cluster.  nodes: dicts with cpu, mem,
    labels, taints and alloc (a name map with "pods"); bound: (node, cpu, mem, {name: int}) of the pods already on the
    nodes that are not drained; cands: (node, [pod dicts with cpu, mem, selector, group, res]) - each drained pod is also
    bound to its candidate unless bind_drained is False (many candidates on few nodes: the call takes any pods).  Returns the dict fit_drain takes, with node_idx, offset, group_rules left to the caller
    (default []), and node_free [R, N] / pod_req [P, R] for the batch's names."""
    pods = [q for _, qs in cands for q in qs]
    allb = list(bound) + ([(n, q["cpu"], q["mem"], q["res"]) for n, qs in cands for q in qs] if bind_drained else [])
    node_labels = [n["labels"] for n in nodes]
    labels, sel = pack_labels(node_labels, [q["selector"] for q in pods])
    ac = np.array([n["cpu"] for n in nodes], np.int64)
    am = np.array([n["mem"] for n in nodes], np.int64)
    fc, fm = ac.copy(), am.copy()
    for b in allb:
        fc[b[0]] -= b[1]
        fm[b[0]] -= b[2]
    d = dict(fc=fc, fm=fm, ac=ac, am=am, labels=labels, sel=sel,
             rc=np.array([q["cpu"] for q in pods], np.int64).reshape(len(pods)),
             rm=np.array([q["mem"] for q in pods], np.int64).reshape(len(pods)),
             group=np.array([q["group"] for q in pods], np.int32).reshape(len(pods)),
             node_labels=node_labels, node_taints=[n["taints"] for n in nodes], alloc=[n["alloc"] for n in nodes],
             bound=[(b[0], b[3]) for b in allb], pod_res=[q["res"] for q in pods], group_rules=[],
             bn=np.array([b[0] for b in allb], np.int32), bc=np.array([b[1] for b in allb], np.int64),
             bm=np.array([b[2] for b in allb], np.int64),
             node_idx=np.array([n for n, _ in cands], np.int32),
             offset=np.concatenate([[0], np.cumsum([len(qs) for _, qs in cands])]).astype(np.uint64))
    names, node_free, pod_req = compile_resources(d["alloc"], d["bound"], d["pod_res"], names)
    d.update(names=names, node_free=node_free, pod_req=pod_req)
    return d


def golden_case(case):
    """cluster() of one case of tests/golden/gv1_fit_drain.json"""
    d = cluster(case["nodes"], [tuple(b) for b in case["bound"]], [(c["node"], c["pods"]) for c in case["candidates"]])
    d["group_rules"] = case["group_rules"]
    return d


TOL_GPU = {"key": "nvidia.com/gpu", "operator": "Exists", "effect": "NoSchedule"}
CORDON = {"key": "node.kubernetes.io/unschedulable", "value": "", "effect": "NoSchedule"}


def random_cluster(rng, N, D, R=3, G=4, max_pods=6, gpu_every=5, share=(5, 40), too_big=0.0, bind_drained=True):
    """A random cluster over every filter, with D candidates (duplicates allowed) each drained of 0 to max_pods pods:
    zone / disk labels, a tainted GPU pool on about one node in gpu_every with 8 GPUs, some cordoned nodes, nodes near
    their pod limit, R - 2 further extended resources; G group rules with the GPU toleration or required zone terms.
    Candidate pods take share[0]-share[1] % of an average node, GPU pods (groups that tolerate the pool) 1-8 GPUs, and
    with probability too_big 9, more than any node has.  bind_drained as cluster() takes it."""
    zones = ["a", "b", "c"]
    extra = [f"example.com/r{i}" for i in range(max(0, R - 2))]
    nodes = []
    for n in range(N):
        gpu = n % gpu_every == 0
        lab = {"zone": zones[int(rng.integers(0, 3))]}
        if rng.random() < 0.5:
            lab["disk"] = "ssd"
        taints = []
        if gpu:
            lab["gpu"] = "h100"
            taints.append({"key": "nvidia.com/gpu", "value": "present", "effect": "NoSchedule"})
        if rng.random() < 0.08:
            taints.append(CORDON)
        alloc = {"pods": int(rng.integers(2, 12))}
        if gpu and R >= 2:
            alloc["nvidia.com/gpu"] = 8
        for r in extra:
            if rng.random() < 0.6:
                alloc[r] = int(rng.integers(0, 6))
        nodes.append(dict(cpu=int(rng.integers(8000, 64000)), mem=int(rng.integers(1 << 30, 1 << 34)), labels=lab,
                          taints=taints, alloc=alloc))
    rules = []
    for g in range(G):
        r = {"tolerations": [TOL_GPU] if g % 2 == 0 else []}
        if g % 3 == 1:
            r["required"] = [[{"key": "zone", "operator": "In", "values": ["a", "b"]}]]
        rules.append(r)
    mc = int(np.mean([n["cpu"] for n in nodes]))
    mm = int(np.mean([n["mem"] for n in nodes]))
    bound = []
    for n in range(N):
        for _ in range(int(rng.integers(0, 3))):
            res = {}
            if "nvidia.com/gpu" in nodes[n]["alloc"] and rng.random() < 0.5:
                res["nvidia.com/gpu"] = int(rng.integers(1, 4))
            bound.append((n, mc * int(rng.integers(2, 15)) // 100, mm // 100 * int(rng.integers(2, 15)), res))
    cands = []
    for _ in range(D):
        n = int(rng.integers(0, N))
        pods = []
        for _ in range(int(rng.integers(0, max_pods + 1))):
            g = int(rng.integers(-1, G))
            res = {}
            if g >= 0 and g % 2 == 0 and R >= 2 and rng.random() < 0.6:
                res["nvidia.com/gpu"] = 9 if rng.random() < too_big else int(rng.integers(1, 9))
            for r in extra:
                if rng.random() < 0.2:
                    res[r] = int(rng.integers(1, 4))
            sel = {"disk": "ssd"} if rng.random() < 0.15 else {}
            pods.append(dict(cpu=mc * int(rng.integers(*share)) // 100, mem=mm // 100 * int(rng.integers(*share)),
                             selector=sel, group=g, res=res))
        cands.append((n, pods))
    names = (["pods", "nvidia.com/gpu"] + extra)[:max(R, 1)]
    d = cluster(nodes, bound, cands, names, bind_drained)
    d["group_rules"] = rules
    return d
