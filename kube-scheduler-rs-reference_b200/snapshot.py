"""Snapshot — Python handle on ks_snapshot (the device-resident node table that replaces
Context.node_store + the per-cell LIST of the reference, /root/reference/src/util.rs:12-15,
src/predicates.rs:21-38).  numpy arrays = host buffers; objects with .data_ptr() (torch tensors) may be
passed for host-pinned or device buffers through select_raw()."""
import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _capi as capi
from ._capi import check, ks_bindings, ks_bound_pods, ks_pods, lib


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    return int(a)


def _c(a, dtype):
    a = np.ascontiguousarray(a, dtype=dtype)
    return a


def replica_outputs(replicas, row_dtype, want_nodes):
    """Output arrays of a replica plan for replicas [T] (uint32): (offset uint64 [T + 1], rows row_dtype [T], node
    int32, score int64).  Spec t's copies go to [offset[t], offset[t+1]) of node / score, which hold no entry when the
    copies exceed capi.KS_REPLICAS_MAX_TOTAL and are None unless want_nodes."""
    offset = np.zeros(len(replicas) + 1, np.uint64)
    np.cumsum(replicas, dtype=np.uint64, out=offset[1:])
    rows = np.zeros(len(replicas), row_dtype)
    if not want_nodes:
        return offset, rows, None, None
    total = int(offset[-1]) if int(offset[-1]) <= capi.KS_REPLICAS_MAX_TOTAL else 0
    return offset, rows, np.empty(total, np.int32), np.empty(total, np.int64)


def node_set(D, members):
    """The set words of a node-affinity expression over a key of D domains (ks_node_rules): bit i for each domain i in
    members, bit D (pass D itself) for "the node lacks the key"."""
    words = np.zeros((D + 64) // 64, np.uint64)
    for i in members:
        words[i // 64] |= np.uint64(1 << (i % 64))
    return words


def node_rules(rules):
    """The ks_node_rules struct of a Snapshot.node_bind rules dict, and the arrays it points into (keep them alive)."""
    hold = []

    def arr(a, dtype):
        if a is None:
            return None
        a = _c(a, dtype).reshape(-1)
        hold.append(a)
        return _ptr(a)
    keys = list(rules.get("rule_keys", ()))
    if len(keys) > capi.KS_NODE_RULES_MAX_KEYS:
        raise ValueError(f"{len(keys)} node-affinity keys (at most {capi.KS_NODE_RULES_MAX_KEYS})")
    terms = list(rules.get("node_terms", ()))
    exprs = [e for t in terms for e in t[2]]
    toff = np.zeros(len(terms) + 1, np.uint32)
    np.cumsum([len(t[2]) for t in terms], out=toff[1:])
    soff = np.zeros(len(exprs) + 1, np.uint64)
    np.cumsum([len(np.asarray(e[1]).reshape(-1)) for e in exprs], out=soff[1:])
    sets = np.concatenate([np.asarray(e[1], np.uint64).reshape(-1) for e in exprs]) if exprs else np.zeros(0, np.uint64)
    nd = [int(d) for _, d in keys] + [0] * (capi.KS_NODE_RULES_MAX_KEYS - len(keys))
    doms = [arr(d, np.int32) for d, _ in keys] + [None] * (capi.KS_NODE_RULES_MAX_KEYS - len(keys))
    nr = capi.ks_node_rules(
        int(rules.get("n_taints", 0)), arr(rules.get("taint_hard"), np.uint64), arr(rules.get("taint_soft"), np.uint64),
        arr(rules.get("tolerate_hard"), np.uint64), arr(rules.get("tolerate_soft"), np.uint64), len(keys),
        (C.c_uint32 * capi.KS_NODE_RULES_MAX_KEYS)(*nd), (C.c_void_p * capi.KS_NODE_RULES_MAX_KEYS)(*doms),
        len(exprs), arr([e[0] for e in exprs], np.uint32), arr(soff, np.uint64), arr(sets, np.uint64), len(terms),
        arr([t[0] for t in terms], np.int32), arr([t[1] for t in terms], np.uint32), arr(toff, np.uint32),
        int(rules.get("weight_taint", 3)), int(rules.get("weight_node_affinity", 2)))
    return nr, hold


def _topology(keys, rows, max_skew, min_domains, existing, what):
    """The ks_spread_multi of keys (a list of K (node_domain, n_domains) pairs) for `rows` specs or groups (`what`):
    max_skew and min_domains [rows, K] or None, existing None or a list of K arrays [rows, n_domains_k].  Returns the
    struct, the arrays it points into (keep them alive) and the K domain counts."""
    k = len(keys)
    if not 1 <= k <= capi.KS_SPREAD_MAX_KEYS:
        raise ValueError(f"{k} topology keys (1 to {capi.KS_SPREAD_MAX_KEYS})")
    doms = [_c(d, np.int32).reshape(-1) for d, _ in keys]
    nd = [int(n) for _, n in keys]

    def per_row(a, name):
        if a is None:
            return None
        a = _c(a, np.uint32).reshape(-1)
        if a.shape[0] != rows * k:
            raise ValueError(f"{name} has {a.shape[0]} entries, {what} x keys {rows * k}")
        return a
    max_skew, min_domains = per_row(max_skew, "max_skew"), per_row(min_domains, "min_domains")
    if existing is not None:
        if len(existing) != k:
            raise ValueError(f"existing has {len(existing)} blocks, keys {k}")
        existing = _c(np.concatenate([np.asarray(e, np.uint32).reshape(rows, n) for e, n in zip(existing, nd)],
                                     axis=1), np.uint32).reshape(-1)
    spread = capi.ks_spread_multi(k, (C.c_uint32 * capi.KS_SPREAD_MAX_KEYS)(*nd),
                                  (C.c_void_p * capi.KS_SPREAD_MAX_KEYS)(*[_ptr(d) for d in doms]),
                                  _ptr(max_skew), _ptr(min_domains), _ptr(existing))
    return spread, (doms, max_skew, min_domains, existing), nd


def _counts(rows, nd, want):
    """The output of per-domain counts [rows, sum(nd)], or None unless want and within KS_SPREAD_MAX_COUNTS"""
    return np.empty((rows, sum(nd)), np.uint32) if want and 0 < rows * sum(nd) <= capi.KS_SPREAD_MAX_COUNTS else None


def _split(counts, nd):
    """counts [rows, sum(nd)] as a list of K arrays [rows, nd[k]], or None"""
    return None if counts is None else np.split(counts, np.cumsum(nd)[:-1], axis=1)


def _pod_affinity(terms, existing_pods):
    """The ks_pod_affinity of terms (a list of (owner group, kind, key index, target groups)) and existing_pods (None
    or (groups, nodes)), and the arrays it points into (keep them alive)."""
    owner = _c([t[0] for t in terms], np.int32)
    kind = _c([t[1] for t in terms], np.uint8)
    key = _c([t[2] for t in terms], np.uint32)
    toff = np.zeros(len(terms) + 1, np.uint64)
    np.cumsum([len(t[3]) for t in terms], out=toff[1:])
    target = _c(np.concatenate([np.asarray(t[3], np.int64).reshape(-1) for t in terms]) if terms else [], np.int32)
    eg, en = (np.zeros(0, np.int32),) * 2 if existing_pods is None else existing_pods
    eg, en = _c(eg, np.int32).reshape(-1), _c(en, np.int32).reshape(-1)
    if eg.shape[0] != en.shape[0]:
        raise ValueError(f"existing pods: {eg.shape[0]} groups, {en.shape[0]} nodes")
    aff = capi.ks_pod_affinity(len(terms), _ptr(owner), _ptr(kind), _ptr(key), _ptr(toff), _ptr(target),
                               eg.shape[0], _ptr(eg), _ptr(en))
    return aff, (owner, kind, key, toff, target, eg, en)


def _rules_arg(rules):
    """The ks_node_rules argument of a rules dict (node_rules) or None (NULL), and what it points into"""
    if rules is None:
        return None, None
    nr, hold = node_rules(rules)
    return C.byref(nr), (nr, hold)


@dataclass
class SelectResult:
    node_idx: np.ndarray
    score: np.ndarray
    feasible_cnt: np.ndarray
    mask: np.ndarray  # uint8 [P, row_bytes] or None
    path: str


class Snapshot:
    def __init__(self, device=0):
        h = C.c_void_p()
        check(lib.ks_snapshot_create(int(device), C.byref(h)), "ks_snapshot_create")
        self._h = h
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            lib.ks_snapshot_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    @property
    def n_nodes(self):
        return int(lib.ks_snapshot_num_nodes(self._h))

    @property
    def label_words(self):
        return int(lib.ks_snapshot_label_words(self._h))

    def set_nodes(self, alloc_cpu, alloc_mem, labels):
        alloc_cpu = _c(alloc_cpu, np.int64)
        alloc_mem = _c(alloc_mem, np.int64)
        labels = _c(labels, np.uint64)
        n = alloc_cpu.shape[0]
        labels = labels.reshape(n, -1) if n else labels.reshape(0, max(1, labels.shape[-1] if labels.ndim > 1 else 1))
        w = labels.shape[1]
        check(lib.ks_snapshot_set_nodes(self._h, n, w, _ptr(alloc_cpu), _ptr(alloc_mem), _ptr(labels)),
              "ks_snapshot_set_nodes")

    def set_bound(self, node_idx, req_cpu, req_mem):
        node_idx = _c(node_idx, np.int32)
        req_cpu = _c(req_cpu, np.int64)
        req_mem = _c(req_mem, np.int64)
        check(lib.ks_snapshot_set_bound(self._h, node_idx.shape[0], _ptr(node_idx), _ptr(req_cpu), _ptr(req_mem)),
              "ks_snapshot_set_bound")

    def apply_bind(self, node_idx, req_cpu, req_mem):
        check(lib.ks_snapshot_apply_bind(self._h, int(node_idx), int(req_cpu), int(req_mem)), "ks_snapshot_apply_bind")

    def free(self):
        n = self.n_nodes
        fc = np.empty(n, np.int64)
        fm = np.empty(n, np.int64)
        check(lib.ks_snapshot_get_free(self._h, _ptr(fc), _ptr(fm)), "ks_snapshot_get_free")
        return fc, fm

    def check_cell(self, req_cpu, req_mem, sel, node_idx):
        sel = _c(sel, np.uint64).reshape(-1)
        return check(lib.ks_check_cell(self._h, int(req_cpu), int(req_mem), _ptr(sel), int(node_idx)), "ks_check_cell")

    def _pods(self, req_cpu, req_mem, sel):
        req_cpu = _c(req_cpu, np.int64)
        req_mem = _c(req_mem, np.int64)
        sel = _c(sel, np.uint64).reshape(req_cpu.shape[0], -1 if req_cpu.shape[0] else self.label_words)
        if sel.shape[1] != self.label_words:
            raise ValueError(f"sel has {sel.shape[1]} words per pod, snapshot has {self.label_words}")
        pods = ks_pods(req_cpu.shape[0], _ptr(req_cpu), _ptr(req_mem), _ptr(sel), capi.KS_MEM_HOST)
        return pods, (req_cpu, req_mem, sel)

    def check_cells(self, req_cpu, req_mem, sel):
        pods, keep = self._pods(req_cpu, req_mem, sel)
        codes = np.empty((pods.n, self.n_nodes), np.uint8)
        check(lib.ks_check_cells(self._h, C.byref(pods), _ptr(codes)), "ks_check_cells")
        return codes

    def select(self, req_cpu, req_mem, sel, policy=capi.KS_SCORE_LEFTOVER, flags=capi.KS_SELECT_AUTO, want_mask=False):
        """Batched select_node_for_pod over host (numpy) pods; returns host results.  policy: KS_SCORE_LEFTOVER,
        KS_SCORE_LEAST_ALLOCATED, KS_SCORE_MOST_ALLOCATED (bin-packing) or KS_SCORE_LEAST_BALANCED (upstream's default
        profile: LeastAllocated + BalancedAllocation), on either kernel path.  Every method here that takes a policy
        takes these four."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        p = int(pods.n)
        idx = np.empty(p, np.int32)
        score = np.empty(p, np.int64)
        cnt = np.empty(p, np.uint32)
        mask = None
        row = capi.mask_row_bytes(self.n_nodes)
        if want_mask:
            mask = np.zeros((p, row), np.uint8)
        out = ks_bindings(_ptr(idx), _ptr(score), _ptr(cnt), capi.KS_MEM_HOST, _ptr(mask), row, capi.KS_MEM_HOST, None, None)
        check(lib.ks_select(self._h, C.byref(pods), int(policy), int(flags), C.byref(out), None), "ks_select")
        return SelectResult(idx, score, cnt, mask, self.last_path())

    def select_raw(self, n_pods, req_cpu, req_mem, sel, pods_space, node_idx, score, cnt, out_space, mask=None,
                   mask_row_bytes=0, mask_space=capi.KS_MEM_DEVICE, policy=capi.KS_SCORE_LEFTOVER,
                   flags=capi.KS_SELECT_AUTO, stream=None, ready_event=None, exchange=None):
        """Pointer-level call (torch tensors / raw addresses); the caller keeps the buffers alive.
        exchange: a multigpu.PeerExchange (fused all-gather of node_idx / score into every rank's gather buffer)."""
        pods = ks_pods(int(n_pods), _ptr(req_cpu), _ptr(req_mem), _ptr(sel), int(pods_space))
        out = ks_bindings(_ptr(node_idx), _ptr(score), _ptr(cnt), int(out_space), _ptr(mask), int(mask_row_bytes),
                          int(mask_space), C.c_void_p(ready_event) if ready_event else None,
                          C.pointer(exchange.desc) if exchange is not None else None)
        check(lib.ks_select(self._h, C.byref(pods), int(policy), int(flags), C.byref(out),
                            C.c_void_p(stream) if stream else None), "ks_select")

    def commit_claims(self, claim_node, req_cpu, req_mem):
        """K3: accept claims per node in arrival order while they fit; decrements free[] on the device."""
        claim_node = _c(claim_node, np.int32)
        req_cpu = _c(req_cpu, np.int64)
        req_mem = _c(req_mem, np.int64)
        acc = np.zeros(claim_node.shape[0], np.uint8)
        check(lib.ks_snapshot_commit_claims(self._h, claim_node.shape[0], _ptr(claim_node), _ptr(req_cpu),
                                            _ptr(req_mem), _ptr(acc)), "ks_snapshot_commit_claims")
        return acc

    def stream_bind(self, req_cpu, req_mem, sel, policy=capi.KS_SCORE_LEFTOVER):
        """One streaming micro-batch: select + commit rounds until every pod is bound or infeasible."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        p = int(pods.n)
        idx = np.empty(p, np.int32)
        score = np.empty(p, np.int64)
        rounds = C.c_uint32()
        check(lib.ks_stream_bind(self._h, C.byref(pods), int(policy), _ptr(idx), _ptr(score), C.byref(rounds)),
              "ks_stream_bind")
        return idx, score, rounds.value

    def gang_bind(self, req_cpu, req_mem, sel, offset, min_member, policy=capi.KS_SCORE_LEFTOVER):
        """Pod groups, all or nothing (ks_gang_bind): group g is pods [offset[g], offset[g+1]) and commits only if at
        least min_member[g] of them are placed.  Returns (node_idx[P], score[P], placed[G], rounds[G])."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        offset = _c(offset, np.uint64).reshape(-1)
        min_member = _c(min_member, np.uint32).reshape(-1)
        g = offset.shape[0] - 1
        if g < 0 or min_member.shape[0] != g:
            raise ValueError(f"need len(offset) >= 1 and len(min_member) == len(offset) - 1 "
                             f"(got {offset.shape[0]} and {min_member.shape[0]})")
        gangs = capi.ks_gangs(g, _ptr(offset), _ptr(min_member))
        p = int(pods.n)
        idx = np.empty(p, np.int32)
        score = np.empty(p, np.int64)
        placed = np.empty(g, np.uint32)
        rounds = np.empty(g, np.uint32)
        check(lib.ks_gang_bind(self._h, C.byref(pods), C.byref(gangs), int(policy), _ptr(idx), _ptr(score),
                               _ptr(placed), _ptr(rounds)), "ks_gang_bind")
        return idx, score, placed, rounds

    def drain_check(self, req_cpu, req_mem, sel, node_idx, offset, policy=capi.KS_SCORE_LEFTOVER, flags=0):
        """Drain simulation (ks_drain_check): candidate d is node node_idx[d] with pods [offset[d], offset[d+1]); each
        candidate's pods are placed in order on the other nodes, against a private copy of free[].  Nothing is charged.
        Returns (placed[D], node_idx[P], score[P]); candidate d is drainable iff placed[d] is its pod count."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        node_idx = _c(node_idx, np.int32).reshape(-1)
        offset = _c(offset, np.uint64).reshape(-1)
        d = node_idx.shape[0]
        if offset.shape[0] != d + 1:
            raise ValueError(f"need len(offset) == len(node_idx) + 1 (got {offset.shape[0]} and {d})")
        cand = capi.ks_drain_candidates(d, _ptr(node_idx), _ptr(offset))
        p = int(pods.n)
        placed = np.empty(d, np.uint32)
        idx = np.empty(p, np.int32)
        score = np.empty(p, np.int64)
        check(lib.ks_drain_check(self._h, C.byref(pods), C.byref(cand), int(policy), int(flags), _ptr(placed),
                                 _ptr(idx), _ptr(score)), "ks_drain_check")
        return placed, idx, score

    def scaleup_estimate(self, req_cpu, req_mem, sel, alloc_cpu, alloc_mem, free_cpu, free_mem, labels, max_nodes,
                         want_nodes=True, want_reasons=True):
        """Scale-up estimate (ks_scaleup_estimate): for every node template, how many new nodes would place which of
        the pods, by first fit in decreasing-size order.  labels is [T, label_words] (the call's own label bits, not the
        snapshot's) and sel [P, label_words].  Nothing is charged.  Returns (rows, best, node, reasons): rows a
        capi.SCALEUP_OPTION_DTYPE record array [T], best the picked template or -1, node int32 [T, P] (the new node's
        ordinal, -1 = not placed; None unless want_nodes), reasons uint32 [P, 4] in ks_explain's columns over the
        templates (None unless want_reasons)."""
        req_cpu, req_mem = _c(req_cpu, np.int64).reshape(-1), _c(req_mem, np.int64).reshape(-1)
        alloc_cpu, alloc_mem = _c(alloc_cpu, np.int64).reshape(-1), _c(alloc_mem, np.int64).reshape(-1)
        free_cpu, free_mem = _c(free_cpu, np.int64).reshape(-1), _c(free_mem, np.int64).reshape(-1)
        max_nodes = _c(max_nodes, np.uint32).reshape(-1)
        t, p = alloc_cpu.shape[0], req_cpu.shape[0]
        labels = _c(labels, np.uint64).reshape(t, -1) if t else None
        sel = _c(sel, np.uint64).reshape(p, -1) if p else None
        w = labels.shape[1] if t else sel.shape[1] if p else 1
        if p and sel.shape[1] != w:
            raise ValueError(f"sel has {sel.shape[1]} words per pod, labels {w}")
        for name, a in (("alloc_mem", alloc_mem), ("free_cpu", free_cpu), ("free_mem", free_mem), ("max_nodes", max_nodes)):
            if a.shape[0] != t:
                raise ValueError(f"{name} has {a.shape[0]} entries, alloc_cpu {t}")
        if req_mem.shape[0] != p:
            raise ValueError(f"req_mem has {req_mem.shape[0]} entries, req_cpu {p}")
        pods = ks_pods(p, _ptr(req_cpu), _ptr(req_mem), _ptr(sel), capi.KS_MEM_HOST)
        tmpl = capi.ks_node_templates(t, w, _ptr(alloc_cpu), _ptr(alloc_mem), _ptr(free_cpu), _ptr(free_mem),
                                      _ptr(labels), _ptr(max_nodes))
        rows = np.zeros(t, capi.SCALEUP_OPTION_DTYPE)
        best = C.c_int32(-1)
        node = np.empty((t, p), np.int32) if want_nodes else None
        why = np.empty((p, 4), np.uint32) if want_reasons else None
        check(lib.ks_scaleup_estimate(self._h, C.byref(pods), C.byref(tmpl), _ptr(rows), C.addressof(best), _ptr(node),
                                      _ptr(why)), "ks_scaleup_estimate")
        return rows, best.value, node, why

    def fit_scaleup_estimate(self, req_cpu, req_mem, sel, alloc_cpu, alloc_mem, free_cpu, free_mem, labels, max_nodes,
                             group, n_groups, rules=None, node_free=None, pod_req=None, want_nodes=True,
                             want_refused=True, want_used=True):
        """scaleup_estimate under the full filter (ks_fit_scaleup_estimate): group [P] and rules as fit_bind takes them
        with the templates as the nodes (rules None = NULL: taint_hard / taint_soft and rule_keys' domains are [T]);
        node_free [R, T] (one empty node of each template) and pod_req [P, R] (int64), or both None (the C call's NULL
        res).  Returns scaleup_estimate's (rows, best, node), then refused uint32 [P, 4] (None unless want_refused)
        and used int64 [T, R] (None unless want_used): the placed pods' requests of each resource."""
        req_cpu, req_mem = _c(req_cpu, np.int64).reshape(-1), _c(req_mem, np.int64).reshape(-1)
        alloc_cpu, alloc_mem = _c(alloc_cpu, np.int64).reshape(-1), _c(alloc_mem, np.int64).reshape(-1)
        free_cpu, free_mem = _c(free_cpu, np.int64).reshape(-1), _c(free_mem, np.int64).reshape(-1)
        max_nodes = _c(max_nodes, np.uint32).reshape(-1)
        t, p = alloc_cpu.shape[0], req_cpu.shape[0]
        labels = _c(labels, np.uint64).reshape(t, -1) if t else None
        sel = _c(sel, np.uint64).reshape(p, -1) if p else None
        w = labels.shape[1] if t else sel.shape[1] if p else 1
        if p and sel.shape[1] != w:
            raise ValueError(f"sel has {sel.shape[1]} words per pod, labels {w}")
        for name, a in (("alloc_mem", alloc_mem), ("free_cpu", free_cpu), ("free_mem", free_mem), ("max_nodes", max_nodes)):
            if a.shape[0] != t:
                raise ValueError(f"{name} has {a.shape[0]} entries, alloc_cpu {t}")
        if req_mem.shape[0] != p:
            raise ValueError(f"req_mem has {req_mem.shape[0]} entries, req_cpu {p}")
        group = _c(group, np.int32).reshape(-1)
        if group.shape[0] != p:
            raise ValueError(f"group has {group.shape[0]} entries, pods {p}")
        if (node_free is None) != (pod_req is None):
            raise ValueError("node_free and pod_req go together")
        br, r = None, 0
        if node_free is not None:
            node_free, pod_req = _c(node_free, np.int64), _c(pod_req, np.int64)
            if node_free.ndim != 2 or node_free.shape[1] != t:
                raise ValueError(f"node_free has shape {node_free.shape}, expected (R, {t})")
            r = node_free.shape[0]
            if pod_req.shape != (p, r):
                raise ValueError(f"pod_req has shape {pod_req.shape}, expected ({p}, {r})")
            br = capi.ks_bind_resources(r, _ptr(node_free), _ptr(pod_req))
        nr, hold = _rules_arg(rules)
        pods = ks_pods(p, _ptr(req_cpu), _ptr(req_mem), _ptr(sel), capi.KS_MEM_HOST)
        tmpl = capi.ks_node_templates(t, w, _ptr(alloc_cpu), _ptr(alloc_mem), _ptr(free_cpu), _ptr(free_mem),
                                      _ptr(labels), _ptr(max_nodes))
        rows = np.zeros(t, capi.SCALEUP_OPTION_DTYPE)
        best = C.c_int32(-1)
        node = np.empty((t, p), np.int32) if want_nodes else None
        refused = np.empty((p, 4), np.uint32) if want_refused else None
        used = np.empty((t, r), np.int64) if want_used else None
        check(lib.ks_fit_scaleup_estimate(self._h, C.byref(pods), _ptr(group), int(n_groups), nr,
                                          None if br is None else C.byref(br), C.byref(tmpl), _ptr(rows),
                                          C.addressof(best), _ptr(node), _ptr(refused), _ptr(used)),
              "ks_fit_scaleup_estimate")
        return rows, best.value, node, refused, used

    def place_replicas(self, req_cpu, req_mem, sel, replicas, policy=capi.KS_SCORE_LEFTOVER, want_nodes=True):
        """Replica placement (ks_place_replicas): spec t (a row of req_cpu / req_mem / sel) asks for replicas[t] copies,
        placed one at a time by ks_select's argmax with the earlier copies bound.  Nothing is charged.  Returns (rows,
        node, score, offset): rows a capi.REPLICA_PLAN_DTYPE record array [T]; node int32 / score int64 [sum replicas],
        spec t's copies in placement order at [offset[t], offset[t+1]) (-1 / 0 past rows['placed'][t]; both None
        unless want_nodes); offset uint64 [T + 1]."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        t = int(pods.n)
        replicas = np.asarray(replicas).reshape(-1)
        if replicas.shape[0] != t:
            raise ValueError(f"replicas has {replicas.shape[0]} entries, specs {t}")
        if t and (replicas.min() < 0 or replicas.max() > 0xFFFFFFFF):
            raise ValueError("replicas must lie in [0, 2^32)")
        replicas = _c(replicas, np.uint32)
        offset, rows, node, score = replica_outputs(replicas, capi.REPLICA_PLAN_DTYPE, want_nodes)
        check(lib.ks_place_replicas(self._h, C.byref(pods), _ptr(replicas), int(policy), _ptr(rows), _ptr(node),
                                    _ptr(score)), "ks_place_replicas")
        return rows, node, score, offset

    def place_replicas_spread(self, req_cpu, req_mem, sel, replicas, node_domain, n_domains, max_skew, min_domains=None,
                              existing=None, policy=capi.KS_SCORE_LEFTOVER, want_nodes=True, want_counts=True):
        """Replica placement under one topology spread constraint (ks_place_replicas_spread, whenUnsatisfiable:
        DoNotSchedule): as place_replicas, but copy r may only go to a node whose domain (node_domain[n] in
        [0, n_domains), -1 = no topology key) keeps the domain's count within max_skew[t] of the minimum over the
        eligible domains.  min_domains [T] and existing [T, n_domains] (matching pods already bound per domain) may be
        None.  Nothing is charged.  Returns (rows, node, score, offset, counts): rows a capi.SPREAD_PLAN_DTYPE record
        array [T]; node / score / offset as place_replicas (node and score None unless want_nodes); counts uint32
        [T, n_domains], the final count per domain (None unless want_counts)."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        t = int(pods.n)
        replicas = np.asarray(replicas).reshape(-1)
        if replicas.shape[0] != t:
            raise ValueError(f"replicas has {replicas.shape[0]} entries, specs {t}")
        if t and (replicas.min() < 0 or replicas.max() > 0xFFFFFFFF):
            raise ValueError("replicas must lie in [0, 2^32)")
        replicas = _c(replicas, np.uint32)
        node_domain = _c(node_domain, np.int32).reshape(-1)
        max_skew = _c(max_skew, np.uint32).reshape(-1)
        if max_skew.shape[0] != t:
            raise ValueError(f"max_skew has {max_skew.shape[0]} entries, specs {t}")
        if min_domains is not None:
            min_domains = _c(min_domains, np.uint32).reshape(-1)
            if min_domains.shape[0] != t:
                raise ValueError(f"min_domains has {min_domains.shape[0]} entries, specs {t}")
        d = int(n_domains)
        if existing is not None:
            existing = _c(existing, np.uint32).reshape(-1)
            if existing.shape[0] != t * d:
                raise ValueError(f"existing has {existing.shape[0]} entries, specs x domains {t * d}")
        spread = capi.ks_spread(d, _ptr(node_domain), _ptr(max_skew), _ptr(min_domains), _ptr(existing))
        offset, rows, node, score = replica_outputs(replicas, capi.SPREAD_PLAN_DTYPE, want_nodes)
        counts = np.empty((t, d), np.uint32) if want_counts and 0 < t * d <= capi.KS_SPREAD_MAX_COUNTS else None
        check(lib.ks_place_replicas_spread(self._h, C.byref(pods), _ptr(replicas), C.byref(spread), int(policy),
                                           _ptr(rows), _ptr(node), _ptr(score), _ptr(counts)),
              "ks_place_replicas_spread")
        return rows, node, score, offset, counts

    def place_replicas_spread_multi(self, req_cpu, req_mem, sel, replicas, keys, max_skew, min_domains=None,
                                    existing=None, policy=capi.KS_SCORE_LEFTOVER, want_nodes=True, want_counts=True):
        """Replica placement under one topology spread constraint per key, every constraint binding at once
        (ks_place_replicas_spread_multi): keys is a list of K (node_domain, n_domains) pairs, max_skew and min_domains
        (None = no minDomains) are [T, K], existing is None or a list of K arrays [T, n_domains_k].  Nothing is charged.
        Returns (rows, node, score, offset, counts): rows a capi.SPREAD_PLAN_DTYPE record array [T, K]; node / score /
        offset as place_replicas; counts a list of K arrays uint32 [T, n_domains_k] (None unless want_counts)."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        t = int(pods.n)
        replicas = np.asarray(replicas).reshape(-1)
        if replicas.shape[0] != t:
            raise ValueError(f"replicas has {replicas.shape[0]} entries, specs {t}")
        if t and (replicas.min() < 0 or replicas.max() > 0xFFFFFFFF):
            raise ValueError("replicas must lie in [0, 2^32)")
        replicas = _c(replicas, np.uint32)
        spread, hold, nd = _topology(keys, t, max_skew, min_domains, existing, "specs")
        offset, _, node, score = replica_outputs(replicas, capi.SPREAD_PLAN_DTYPE, want_nodes)
        rows = np.zeros((t, len(keys)), capi.SPREAD_PLAN_DTYPE)
        counts = _counts(t, nd, want_counts)
        check(lib.ks_place_replicas_spread_multi(self._h, C.byref(pods), _ptr(replicas), C.byref(spread), int(policy),
                                                 _ptr(rows), _ptr(node), _ptr(score), _ptr(counts)),
              "ks_place_replicas_spread_multi")
        return rows, node, score, offset, _split(counts, nd)

    def spread_bind(self, req_cpu, req_mem, sel, group, keys, max_skew, min_domains=None, existing=None,
                    policy=capi.KS_SCORE_LEFTOVER, want_counts=True):
        """Bind a mixed pod queue one pod at a time under each workload's spread constraints (ks_spread_bind): pod p
        belongs to group group[p] (-1 = unconstrained); keys is a list of K (node_domain, n_domains) pairs; max_skew
        [G, K] (0 = the group does not constrain that key), min_domains [G, K] or None, existing None or a list of K
        arrays [G, n_domains_k].  G = len(max_skew).  Charges free[].  Returns (node_idx int32 [P], score int64 [P],
        refused uint32 [P], counts): counts a list of K arrays uint32 [G, n_domains_k] (None unless want_counts)."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        p = int(pods.n)
        group = _c(group, np.int32).reshape(-1)
        if group.shape[0] != p:
            raise ValueError(f"group has {group.shape[0]} entries, pods {p}")
        g = _c(max_skew, np.uint32).reshape(-1, max(len(keys), 1)).shape[0]
        spread, hold, nd = _topology(keys, g, max_skew, min_domains, existing, "groups")
        idx = np.empty(p, np.int32)
        score = np.empty(p, np.int64)
        refused = np.empty(p, np.uint32)
        counts = _counts(g, nd, want_counts)
        check(lib.ks_spread_bind(self._h, C.byref(pods), _ptr(group), g, C.byref(spread), int(policy), _ptr(idx),
                                 _ptr(score), _ptr(refused), _ptr(counts)), "ks_spread_bind")
        return idx, score, refused, _split(counts, nd)

    def affinity_bind(self, req_cpu, req_mem, sel, group, n_groups, keys, terms=(), existing_pods=None, max_skew=None,
                      min_domains=None, existing=None, policy=capi.KS_SCORE_LEFTOVER, want_counts=True):
        """spread_bind with required inter-pod affinity and anti-affinity (ks_affinity_bind): G = n_groups groups;
        terms a list of (owner group, kind KS_POD_AFFINITY / KS_POD_ANTI_AFFINITY, key index, target groups);
        existing_pods None or (groups, nodes) of the bound pods the terms see; max_skew [G, K] or None (no spread
        constraint), min_domains and existing as in spread_bind.  Charges free[].  Returns (node_idx int32 [P], score
        int64 [P], refused uint32 [P, 2] (spread, affinity), counts)."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        p, g = int(pods.n), int(n_groups)
        group = _c(group, np.int32).reshape(-1)
        if group.shape[0] != p:
            raise ValueError(f"group has {group.shape[0]} entries, pods {p}")
        topo, hold, nd = _topology(keys, g, max_skew, min_domains, existing, "groups")
        aff, hold_aff = _pod_affinity(terms, existing_pods)
        idx = np.empty(p, np.int32)
        score = np.empty(p, np.int64)
        refused = np.empty((p, 2), np.uint32)
        counts = _counts(g, nd, want_counts)
        check(lib.ks_affinity_bind(self._h, C.byref(pods), _ptr(group), g, C.byref(topo), C.byref(aff), int(policy),
                                   _ptr(idx), _ptr(score), _ptr(refused), _ptr(counts)), "ks_affinity_bind")
        return idx, score, refused, _split(counts, nd)

    def profile_bind(self, req_cpu, req_mem, sel, group, n_groups, keys, terms=(), existing_pods=None, max_skew=None,
                     min_domains=None, existing=None, policy=capi.KS_SCORE_LEAST_BALANCED, soft_skew=None,
                     soft_all_keys=None, term_weight=None, hard_affinity_weight=1, weight_spread=2, weight_affinity=2,
                     want_counts=True):
        """affinity_bind scored as the default profile (ks_profile_bind): terms may also be
        KS_POD_AFFINITY_PREFERRED / KS_POD_ANTI_AFFINITY_PREFERRED, each with its term_weight [T] (0 for required
        terms); soft_skew [G, K] or None (ScheduleAnyway maxSkew, 0 = none); soft_all_keys [G] or None (all 1).
        Charges free[].  Returns (node_idx int32 [P], score int64 [P], parts int64 [P, 3] (policy, pts, ipa),
        refused uint32 [P, 2], counts, soft_counts); both counts lists of K arrays [G, D_k], or None."""
        return self._scored_bind("ks_profile_bind", (), (), (3, 2), req_cpu, req_mem, sel, group, n_groups, keys,
                                 terms, existing_pods, max_skew, min_domains, existing, policy, soft_skew,
                                 soft_all_keys, term_weight, hard_affinity_weight, weight_spread, weight_affinity,
                                 want_counts)

    def node_bind(self, req_cpu, req_mem, sel, group, n_groups, keys, terms=(), existing_pods=None, max_skew=None,
                  min_domains=None, existing=None, policy=capi.KS_SCORE_LEAST_BALANCED, soft_skew=None,
                  soft_all_keys=None, term_weight=None, hard_affinity_weight=1, weight_spread=2, weight_affinity=2,
                  rules=None, want_counts=True):
        """profile_bind with TaintToleration and NodeAffinity (ks_node_bind).  rules: None (the C call's NULL) or a
        dict with any of n_taints, taint_hard [N], taint_soft [N], tolerate_hard [G], tolerate_soft [G] (uint64 taint
        masks), rule_keys (a list of (node_domain [N], D_k)), node_terms (a list of (owner, weight, [(key, set words
        uint64), ...]); weight 0 = required), weight_taint (default 3) and weight_node_affinity (default 2); see
        node_set for the words.  Returns profile_bind's tuple with parts [P, 5] (policy, pts, ipa, tt, na) and refused
        [P, 4] (taint, node affinity, spread, inter-pod affinity)."""
        nr, hold = _rules_arg(rules)
        return self._scored_bind("ks_node_bind", (nr,), (), (5, 4), req_cpu, req_mem, sel, group, n_groups, keys, terms,
                                 existing_pods, max_skew, min_domains, existing, policy, soft_skew, soft_all_keys,
                                 term_weight, hard_affinity_weight, weight_spread, weight_affinity, want_counts)

    def fit_bind(self, req_cpu, req_mem, sel, group, n_groups, keys, terms=(), existing_pods=None, max_skew=None,
                 min_domains=None, existing=None, policy=capi.KS_SCORE_LEAST_BALANCED, soft_skew=None,
                 soft_all_keys=None, term_weight=None, hard_affinity_weight=1, weight_spread=2, weight_affinity=2,
                 rules=None, node_free=None, pod_req=None, want_counts=True, _gangs=None):
        """node_bind with the pod count and scalar resources of NodeResourcesFit (ks_fit_bind).  node_free [R, N] and
        pod_req [P, R] (int64), or both None (the C call's NULL res); rules as node_bind takes them (None = NULL).
        Returns node_bind's tuple with refused [P, 5] (resources, taint, node affinity, spread, inter-pod affinity),
        then free_r int64 [R, N] after the call."""
        if (node_free is None) != (pod_req is None):
            raise ValueError("node_free and pod_req go together")
        r, br = 0, None
        if node_free is not None:
            node_free = _c(node_free, np.int64)
            pod_req = _c(pod_req, np.int64)
            p = int(np.asarray(req_cpu).reshape(-1).shape[0])
            if node_free.ndim != 2 or node_free.shape[1] != self.n_nodes:
                raise ValueError(f"node_free has shape {node_free.shape}, expected (R, {self.n_nodes})")
            r = node_free.shape[0]
            if pod_req.shape != (p, r):
                raise ValueError(f"pod_req has shape {pod_req.shape}, expected ({p}, {r})")
            br = capi.ks_bind_resources(r, _ptr(node_free), _ptr(pod_req))
        nr, hold = _rules_arg(rules)
        free_r = np.empty((r, self.n_nodes), np.int64)
        entry, mid, outs = "ks_fit_bind", (nr, None if br is None else C.byref(br)), (_ptr(free_r),)
        if _gangs is not None:  # gang_fit_bind's (ks_gangs, placed)
            entry, mid, outs = "ks_gang_fit_bind", mid + (C.byref(_gangs[0]),), outs + (_ptr(_gangs[1]),)
        return self._scored_bind(entry, mid, outs, (5, 5), req_cpu, req_mem, sel, group, n_groups, keys, terms,
                                 existing_pods, max_skew, min_domains, existing, policy, soft_skew, soft_all_keys,
                                 term_weight, hard_affinity_weight, weight_spread, weight_affinity,
                                 want_counts) + (free_r,)

    def gang_fit_bind(self, req_cpu, req_mem, sel, group, n_groups, keys, offset, min_member, terms=(),
                      existing_pods=None, max_skew=None, min_domains=None, existing=None,
                      policy=capi.KS_SCORE_LEAST_BALANCED, soft_skew=None, soft_all_keys=None, term_weight=None,
                      hard_affinity_weight=1, weight_spread=2, weight_affinity=2, rules=None, node_free=None,
                      pod_req=None, want_counts=True):
        """fit_bind with the queue cut into gangs placed all or nothing (ks_gang_fit_bind): gang j is the pods
        [offset[j], offset[j+1]) and keeps its bindings only when at least min_member[j] of them bound; otherwise it
        rolls back and the next gang sees exactly what it saw.  Returns fit_bind's tuple, then placed uint32 [n] (the
        gang's pods that bound, before any rollback)."""
        offset = _c(offset, np.uint64).reshape(-1)
        min_member = _c(min_member, np.uint32).reshape(-1)
        n = offset.shape[0] - 1
        if n < 0 or min_member.shape[0] != n:
            raise ValueError(f"need len(offset) >= 1 and len(min_member) == len(offset) - 1 "
                             f"(got {offset.shape[0]} and {min_member.shape[0]})")
        placed = np.empty(n, np.uint32)
        gangs = capi.ks_gangs(n, _ptr(offset), _ptr(min_member))
        return self.fit_bind(req_cpu, req_mem, sel, group, n_groups, keys, terms, existing_pods, max_skew, min_domains,
                             existing, policy, soft_skew, soft_all_keys, term_weight, hard_affinity_weight,
                             weight_spread, weight_affinity, rules, node_free, pod_req, want_counts,
                             _gangs=(gangs, placed)) + (placed,)

    def _scored_bind(self, entry, mid, outs, widths, req_cpu, req_mem, sel, group, n_groups, keys, terms,
                     existing_pods, max_skew, min_domains, existing, policy, soft_skew, soft_all_keys, term_weight,
                     hard_affinity_weight, weight_spread, weight_affinity, want_counts):
        """The C call `entry` with its scoring, then mid (rules, resources, gangs), the policy, the six outputs every
        scored bind returns (parts and refused of widths words per pod) and outs"""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        p, g = int(pods.n), int(n_groups)
        group = _c(group, np.int32).reshape(-1)
        if group.shape[0] != p:
            raise ValueError(f"group has {group.shape[0]} entries, pods {p}")
        topo, hold, nd = _topology(keys, g, max_skew, min_domains, existing, "groups")
        aff, hold_aff = _pod_affinity(terms, existing_pods)

        def per_group(a, dtype, width, name):
            if a is None:
                return None
            a = _c(a, dtype).reshape(-1)
            if a.shape[0] != g * width:
                raise ValueError(f"{name} has {a.shape[0]} entries, expected {g * width}")
            return a
        soft_skew = per_group(soft_skew, np.uint32, len(keys), "soft_skew")
        soft_all_keys = per_group(soft_all_keys, np.uint8, 1, "soft_all_keys")
        if term_weight is not None:
            term_weight = _c(term_weight, np.uint32).reshape(-1)
            if term_weight.shape[0] != len(terms):
                raise ValueError(f"term_weight has {term_weight.shape[0]} entries, terms {len(terms)}")
        scoring = capi.ks_bind_scoring(_ptr(soft_skew), _ptr(soft_all_keys), _ptr(term_weight),
                                       int(hard_affinity_weight), int(weight_spread), int(weight_affinity))
        idx = np.empty(p, np.int32)
        score = np.empty(p, np.int64)
        parts = np.empty((p, widths[0]), np.int64)
        refused = np.empty((p, widths[1]), np.uint32)
        counts, soft = _counts(g, nd, want_counts), _counts(g, nd, want_counts)
        check(getattr(lib, entry)(self._h, C.byref(pods), _ptr(group), g, C.byref(topo), C.byref(aff),
                                  C.byref(scoring), *mid, int(policy), _ptr(idx), _ptr(score), _ptr(parts),
                                  _ptr(refused), _ptr(counts), _ptr(soft), *outs), entry)
        return idx, score, parts, refused, _split(counts, nd), _split(soft, nd)

    def select_sampling(self, req_cpu, req_mem, sel, attempts=capi.KS_REFERENCE_ATTEMPTS, seed=0, first_pod_index=0):
        """The reference's own policy (src/main.rs:49-71), seeded: (node_idx, attempts_used, draw_node, draw_code)."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        p = int(pods.n)
        idx = np.empty(p, np.int32)
        used = np.empty(p, np.uint32)
        dn = np.empty((p, attempts), np.int32)
        dc = np.empty((p, attempts), np.uint8)
        check(lib.ks_select_sampling(self._h, C.byref(pods), int(attempts), int(seed), int(first_pod_index), _ptr(idx),
                                     _ptr(used), _ptr(dn), _ptr(dc)), "ks_select_sampling")
        return idx, used, dn, dc

    def explain(self, req_cpu, req_mem, sel):
        """Per-pod rejection counts (ks_explain) over host (numpy) pods: uint32 [P, 4] with columns insufficient_cpu,
        insufficient_memory, not_enough_resources, node_selector_mismatch."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        out = np.empty((int(pods.n), 4), np.uint32)
        check(lib.ks_explain(self._h, C.byref(pods), _ptr(out), capi.KS_MEM_HOST, None), "ks_explain")
        return out

    def explain_raw(self, n_pods, req_cpu, req_mem, sel, pods_space, out, out_space, stream=None):
        """Pointer-level ks_explain (torch tensors / raw addresses); out holds n_pods x 16 bytes.  The caller keeps the
        buffers alive; with device pods and output the call returns after enqueue on `stream`."""
        pods = ks_pods(int(n_pods), _ptr(req_cpu), _ptr(req_mem), _ptr(sel), int(pods_space))
        check(lib.ks_explain(self._h, C.byref(pods), _ptr(out), int(out_space), C.c_void_p(stream) if stream else None),
              "ks_explain")

    def select_topk(self, req_cpu, req_mem, sel, k, policy=capi.KS_SCORE_LEFTOVER):
        """The k best feasible nodes per pod (ks_select_topk) over host (numpy) pods: node_idx int32 [P, k] (-1 past the
        feasible count), score int64 [P, k] (0 there), feasible_cnt uint32 [P].  Entry 0 of a row is select()'s pick."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        p = int(pods.n)
        idx = np.empty((p, int(k)), np.int32)
        score = np.empty((p, int(k)), np.int64)
        cnt = np.empty(p, np.uint32)
        check(lib.ks_select_topk(self._h, C.byref(pods), int(policy), int(k), _ptr(idx), _ptr(score), _ptr(cnt),
                                 capi.KS_MEM_HOST, None), "ks_select_topk")
        return idx, score, cnt

    def select_topk_raw(self, n_pods, req_cpu, req_mem, sel, pods_space, k, node_idx, score, cnt, out_space,
                        policy=capi.KS_SCORE_LEFTOVER, stream=None):
        """Pointer-level ks_select_topk (torch tensors / raw addresses); node_idx / score hold n_pods x k entries, cnt
        n_pods (score and cnt may be None).  The caller keeps the buffers alive; with device pods and outputs the call
        returns after enqueue on `stream`."""
        pods = ks_pods(int(n_pods), _ptr(req_cpu), _ptr(req_mem), _ptr(sel), int(pods_space))
        check(lib.ks_select_topk(self._h, C.byref(pods), int(policy), int(k), _ptr(node_idx), _ptr(score), _ptr(cnt),
                                 int(out_space), C.c_void_p(stream) if stream else None), "ks_select_topk")

    @staticmethod
    def _bound(node_idx, req_cpu, req_mem, priority):
        arrs = (_c(node_idx, np.int32), _c(req_cpu, np.int64), _c(req_mem, np.int64), _c(priority, np.int32))
        return ks_bound_pods(arrs[0].shape[0], *[_ptr(a) for a in arrs]), arrs

    def preempt(self, req_cpu, req_mem, sel, priority, bound_node, bound_cpu, bound_mem, bound_priority, max_victims):
        """Priority preemption (ks_preempt) over host (numpy) pods.  The bound list (node, requests, priority) must be
        the one that produced free[].  Returns (rows, victims): rows = PREEMPTION_DTYPE records [P] (node_idx -1 = no
        plan), victims = int32 [P, max_victims] bound indices in visit order, -1 past n_victims."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        priority = _c(priority, np.int32)
        bound, keep_b = self._bound(bound_node, bound_cpu, bound_mem, bound_priority)
        p = int(pods.n)
        rows = np.empty(p, capi.PREEMPTION_DTYPE)
        victims = np.empty((p, int(max_victims)), np.int32)
        check(lib.ks_preempt(self._h, C.byref(pods), _ptr(priority), C.byref(bound), int(max_victims), _ptr(rows),
                             _ptr(victims), capi.KS_MEM_HOST, None), "ks_preempt")
        return rows, victims

    def preempt_raw(self, n_pods, req_cpu, req_mem, sel, pods_space, priority, bound, max_victims, out, victims,
                    out_space, stream=None):
        """Pointer-level ks_preempt (torch tensors / raw addresses): priority in pods_space; bound = (node, cpu, mem,
        priority) host arrays; out holds n_pods x 32 bytes, victims n_pods x max_victims int32 (may be None).  With device
        pods and outputs the call returns after enqueue on `stream`."""
        pods = ks_pods(int(n_pods), _ptr(req_cpu), _ptr(req_mem), _ptr(sel), int(pods_space))
        b, keep_b = self._bound(*bound)
        check(lib.ks_preempt(self._h, C.byref(pods), _ptr(priority), C.byref(b), int(max_victims), _ptr(out),
                             _ptr(victims), int(out_space), C.c_void_p(stream) if stream else None), "ks_preempt")

    def fit_preempt(self, req_cpu, req_mem, sel, priority, group, n_groups, bound_node, bound_cpu, bound_mem,
                    bound_priority, max_victims, rules=None, node_free=None, pod_req=None, bound_req=None):
        """preempt under the full filter (ks_fit_preempt): group [P] and rules as fit_bind takes them (rules None =
        NULL); node_free [R, N], pod_req [P, R] and bound_req [B, R] (int64), or all three None (the C call's NULL res).
        Returns preempt's (rows, victims), then unresolvable uint32 [P]: the nodes no eviction can open to the pod."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        p = int(pods.n)
        priority = _c(priority, np.int32).reshape(-1)
        group = _c(group, np.int32).reshape(-1)
        if priority.shape[0] != p or group.shape[0] != p:
            raise ValueError(f"priority has {priority.shape[0]} and group {group.shape[0]} entries, pods {p}")
        bound, keep_b = self._bound(bound_node, bound_cpu, bound_mem, bound_priority)
        if (node_free is None) != (pod_req is None) or (node_free is None) != (bound_req is None):
            raise ValueError("node_free, pod_req and bound_req go together")
        br, r = None, 0
        if node_free is not None:
            node_free, pod_req, bound_req = _c(node_free, np.int64), _c(pod_req, np.int64), _c(bound_req, np.int64)
            if node_free.ndim != 2 or node_free.shape[1] != self.n_nodes:
                raise ValueError(f"node_free has shape {node_free.shape}, expected (R, {self.n_nodes})")
            r = node_free.shape[0]
            if pod_req.shape != (p, r):
                raise ValueError(f"pod_req has shape {pod_req.shape}, expected ({p}, {r})")
            if bound_req.shape != (int(bound.n), r):
                raise ValueError(f"bound_req has shape {bound_req.shape}, expected ({int(bound.n)}, {r})")
            br = capi.ks_bind_resources(r, _ptr(node_free), _ptr(pod_req))
        nr, hold = _rules_arg(rules)
        rows = np.empty(p, capi.PREEMPTION_DTYPE)
        victims = np.empty((p, int(max_victims)), np.int32)
        unres = np.empty(p, np.uint32)
        check(lib.ks_fit_preempt(self._h, C.byref(pods), _ptr(group), int(n_groups), nr,
                                 None if br is None else C.byref(br), _ptr(priority), C.byref(bound),
                                 _ptr(bound_req), int(max_victims), _ptr(rows), _ptr(victims), _ptr(unres)),
              "ks_fit_preempt")
        return rows, victims, unres

    def fit_drain_check(self, req_cpu, req_mem, sel, group, n_groups, node_idx, offset, policy=capi.KS_SCORE_LEFTOVER,
                        flags=0, rules=None, node_free=None, pod_req=None, want_refused=True):
        """drain_check under the full filter (ks_fit_drain_check): group [P] and rules as fit_bind takes them (rules
        None = NULL); node_free [R, N] and pod_req [P, R] (int64), or both None (the C call's NULL res).  Returns
        drain_check's (placed[D], node_idx[P], score[P]), then refused uint32 [D, 4] (None unless want_refused): why
        each stopped candidate's stopping pod found no destination."""
        pods, keep = self._pods(req_cpu, req_mem, sel)
        p = int(pods.n)
        group = _c(group, np.int32).reshape(-1)
        if group.shape[0] != p:
            raise ValueError(f"group has {group.shape[0]} entries, pods {p}")
        node_idx = _c(node_idx, np.int32).reshape(-1)
        offset = _c(offset, np.uint64).reshape(-1)
        d = node_idx.shape[0]
        if offset.shape[0] != d + 1:
            raise ValueError(f"need len(offset) == len(node_idx) + 1 (got {offset.shape[0]} and {d})")
        if (node_free is None) != (pod_req is None):
            raise ValueError("node_free and pod_req go together")
        br = None
        if node_free is not None:
            node_free, pod_req = _c(node_free, np.int64), _c(pod_req, np.int64)
            if node_free.ndim != 2 or node_free.shape[1] != self.n_nodes:
                raise ValueError(f"node_free has shape {node_free.shape}, expected (R, {self.n_nodes})")
            r = node_free.shape[0]
            if pod_req.shape != (p, r):
                raise ValueError(f"pod_req has shape {pod_req.shape}, expected ({p}, {r})")
            br = capi.ks_bind_resources(r, _ptr(node_free), _ptr(pod_req))
        nr, hold = _rules_arg(rules)
        cand = capi.ks_drain_candidates(d, _ptr(node_idx), _ptr(offset))
        placed = np.empty(d, np.uint32)
        idx = np.empty(p, np.int32)
        score = np.empty(p, np.int64)
        refused = np.empty((d, 4), np.uint32) if want_refused else None
        check(lib.ks_fit_drain_check(self._h, C.byref(pods), _ptr(group), int(n_groups), nr,
                                     None if br is None else C.byref(br), C.byref(cand), int(policy), int(flags),
                                     _ptr(placed), _ptr(idx), _ptr(score), _ptr(refused)), "ks_fit_drain_check")
        return placed, idx, score, refused

    def last_timings(self):
        ms = (C.c_float * 3)()
        check(lib.ks_last_timings(self._h, ms), "ks_last_timings")
        return float(ms[0]), float(ms[1]), float(ms[2])

    def last_path(self):
        return lib.ks_last_path(self._h).decode()

    def last_trace(self):
        """Timeline of the last bit-parallel select (ks_last_trace; needs KS_TRACE=1 in the environment): microseconds
        from the start of the pod-rank kernel, {name: (start, end)}; kernels that did not run are left out."""
        ns = (C.c_uint64 * 16)()
        check(lib.ks_last_trace(self._h, ns), "ks_last_trace")
        t0 = ns[0]
        out = {}
        for name, a, b in (("pod_ranks", 0, 1), ("argmax1", 2, 3), ("argmax2", 4, 5), ("mask", 6, 7)):
            if ns[a] and ns[b]:
                out[name] = ((ns[a] - t0) / 1e3, (ns[b] - t0) / 1e3)
        if ns[8]:
            out["mask_first_cta_end"] = (ns[8] - t0) / 1e3
        out["t0_ns"] = int(t0)
        return out

    def exchange_check(self):
        """Synchronise and raise if a fused all-gather (ks_exchange) timed out waiting for a peer."""
        check(lib.ks_exchange_check(self._h), "ks_exchange_check")


class Stream:
    """ks_stream: the reference's Controller queue in front of one snapshot (asynchronous submit / poll)."""

    def __init__(self, snap, policy=capi.KS_SCORE_LEFTOVER, max_batch=0):
        h = C.c_void_p()
        check(lib.ks_stream_open(snap._h, int(policy), int(max_batch), C.byref(h)), "ks_stream_open")
        self._h, self._snap = h, snap
        self._cap = 4096
        self._t = np.empty(self._cap, np.uint64)
        self._i = np.empty(self._cap, np.int32)
        self._s = np.empty(self._cap, np.int64)

    def submit(self, req_cpu, req_mem, sel, tickets):
        req_cpu, req_mem = _c(req_cpu, np.int64), _c(req_mem, np.int64)
        sel, tickets = _c(sel, np.uint64), _c(tickets, np.uint64)
        check(lib.ks_stream_submit(self._h, req_cpu.shape[0], _ptr(req_cpu), _ptr(req_mem), _ptr(sel), _ptr(tickets)),
              "ks_stream_submit")

    def poll(self):
        """(tickets, node_idx, score) of the pods finished since the last poll (possibly empty); never blocks."""
        n = C.c_uint64()
        check(lib.ks_stream_poll(self._h, self._cap, _ptr(self._t), _ptr(self._i), _ptr(self._s), C.byref(n)),
              "ks_stream_poll")
        k = int(n.value)
        return self._t[:k].copy(), self._i[:k].copy(), self._s[:k].copy()

    def flush(self):
        check(lib.ks_stream_flush(self._h), "ks_stream_flush")

    def stats(self):
        b, r, m = C.c_uint64(), C.c_uint64(), C.c_uint64()
        lib.ks_stream_stats(self._h, C.byref(b), C.byref(r), C.byref(m))
        return int(b.value), int(r.value), int(m.value)

    def close(self):
        if getattr(self, "_h", None):
            lib.ks_stream_close(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()
