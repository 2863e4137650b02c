"""Python face of the C++ host layer (include/ksched_host.h): the reference's surface over Pod/Node OBJECTS —
check_node_validity / select_node_for_pod (batched) / reconcile, plus the quantity parser and packer."""
import ctypes as C

import numpy as np

from . import _capi as capi
from ._capi import _proto, check, lib
from .objects import ks_node_obj, ks_pod_obj
from .snapshot import replica_outputs

_vp = C.c_void_p
for _name, _res, _args in [
    ("ksh_parse_cpu_millicores", C.c_int, [C.c_char_p, C.POINTER(C.c_int64)]),
    ("ksh_parse_memory_bytes", C.c_int, [C.c_char_p, C.POINTER(C.c_int64)]),
    ("ksh_total_pod_resources", C.c_int, [_vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    ("ksh_is_pod_bound", C.c_int, [_vp]),
    ("ksh_context_create", C.c_int, [C.c_int, C.POINTER(_vp)]),
    ("ksh_context_destroy", None, [_vp]),
    ("ksh_context_set_nodes", C.c_int, [_vp, _vp, C.c_uint32]),
    ("ksh_context_set_cluster_pods", C.c_int, [_vp, _vp, C.c_uint64]),
    ("ksh_context_upsert_node", C.c_int, [_vp, _vp, C.POINTER(C.c_uint32)]),
    ("ksh_context_remove_node", C.c_int, [_vp, C.c_char_p]),
    ("ksh_context_pod_bound", C.c_int, [_vp, _vp]),
    ("ksh_context_pod_deleted", C.c_int, [_vp, _vp]),
    ("ksh_context_node_name", C.c_char_p, [_vp, C.c_uint32]),
    ("ksh_context_num_nodes", C.c_uint32, [_vp]),
    ("ksh_context_label_words", C.c_uint32, [_vp]),
    ("ksh_context_num_bound", C.c_uint64, [_vp]),
    ("ksh_context_export_packed", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("ksh_context_snapshot", _vp, [_vp]),
    ("ksh_pack_pods", C.c_int, [_vp, _vp, C.c_uint64, _vp, _vp, _vp, C.c_uint32]),
    ("ksh_check_node_validity", C.c_int, [_vp, _vp, C.c_uint32]),
    ("ksh_select_nodes", C.c_int, [_vp, _vp, C.c_uint64, C.c_int, _vp, _vp, _vp]),
    ("ksh_rank_nodes", C.c_int, [_vp, _vp, C.c_uint64, C.c_int, C.c_uint32, _vp, _vp, _vp]),
    ("ksh_select_node_for_pod", C.c_int, [_vp, _vp, C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint64, _vp, _vp, _vp, _vp]),
    ("ksh_reconcile_batch", C.c_int, [_vp, _vp, C.c_uint64, C.c_int, _vp, _vp, _vp, C.c_size_t, _vp, C.POINTER(C.c_uint32)]),
    ("ksh_reconcile", C.c_int, [_vp, _vp, C.c_int, C.POINTER(C.c_int32), C.c_char_p, C.c_size_t]),
    ("ksh_explain_pods", C.c_int, [_vp, _vp, C.c_uint64, _vp, _vp, C.c_size_t, _vp]),
    ("ksh_format_unschedulable", C.c_int, [C.c_uint32, C.POINTER(capi.ks_pod_reasons), _vp, C.c_size_t]),
    ("ksh_context_set_pod_priorities", C.c_int, [_vp, _vp, _vp, C.c_uint64]),
    ("ksh_preempt_pods", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_uint32, _vp, _vp, C.c_size_t, _vp]),
    ("ksh_reconcile_gangs", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_uint64, _vp, C.c_int, _vp, _vp, _vp, _vp,
                                      C.c_size_t, _vp]),
    ("ksh_drain_nodes", C.c_int, [_vp, _vp, C.c_uint64, _vp, _vp, C.c_int, C.c_uint32, _vp, _vp]),
    ("ksh_scaleup_estimate", C.c_int, [_vp, _vp, C.c_uint64, _vp, _vp, C.c_uint64, _vp, C.c_uint64, _vp, _vp, _vp, _vp]),
    ("ksh_place_replicas", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_int, _vp, _vp, _vp]),
    ("ksh_context_topology_domains", C.c_int, [_vp, C.c_char_p, _vp, C.POINTER(C.c_uint32), _vp, C.c_size_t, _vp]),
    ("ksh_place_replicas_spread", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_char_p, _vp, _vp, _vp, _vp, C.c_int, _vp,
                                            _vp, _vp, _vp]),
    ("ksh_place_replicas_spread_multi", C.c_int, [_vp, _vp, C.c_uint64, _vp, _vp, C.c_uint32, _vp, _vp, _vp, _vp,
                                                  C.c_int, _vp, _vp, _vp, _vp]),
    ("ksh_reconcile_spread", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_uint32, _vp, C.c_uint32, _vp, _vp, _vp, _vp, C.c_int,
                                       _vp, _vp, _vp, C.c_size_t, _vp]),
    ("ksh_reconcile_affinity", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_uint32, _vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp,
                                         C.c_int, _vp, _vp, _vp, C.c_size_t, _vp]),
    ("ksh_reconcile_profile", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_uint32, _vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp,
                                        _vp, C.c_int, _vp, _vp, _vp, C.c_size_t, _vp]),
    ("ksh_context_set_node_taints", C.c_int, [_vp, _vp, _vp, _vp, C.c_uint64]),
    ("ksh_compile_node_rules", C.c_int, [_vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp]),
    ("ksh_reconcile_nodes", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_uint32, _vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp,
                                      _vp, _vp, C.c_int, _vp, _vp, _vp, C.c_size_t, _vp]),
    ("ksh_compile_resources", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_size_t, _vp, _vp]),
    ("ksh_reconcile_fit", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_uint32, _vp, C.c_uint32, _vp, _vp, _vp, _vp, _vp,
                                    _vp, _vp, C.c_int, _vp, _vp, _vp, C.c_size_t, _vp]),
    ("ksh_reconcile_fit_gangs", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_uint32, _vp, C.c_uint32, _vp, _vp, _vp, _vp,
                                          _vp, _vp, _vp, _vp, C.c_uint64, _vp, C.c_int, _vp, _vp, _vp, _vp,
                                          C.c_size_t, _vp]),
    ("ksh_preempt_fit_pods", C.c_int, [_vp, _vp, C.c_uint64, _vp, C.c_uint32, _vp, _vp, C.c_uint32, _vp, _vp,
                                       C.c_size_t, _vp]),
    ("ksh_drain_fit_nodes", C.c_int, [_vp, _vp, C.c_uint64, _vp, _vp, _vp, C.c_uint32, _vp, C.c_int, C.c_uint32, _vp,
                                      _vp, _vp]),
    ("ksh_scaleup_fit_estimate", C.c_int, [_vp, _vp, C.c_uint64, _vp, _vp, _vp, _vp, C.c_uint64, _vp, C.c_uint64, _vp,
                                           C.c_uint32, _vp, _vp, _vp, _vp, _vp]),
]:
    _proto(_name, _res, *_args)

KSH_DEVICE_NONE = -1  # packing-only context: objects -> SoA arrays on the host, no predicate is ever evaluated
KSH_RECONCILE_OK, KSH_RECONCILE_NO_NODE_FOUND, KSH_RECONCILE_BINDING_OBJECT_FAILED = 0, 1, 2
KSH_RECONCILE_GANG_UNSATISFIED = 4
KSH_RECONCILE_SPREAD_UNSATISFIED = 5
KSH_RECONCILE_AFFINITY_UNSATISFIED = 6
KSH_RECONCILE_NODE_RULES_UNSATISFIED = 7
KSH_RECONCILE_INSUFFICIENT_RESOURCES = 8


class ksh_taint(C.Structure):
    _fields_ = [("key", C.c_char_p), ("value", C.c_char_p), ("effect", C.c_char_p)]


class ksh_toleration(C.Structure):
    _fields_ = [("key", C.c_char_p), ("op", C.c_char_p), ("value", C.c_char_p), ("effect", C.c_char_p)]


class ksh_node_selector_requirement(C.Structure):
    _fields_ = [("key", C.c_char_p), ("op", C.c_char_p), ("values", C.c_void_p), ("n_values", C.c_uint32)]


class ksh_node_rules(C.Structure):
    _fields_ = [("toleration_offset", C.c_void_p), ("tolerations", C.c_void_p), ("n_terms", C.c_uint32),
                ("term_owner", C.c_void_p), ("term_weight", C.c_void_p), ("term_req_offset", C.c_void_p),
                ("requirements", C.c_void_p), ("weight_taint", C.c_uint32), ("weight_node_affinity", C.c_uint32)]


def _b(s):
    return None if s is None else s.encode()


def node_rules(group_rules, weight_taint=3, weight_node_affinity=2):
    """The ksh_node_rules of per-group rule dicts, and the objects its pointers reach (keep them alive).  group_rules[g]:
    {"tolerations": [{"key", "operator", "value", "effect"}, ...], "required": [term, ...] or None,
    "preferred": [(weight, term), ...]}, a term a list of {"key", "operator", "values"}."""
    hold = []
    tols = [t for r in group_rules for t in r.get("tolerations", ())]
    toff = np.zeros(len(group_rules) + 1, np.uint64)
    np.cumsum([len(r.get("tolerations", ())) for r in group_rules], out=toff[1:])
    tarr = (ksh_toleration * max(len(tols), 1))(*[ksh_toleration(_b(t.get("key", "")), _b(t.get("operator", "")),
                                                                 _b(t.get("value", "")), _b(t.get("effect", "")))
                                                  for t in tols])
    terms = []  # (owner, weight, requirements)
    for g, r in enumerate(group_rules):
        terms += [(g, 0, t) for t in (r.get("required") or [])]
        terms += [(g, int(w), t) for w, t in r.get("preferred", ())]
    reqs = [q for _, _, t in terms for q in t]
    roff = np.zeros(len(terms) + 1, np.uint64)
    np.cumsum([len(t) for _, _, t in terms], out=roff[1:])
    rarr = (ksh_node_selector_requirement * max(len(reqs), 1))()
    for i, q in enumerate(reqs):
        vals = (C.c_char_p * max(len(q.get("values", ())), 1))(*[_b(v) for v in q.get("values", ())])
        hold.append(vals)
        rarr[i] = ksh_node_selector_requirement(_b(q["key"]), _b(q["operator"]), C.cast(vals, _vp),
                                                len(q.get("values", ())))
    owner = np.ascontiguousarray([t[0] for t in terms], np.int32)
    weight = np.ascontiguousarray([t[1] for t in terms], np.uint32)
    hold += [toff, tarr, rarr, roff, owner, weight]
    nr = ksh_node_rules(toff.ctypes.data, C.addressof(tarr), len(terms), owner.ctypes.data, weight.ctypes.data,
                        roff.ctypes.data, C.addressof(rarr), int(weight_taint), int(weight_node_affinity))
    return nr, hold


def _scoring(n_groups, k, n_terms, soft_skew, soft_all_keys, term_weight, hard_affinity_weight, weight_spread,
             weight_affinity):
    """The ks_bind_scoring of the reconcile calls that score, and the arrays it points into (keep them alive):
    soft_skew [n_groups, K], soft_all_keys [n_groups] and term_weight [n_terms], each None or of exactly that length."""
    def arr(a, dtype, n, name):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype).reshape(-1)
        if a.shape[0] != n:
            raise ValueError(f"{name} has {a.shape[0]} entries, expected {n}")
        return a
    hold = (arr(soft_skew, np.uint32, n_groups * k, "soft_skew"),
            arr(soft_all_keys, np.uint8, n_groups, "soft_all_keys"), arr(term_weight, np.uint32, n_terms, "term_weight"))
    scoring = capi.ks_bind_scoring(*[None if a is None else a.ctypes.data for a in hold], int(hard_affinity_weight),
                                   int(weight_spread), int(weight_affinity))
    return scoring, hold


class ksh_pod_affinity(C.Structure):
    _fields_ = [("n_terms", C.c_uint32), ("owner", C.c_void_p), ("kind", C.c_void_p), ("key", C.c_void_p),
                ("target_offset", C.c_void_p), ("target", C.c_void_p), ("n_existing", C.c_uint64),
                ("existing_group", C.c_void_p), ("existing_node_name", C.c_void_p)]


def _addr(arr, i=0):
    return C.addressof(arr) + i * C.sizeof(arr._type_)


def _string_list(buf, off, counts=None):
    """Decode a string-list output (include/ksched_host.h): entry i starts at byte off[i] of buf (-1 = no entry) and
    holds counts[i] NUL-terminated strings, or one when counts is None.  Returns per entry a str (a list of str with
    counts) or None."""
    out = []
    for i, o in enumerate(off.tolist()):
        if o < 0:
            out.append(None)
            continue
        at, strs = C.addressof(buf) + o, []
        for _ in range(1 if counts is None else int(counts[i])):
            strs.append(C.string_at(at))
            at += len(strs[-1]) + 1
        out.append(strs[0].decode() if counts is None else [k.decode() for k in strs])
    return out


def parse_cpu_millicores(s):
    out = C.c_int64()
    rc = lib.ksh_parse_cpu_millicores(s.encode() if isinstance(s, str) else s, C.byref(out))
    return rc, out.value


def parse_memory_bytes(s):
    out = C.c_int64()
    rc = lib.ksh_parse_memory_bytes(s.encode() if isinstance(s, str) else s, C.byref(out))
    return rc, out.value


def total_pod_resources(pods, i=0):
    c, m = C.c_int64(), C.c_int64()
    rc = lib.ksh_total_pod_resources(_addr(pods, i), C.byref(c), C.byref(m))
    return rc, c.value, m.value


def is_pod_bound(pods, i=0):
    return bool(lib.ksh_is_pod_bound(_addr(pods, i)))


def format_unschedulable(n_nodes, reasons, cap=256):
    """FailedScheduling message for one pod's counts (4 ints in ks_pod_reasons order): (full length, text in cap bytes)."""
    r = capi.ks_pod_reasons(*[int(x) for x in reasons])
    buf = C.create_string_buffer(max(cap, 1))
    n = check(lib.ksh_format_unschedulable(int(n_nodes), C.byref(r), C.addressof(buf) if cap else None, int(cap)),
              "ksh_format_unschedulable")
    return n, buf.value.decode()


class Context:
    """ksh_context = the reference's Context{client, node_store} for this path (src/util.rs:12-15).  Every method that
    takes a policy passes it through to the packed call: KS_SCORE_LEFTOVER, KS_SCORE_LEAST_ALLOCATED,
    KS_SCORE_MOST_ALLOCATED (bin-packing) or KS_SCORE_LEAST_BALANCED (upstream's default profile)."""

    def __init__(self, device=0):
        h = _vp()
        check(lib.ksh_context_create(int(device), C.byref(h)), "ksh_context_create")
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            lib.ksh_context_destroy(self._h)
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

    def set_nodes(self, nodes, n):
        check(lib.ksh_context_set_nodes(self._h, C.addressof(nodes), n), "ksh_context_set_nodes")

    def set_cluster_pods(self, pods, n):
        check(lib.ksh_context_set_cluster_pods(self._h, C.addressof(pods), n), "ksh_context_set_cluster_pods")

    @property
    def label_words(self):
        return int(lib.ksh_context_label_words(self._h))

    @property
    def n_nodes(self):
        return int(lib.ksh_context_num_nodes(self._h))

    @property
    def num_bound(self):
        return int(lib.ksh_context_num_bound(self._h))

    def upsert_node(self, nodes, i=0):
        idx = C.c_uint32()
        check(lib.ksh_context_upsert_node(self._h, _addr(nodes, i), C.byref(idx)), "ksh_context_upsert_node")
        return idx.value

    def remove_node(self, name):
        check(lib.ksh_context_remove_node(self._h, name.encode()), "ksh_context_remove_node")

    def pod_bound(self, pods, i=0):
        check(lib.ksh_context_pod_bound(self._h, _addr(pods, i)), "ksh_context_pod_bound")

    def pod_deleted(self, pods, i=0):
        check(lib.ksh_context_pod_deleted(self._h, _addr(pods, i)), "ksh_context_pod_deleted")

    def node_name(self, idx):
        n = lib.ksh_context_node_name(self._h, int(idx))
        return None if n is None else n.decode()

    def pack_pods(self, pods, n):
        rc_ = np.empty(n, np.int64)
        rm_ = np.empty(n, np.int64)
        sel = np.zeros((n, 8), np.uint64)
        w = check(lib.ksh_pack_pods(self._h, C.addressof(pods), n, rc_.ctypes.data, rm_.ctypes.data, sel.ctypes.data,
                                    8), "ksh_pack_pods")
        return rc_, rm_, np.ascontiguousarray(sel[:, :w])

    def export_packed(self):
        """(alloc_cpu, alloc_mem, labels[N,W], bound_node, bound_cpu, bound_mem): what the next device upload sends."""
        n, w, b = self.n_nodes, self.label_words, int(lib.ksh_context_num_bound(self._h))
        ac, am = np.empty(n, np.int64), np.empty(n, np.int64)
        lab = np.zeros((n, w), np.uint64)
        bn, bc, bm = np.empty(b, np.int32), np.empty(b, np.int64), np.empty(b, np.int64)
        check(lib.ksh_context_export_packed(self._h, ac.ctypes.data, am.ctypes.data, lab.ctypes.data, bn.ctypes.data,
                                            bc.ctypes.data, bm.ctypes.data), "ksh_context_export_packed")
        return ac, am, lab, bn, bc, bm

    def check_node_validity(self, pods, i, node_idx):
        return check(lib.ksh_check_node_validity(self._h, _addr(pods, i), int(node_idx)), "ksh_check_node_validity")

    def place_replicas(self, pods, n, replicas, policy=capi.KS_SCORE_LEFTOVER, want_nodes=True, first=0):
        """Replica placement over objects (ksh_place_replicas): pod t asks for replicas[t] copies of itself.  Charges
        nothing.  Returns (rows, node, score, offset) as Snapshot.place_replicas; node indices name nodes through
        node_name()."""
        replicas = np.ascontiguousarray(replicas, np.uint32).reshape(-1)
        if replicas.shape[0] != n:
            raise ValueError(f"replicas has {replicas.shape[0]} entries, pods {n}")
        offset, rows, node, score = replica_outputs(replicas, capi.REPLICA_PLAN_DTYPE, want_nodes)
        check(lib.ksh_place_replicas(self._h, _addr(pods, first), n, replicas.ctypes.data, int(policy),
                                     rows.ctypes.data, None if node is None else node.ctypes.data,
                                     None if score is None else score.ctypes.data), "ksh_place_replicas")
        return rows, node, score, offset

    def topology_domains(self, key):
        """(node_domain int32 [N], values): dense domain ids of the topology key `key' over the node store, numbered by
        each value's first appearance in node order (-1 = the node lacks the key), and values[d] = domain d's value."""
        n = self.n_nodes
        dom = np.empty(n, np.int32)
        d = C.c_uint32()
        # every value is at most a label value's length; grow once if some did not fit
        cap = 64 * max(n, 1)
        while True:
            buf = C.create_string_buffer(cap)
            off = np.empty(max(n, 1), np.int64)
            check(lib.ksh_context_topology_domains(self._h, key.encode(), dom.ctypes.data, C.byref(d), buf, cap,
                                                   off.ctypes.data), "ksh_context_topology_domains")
            if (off[:d.value] >= 0).all():
                break
            cap *= 4
        return dom, _string_list(buf, off[:d.value])

    def place_replicas_spread(self, pods, n, replicas, topology_key, max_skew, min_domains=None, existing_nodes=None,
                              policy=capi.KS_SCORE_LEFTOVER, want_nodes=True, first=0):
        """Replica placement under one topology spread constraint over objects (ksh_place_replicas_spread): pod t asks
        for replicas[t] copies of itself, spread over the domains of topology_key with max_skew[t] (and min_domains[t]).
        existing_nodes[t] lists the node names of the bound pods that match spec t's constraint selector (None: none).
        Charges nothing.  Returns (rows, node, score, offset, counts) as Snapshot.place_replicas_spread, with the
        domains numbered as topology_domains(topology_key) numbers them (counts None when no node has the key)."""
        replicas = np.ascontiguousarray(replicas, np.uint32).reshape(-1)
        max_skew = np.ascontiguousarray(max_skew, np.uint32).reshape(-1)
        if replicas.shape[0] != n or max_skew.shape[0] != n:
            raise ValueError(f"replicas / max_skew have {replicas.shape[0]} / {max_skew.shape[0]} entries, pods {n}")
        mind = None if min_domains is None else np.ascontiguousarray(min_domains, np.uint32).reshape(-1)
        names, ex_off = None, None
        if existing_nodes is not None:
            flat = [s.encode() for lst in existing_nodes for s in lst]
            names = (C.c_char_p * max(len(flat), 1))(*flat)
            ex_off = np.zeros(n + 1, np.uint64)
            np.cumsum([len(lst) for lst in existing_nodes], out=ex_off[1:])
        D = len(self.topology_domains(topology_key)[1])
        offset, rows, node, score = replica_outputs(replicas, capi.SPREAD_PLAN_DTYPE, want_nodes)
        counts = np.empty((n, D), np.uint32) if D and n * D <= capi.KS_SPREAD_MAX_COUNTS else None
        check(lib.ksh_place_replicas_spread(self._h, _addr(pods, first), n, replicas.ctypes.data, topology_key.encode(),
                                            max_skew.ctypes.data, None if mind is None else mind.ctypes.data,
                                            None if names is None else C.cast(names, _vp),
                                            None if ex_off is None else ex_off.ctypes.data, int(policy),
                                            rows.ctypes.data,
                                            None if node is None else node.ctypes.data,
                                            None if score is None else score.ctypes.data,
                                            None if counts is None else counts.ctypes.data),
              "ksh_place_replicas_spread")
        return rows, node, score, offset, counts

    def place_replicas_spread_multi(self, pods, n, replicas, topology_keys, max_skew, min_domains=None,
                                    existing_nodes=None, policy=capi.KS_SCORE_LEFTOVER, want_nodes=True, first=0):
        """Replica placement under one topology spread constraint per key over objects (ksh_place_replicas_spread_multi):
        as place_replicas_spread, with topology_keys a list of K keys, max_skew and min_domains [n, K], and
        existing_nodes[t][k] the node names of the bound pods that match spec t's constraint for key k (None: none).
        Returns (rows [n, K], node, score, offset, counts) as Snapshot.place_replicas_spread_multi, with each key's
        domains numbered as topology_domains(key) numbers them (counts None when some key is on no node)."""
        k = len(topology_keys)
        replicas = np.ascontiguousarray(replicas, np.uint32).reshape(-1)
        max_skew = np.ascontiguousarray(max_skew, np.uint32).reshape(-1)
        if replicas.shape[0] != n or max_skew.shape[0] != n * k:
            raise ValueError(f"replicas / max_skew have {replicas.shape[0]} / {max_skew.shape[0]} entries, pods {n}, "
                             f"keys {k}")
        mind = None if min_domains is None else np.ascontiguousarray(min_domains, np.uint32).reshape(-1)
        names, ex_off = None, None
        if existing_nodes is not None:
            lists = [lst for per_spec in existing_nodes for lst in per_spec]
            flat = [s.encode() for lst in lists for s in lst]
            names = (C.c_char_p * max(len(flat), 1))(*flat)
            ex_off = np.zeros(n * k + 1, np.uint64)
            np.cumsum([len(lst) for lst in lists], out=ex_off[1:])
        keys = (C.c_char_p * max(k, 1))(*[key.encode() for key in topology_keys])
        nd = [len(self.topology_domains(key)[1]) for key in topology_keys]
        offset, _, node, score = replica_outputs(replicas, capi.SPREAD_PLAN_DTYPE, want_nodes)
        rows = np.zeros((n, k), capi.SPREAD_PLAN_DTYPE)
        s = sum(nd)
        counts = np.empty((n, s), np.uint32) if min(nd, default=0) and n * s <= capi.KS_SPREAD_MAX_COUNTS else None
        check(lib.ksh_place_replicas_spread_multi(self._h, _addr(pods, first), n, replicas.ctypes.data,
                                                  C.cast(keys, _vp), k, max_skew.ctypes.data,
                                                  None if mind is None else mind.ctypes.data,
                                                  None if names is None else C.cast(names, _vp),
                                                  None if ex_off is None else ex_off.ctypes.data, int(policy),
                                                  rows.ctypes.data,
                                                  None if node is None else node.ctypes.data,
                                                  None if score is None else score.ctypes.data,
                                                  None if counts is None else counts.ctypes.data),
              "ksh_place_replicas_spread_multi")
        if counts is not None:
            counts = np.split(counts, np.cumsum(nd)[:-1], axis=1)
        return rows, node, score, offset, counts

    def select_nodes(self, pods, n, policy=capi.KS_SCORE_LEFTOVER, first=0):
        idx = np.empty(n, np.int32)
        score = np.empty(n, np.int64)
        cnt = np.empty(n, np.uint32)
        check(lib.ksh_select_nodes(self._h, _addr(pods, first), n, int(policy), idx.ctypes.data, score.ctypes.data,
                                   cnt.ctypes.data), "ksh_select_nodes")
        return idx, score, cnt

    def rank_nodes(self, pods, n, k, policy=capi.KS_SCORE_LEFTOVER, first=0):
        """Ranked alternatives (ksh_rank_nodes): (node_idx int32 [n, k], score int64 [n, k], feasible_cnt uint32 [n]);
        entry 0 of a row is select_nodes()'s pick, -1 fills the slots past the feasible count.  Charges nothing."""
        idx = np.empty((n, int(k)), np.int32)
        score = np.empty((n, int(k)), np.int64)
        cnt = np.empty(n, np.uint32)
        check(lib.ksh_rank_nodes(self._h, _addr(pods, first), n, int(policy), int(k), idx.ctypes.data,
                                 score.ctypes.data, cnt.ctypes.data), "ksh_rank_nodes")
        return idx, score, cnt

    def select_node_for_pod(self, pods, n, attempts=capi.KS_REFERENCE_ATTEMPTS, seed=0, first=0):
        """select_node_for_pod with the reference's own seeded <=attempts-draw policy (src/main.rs:49-71)."""
        idx = np.empty(n, np.int32)
        used = np.empty(n, np.uint32)
        dn = np.empty((n, attempts), np.int32)
        dc = np.empty((n, attempts), np.uint8)
        check(lib.ksh_select_node_for_pod(self._h, _addr(pods, first), n, int(attempts), int(seed), int(first),
                                          idx.ctypes.data, used.ctypes.data, dn.ctypes.data, dc.ctypes.data),
              "ksh_select_node_for_pod")
        return idx, used, dn, dc

    def explain_pods(self, pods, n, first=0, msg_cap=None):
        """Why pods do not schedule: (reasons uint32 [n, 4], messages[n]) where messages[i] is the FailedScheduling
        message of a pod with no feasible node (str) or None."""
        out = np.empty((n, 4), np.uint32)
        off = np.empty(n, np.int64)
        cap = int(msg_cap if msg_cap is not None else 256 * max(n, 1))
        buf = C.create_string_buffer(max(cap, 1))
        check(lib.ksh_explain_pods(self._h, _addr(pods, first), n, out.ctypes.data, C.addressof(buf), cap,
                                   off.ctypes.data), "ksh_explain_pods")
        return out, _string_list(buf, off)

    def set_pod_priorities(self, pods, priority, n, first=0):
        """spec.priority of bound pods known by namespace/name (others are ignored)."""
        priority = np.ascontiguousarray(priority, np.int32)
        check(lib.ksh_context_set_pod_priorities(self._h, _addr(pods, first), priority.ctypes.data, n),
              "ksh_context_set_pod_priorities")

    def preempt_pods(self, pods, n, priority, max_victims, first=0, victims_cap=None):
        """Priority preemption (ksh_preempt_pods): (rows PREEMPTION_DTYPE [n], victims[n]) where victims[i] is the list
        of "namespace/name" keys to evict for pod i, in visit order, or None (no plan, or the buffer was full)."""
        priority = np.ascontiguousarray(priority, np.int32)
        rows = np.empty(n, capi.PREEMPTION_DTYPE)
        off = np.empty(n, np.int64)
        cap = int(victims_cap if victims_cap is not None else 64 * int(max_victims) * max(n, 1))
        buf = C.create_string_buffer(max(cap, 1))
        check(lib.ksh_preempt_pods(self._h, _addr(pods, first), n, priority.ctypes.data, int(max_victims),
                                   rows.ctypes.data, C.addressof(buf), cap, off.ctypes.data), "ksh_preempt_pods")
        return rows, _string_list(buf, off, rows["n_victims"])

    def preempt_fit_pods(self, pods, n, group, n_groups, priority, max_victims, group_rules=None, first=0,
                         victims_cap=None):
        """Priority preemption under the full filter (ksh_preempt_fit_pods): preempt_pods with group [n] and
        group_rules [n_groups] as reconcile_nodes takes them (None: no toleration and no term); the context's taints,
        the batch's extended resources and the pod limit apply.  Returns (rows, victims) as preempt_pods."""
        priority = np.ascontiguousarray(priority, np.int32).reshape(-1)
        group = np.ascontiguousarray(group, np.int32).reshape(-1)
        if priority.shape[0] != n or group.shape[0] != n:
            raise ValueError(f"priority has {priority.shape[0]} and group {group.shape[0]} entries, pods {n}")
        nr = None
        if group_rules is not None:
            if len(group_rules) != n_groups:
                raise ValueError(f"group_rules has {len(group_rules)} entries, groups {n_groups}")
            nr = node_rules(group_rules)
        rows = np.empty(n, capi.PREEMPTION_DTYPE)
        off = np.empty(n, np.int64)
        cap = int(victims_cap if victims_cap is not None else 64 * int(max_victims) * max(n, 1))
        buf = C.create_string_buffer(max(cap, 1))
        check(lib.ksh_preempt_fit_pods(self._h, _addr(pods, first), n, group.ctypes.data, int(n_groups),
                                       None if nr is None else C.addressof(nr[0]), priority.ctypes.data,
                                       int(max_victims), rows.ctypes.data, C.addressof(buf), cap, off.ctypes.data),
              "ksh_preempt_fit_pods")
        return rows, _string_list(buf, off, rows["n_victims"])

    def reconcile(self, pods, i, policy=capi.KS_SCORE_LEFTOVER):
        node = C.c_int32(-1)
        buf = C.create_string_buffer(1024)
        rc = check(lib.ksh_reconcile(self._h, _addr(pods, i), int(policy), C.byref(node), buf, len(buf)),
                   "ksh_reconcile")
        return rc, node.value, buf.value.decode()

    def reconcile_batch(self, pods, n, policy=capi.KS_SCORE_LEFTOVER, json_cap=None):
        """reconcile() over a drained queue: (status[n], node_idx[n], bodies[n] (str | None), rounds)."""
        status = np.empty(n, np.int32)
        node = np.empty(n, np.int32)
        off = np.empty(n, np.int64)
        cap = int(json_cap if json_cap is not None else 512 * max(n, 1))
        buf = C.create_string_buffer(cap)
        rounds = C.c_uint32()
        check(lib.ksh_reconcile_batch(self._h, C.addressof(pods), n, int(policy), status.ctypes.data, node.ctypes.data,
                                      C.addressof(buf), cap, off.ctypes.data, C.byref(rounds)), "ksh_reconcile_batch")
        bodies = _string_list(buf, off)
        return status, node, bodies, rounds.value

    def reconcile_gangs(self, pods, n, offset, min_member, policy=capi.KS_SCORE_LEFTOVER, json_cap=None):
        """reconcile() over pod groups, all or nothing (ksh_reconcile_gangs): group g is pods [offset[g], offset[g+1]).
        Returns (status[n], node_idx[n], bodies[n] (str | None), placed[G])."""
        offset = np.ascontiguousarray(offset, np.uint64).reshape(-1)
        min_member = np.ascontiguousarray(min_member, np.uint32).reshape(-1)
        g = offset.shape[0] - 1
        if g < 0 or min_member.shape[0] != g:
            raise ValueError(f"need len(offset) >= 1 and len(min_member) == len(offset) - 1 "
                             f"(got {offset.shape[0]} and {min_member.shape[0]})")
        status = np.empty(n, np.int32)
        node = np.empty(n, np.int32)
        off = np.empty(n, np.int64)
        placed = np.empty(g, np.uint32)
        cap = int(json_cap if json_cap is not None else 512 * max(n, 1))
        buf = C.create_string_buffer(max(cap, 1))
        check(lib.ksh_reconcile_gangs(self._h, C.addressof(pods), n, offset.ctypes.data, g, min_member.ctypes.data,
                                      int(policy), status.ctypes.data, node.ctypes.data, placed.ctypes.data,
                                      C.addressof(buf), cap, off.ctypes.data), "ksh_reconcile_gangs")
        bodies = _string_list(buf, off)
        return status, node, bodies, placed

    def reconcile_spread(self, pods, n, group, n_groups, topology_keys, max_skew, min_domains=None, existing_nodes=None,
                         policy=capi.KS_SCORE_LEFTOVER, json_cap=None):
        """reconcile() under topology spread (ksh_reconcile_spread): pod i belongs to group group[i] (-1 = none), each
        group with max_skew and min_domains [n_groups, K] over topology_keys (max_skew 0 = the key is not constrained);
        existing_nodes[g][k] lists the node names of group g's bound pods for key k (None: none).  Pods are bound one at
        a time in arrival order.  Returns (status[n], node_idx[n], bodies[n] (str | None))."""
        return self._reconcile_terms("ksh_reconcile_spread", pods, n, group, n_groups, topology_keys, None, (),
                                     max_skew, min_domains, existing_nodes, policy, json_cap)

    def reconcile_affinity(self, pods, n, group, n_groups, topology_keys, terms=(), existing_pods=(), max_skew=None,
                           min_domains=None, existing_nodes=None, policy=capi.KS_SCORE_LEFTOVER, json_cap=None):
        """reconcile() under spread and required inter-pod affinity (ksh_reconcile_affinity): reconcile_spread with
        max_skew optional (None: no spread constraint), terms a list of (owner group, kind KS_POD_AFFINITY /
        KS_POD_ANTI_AFFINITY, index into topology_keys, target groups) and existing_pods a list of (group, node name) of
        bound pods the terms see.  Returns (status[n], node_idx[n], bodies[n] (str | None))."""
        return self._reconcile_terms("ksh_reconcile_affinity", pods, n, group, n_groups, topology_keys, terms,
                                     existing_pods, max_skew, min_domains, existing_nodes, policy, json_cap)

    def reconcile_profile(self, pods, n, group, n_groups, topology_keys, terms=(), existing_pods=(), max_skew=None,
                          min_domains=None, existing_nodes=None, policy=capi.KS_SCORE_LEAST_BALANCED, json_cap=None,
                          soft_skew=None, soft_all_keys=None, term_weight=None, hard_affinity_weight=1, weight_spread=2,
                          weight_affinity=2):
        """reconcile_affinity scored as the default profile (ksh_reconcile_profile): terms may also be
        KS_POD_AFFINITY_PREFERRED / KS_POD_ANTI_AFFINITY_PREFERRED with term_weight [T]; soft_skew [n_groups, K] or
        None, soft_all_keys [n_groups] or None (all 1), and the three weights as Snapshot.profile_bind takes them.
        Returns (status[n], node_idx[n], bodies[n] (str | None))."""
        scoring, hold = _scoring(n_groups, len(topology_keys), len(terms), soft_skew, soft_all_keys, term_weight,
                                 hard_affinity_weight, weight_spread, weight_affinity)
        return self._reconcile_terms("ksh_reconcile_profile", pods, n, group, n_groups, topology_keys, terms,
                                     existing_pods, max_skew, min_domains, existing_nodes, policy, json_cap,
                                     (C.byref(scoring),))

    def set_node_taints(self, taints):
        """spec.taints of nodes by name (ksh_context_set_node_taints): taints maps a node name to a list of
        {"key", "value", "effect"}; it replaces what that node carried.  Unknown names are ignored."""
        names = list(taints)
        flat = [t for nm in names for t in taints[nm]]
        off = np.zeros(len(names) + 1, np.uint64)
        np.cumsum([len(taints[nm]) for nm in names], out=off[1:])
        arr = (ksh_taint * max(len(flat), 1))(*[ksh_taint(_b(t["key"]), _b(t.get("value", "")), _b(t["effect"]))
                                                 for t in flat])
        cn = (C.c_char_p * max(len(names), 1))(*[nm.encode() for nm in names])
        check(lib.ksh_context_set_node_taints(self._h, C.cast(cn, _vp), off.ctypes.data, C.addressof(arr), len(names)),
              "ksh_context_set_node_taints")

    def compile_node_rules(self, group_rules):
        """The compiled rules evaluated per (group, node) (ksh_compile_node_rules): (hard uint8 [G, N], affinity uint8
        [G, N], soft uint32 [G, N], preferred uint32 [G, N]); group_rules as node_rules takes them."""
        G, N = len(group_rules), self.n_nodes
        nr, hold = node_rules(group_rules)
        out = (np.zeros((G, N), np.uint8), np.zeros((G, N), np.uint8), np.zeros((G, N), np.uint32),
               np.zeros((G, N), np.uint32))
        check(lib.ksh_compile_node_rules(self._h, G, C.byref(nr), *[o.ctypes.data for o in out]),
              "ksh_compile_node_rules")
        return out

    def reconcile_nodes(self, pods, n, group, n_groups, topology_keys, terms=(), existing_pods=(), max_skew=None,
                        min_domains=None, existing_nodes=None, policy=capi.KS_SCORE_LEAST_BALANCED, json_cap=None,
                        soft_skew=None, soft_all_keys=None, term_weight=None, hard_affinity_weight=1, weight_spread=2,
                        weight_affinity=2, group_rules=None, weight_taint=3, weight_node_affinity=2):
        """reconcile_profile with the context's node taints and per-group rules (ksh_reconcile_nodes): group_rules
        [n_groups] as node_rules takes them, or None (no toleration and no term).  Status 7
        (KSH_RECONCILE_NODE_RULES_UNSATISFIED) for a pod that fit some node but taints or node affinity refused every
        such node.  Returns (status[n], node_idx[n], bodies[n])."""
        return self._reconcile_rules(pods, n, group, n_groups, topology_keys, terms, existing_pods, max_skew,
                                     min_domains, existing_nodes, policy, json_cap, soft_skew, soft_all_keys,
                                     term_weight, hard_affinity_weight, weight_spread, weight_affinity, group_rules,
                                     weight_taint, weight_node_affinity, "ksh_reconcile_nodes")

    def compile_resources(self, pods, n):
        """The scalar resources of the pending batch pods[0:n] (ksh_compile_resources): (names, node_free int64 [R, N],
        pod_req int64 [n, R]); names[0] == "pods"."""
        N, M = self.n_nodes, capi.KS_BIND_MAX_RESOURCES
        free = np.zeros(M * N, np.int64)
        req = np.zeros(M * n, np.int64)
        cap = 64 * 1024
        buf = C.create_string_buffer(cap)
        r = lib.ksh_compile_resources(self._h, C.addressof(pods) if n else None, n, C.addressof(buf), cap,
                                      free.ctypes.data, req.ctypes.data)
        check(min(r, 0), "ksh_compile_resources")
        names = [x.decode() for x in buf.raw.split(b"\0")[:r]]
        return names, free[:r * N].reshape(r, N), req[:n * r].reshape(n, r)

    def reconcile_fit(self, pods, n, group, n_groups, topology_keys, terms=(), existing_pods=(), max_skew=None,
                      min_domains=None, existing_nodes=None, policy=capi.KS_SCORE_LEAST_BALANCED, json_cap=None,
                      soft_skew=None, soft_all_keys=None, term_weight=None, hard_affinity_weight=1, weight_spread=2,
                      weight_affinity=2, group_rules=None, weight_taint=3, weight_node_affinity=2):
        """reconcile_nodes with the pod count and the scalar resources of NodeResourcesFit (ksh_reconcile_fit): the
        batch's resources are compile_resources'.  Status 8 (KSH_RECONCILE_INSUFFICIENT_RESOURCES) for a pod that fit
        some node by cpu, memory and selector but every such node lacked a resource or was at its pod limit.  Returns
        (status[n], node_idx[n], bodies[n])."""
        return self._reconcile_rules(pods, n, group, n_groups, topology_keys, terms, existing_pods, max_skew,
                                     min_domains, existing_nodes, policy, json_cap, soft_skew, soft_all_keys,
                                     term_weight, hard_affinity_weight, weight_spread, weight_affinity, group_rules,
                                     weight_taint, weight_node_affinity, "ksh_reconcile_fit")

    def reconcile_fit_gangs(self, pods, n, group, n_groups, topology_keys, offset, min_member, terms=(),
                            existing_pods=(), max_skew=None, min_domains=None, existing_nodes=None,
                            policy=capi.KS_SCORE_LEAST_BALANCED, json_cap=None, soft_skew=None, soft_all_keys=None,
                            term_weight=None, hard_affinity_weight=1, weight_spread=2, weight_affinity=2,
                            group_rules=None, weight_taint=3, weight_node_affinity=2):
        """reconcile_fit over gangs placed all or nothing (ksh_reconcile_fit_gangs): gang j is pods
        [offset[j], offset[j+1]), its running members count toward min_member[j], and the pods of a gang that cannot
        commit get KSH_RECONCILE_GANG_UNSATISFIED.  Returns (status[n], node_idx[n], bodies[n], placed[n_gangs])."""
        offset = np.ascontiguousarray(offset, np.uint64).reshape(-1)
        min_member = np.ascontiguousarray(min_member, np.uint32).reshape(-1)
        g = offset.shape[0] - 1
        if g < 0 or min_member.shape[0] != g:
            raise ValueError(f"need len(offset) >= 1 and len(min_member) == len(offset) - 1 "
                             f"(got {offset.shape[0]} and {min_member.shape[0]})")
        placed = np.empty(g, np.uint32)
        return self._reconcile_rules(pods, n, group, n_groups, topology_keys, terms, existing_pods, max_skew,
                                     min_domains, existing_nodes, policy, json_cap, soft_skew, soft_all_keys,
                                     term_weight, hard_affinity_weight, weight_spread, weight_affinity, group_rules,
                                     weight_taint, weight_node_affinity, "ksh_reconcile_fit_gangs",
                                     (offset.ctypes.data, g, min_member.ctypes.data), placed) + (placed,)

    def _reconcile_rules(self, pods, n, group, n_groups, topology_keys, terms, existing_pods, max_skew, min_domains,
                         existing_nodes, policy, json_cap, soft_skew, soft_all_keys, term_weight, hard_affinity_weight,
                         weight_spread, weight_affinity, group_rules, weight_taint, weight_node_affinity, entry,
                         gangs=(), placed=None):
        # ksh_reconcile_nodes, ksh_reconcile_fit, or ksh_reconcile_fit_gangs with gangs (offset, n_gangs, min_member)
        nr = None
        if group_rules is not None:
            if len(group_rules) != n_groups:
                raise ValueError(f"group_rules has {len(group_rules)} entries, groups {n_groups}")
            nr = node_rules(group_rules, weight_taint, weight_node_affinity)
        scoring, hold = _scoring(n_groups, len(topology_keys), len(terms), soft_skew, soft_all_keys, term_weight,
                                 hard_affinity_weight, weight_spread, weight_affinity)
        return self._reconcile_terms(entry, pods, n, group, n_groups, topology_keys, terms, existing_pods, max_skew,
                                     min_domains, existing_nodes, policy, json_cap,
                                     (C.byref(scoring), None if nr is None else C.byref(nr[0]), *gangs), placed)

    def _reconcile_terms(self, entry, pods, n, group, n_groups, topology_keys, terms, existing_pods, max_skew,
                         min_domains, existing_nodes, policy, json_cap, mid=(), placed=None):
        # the host-layer call `entry`: its queue and topology, then (terms not None) the terms and existing pods, then
        # mid (scoring, rules, gangs), the policy and the outputs, with placed before the bodies when given
        k = len(topology_keys)
        group = np.ascontiguousarray(group, np.int32).reshape(-1)
        if group.shape[0] != n:
            raise ValueError(f"group has {group.shape[0]} entries, pods {n}")
        if max_skew is not None:
            max_skew = np.ascontiguousarray(max_skew, np.uint32).reshape(-1)
            if max_skew.shape[0] != n_groups * k:
                raise ValueError(f"max_skew has {max_skew.shape[0]} entries, groups {n_groups}, keys {k}")
        mind = None if min_domains is None else np.ascontiguousarray(min_domains, np.uint32).reshape(-1)
        names, ex_off = None, None
        if existing_nodes is not None:
            lists = [lst for per_group in existing_nodes for lst in per_group]
            flat = [s.encode() for lst in lists for s in lst]
            names = (C.c_char_p * max(len(flat), 1))(*flat)
            ex_off = np.zeros(n_groups * k + 1, np.uint64)
            np.cumsum([len(lst) for lst in lists], out=ex_off[1:])
        keys = (C.c_char_p * max(k, 1))(*[key.encode() for key in topology_keys])
        args = [self._h, C.addressof(pods) if n else None, n, group.ctypes.data, int(n_groups), C.cast(keys, _vp), k,
                None if max_skew is None else max_skew.ctypes.data, None if mind is None else mind.ctypes.data,
                None if names is None else C.cast(names, _vp), None if ex_off is None else ex_off.ctypes.data]
        if terms is not None:
            owner = np.ascontiguousarray([t[0] for t in terms], np.int32)
            kind = np.ascontiguousarray([t[1] for t in terms], np.uint8)
            tkey = np.ascontiguousarray([t[2] for t in terms], np.uint32)
            toff = np.zeros(len(terms) + 1, np.uint64)
            np.cumsum([len(t[3]) for t in terms], out=toff[1:])
            target = np.ascontiguousarray([g for t in terms for g in t[3]], np.int32)
            egroup = np.ascontiguousarray([e[0] for e in existing_pods], np.int32)
            enames = (C.c_char_p * max(len(existing_pods), 1))(*[e[1].encode() for e in existing_pods])
            aff = ksh_pod_affinity(len(terms), owner.ctypes.data, kind.ctypes.data, tkey.ctypes.data,
                                   toff.ctypes.data, target.ctypes.data, len(existing_pods), egroup.ctypes.data,
                                   C.cast(enames, _vp))
            args.append(C.byref(aff))
        status = np.empty(n, np.int32)
        node = np.empty(n, np.int32)
        off = np.empty(n, np.int64)
        cap = int(json_cap if json_cap is not None else 512 * max(n, 1))
        buf = C.create_string_buffer(max(cap, 1))
        args += [*mid, int(policy), status.ctypes.data, node.ctypes.data]
        args += ([] if placed is None else [placed.ctypes.data]) + [C.addressof(buf), cap, off.ctypes.data]
        check(getattr(lib, entry)(*args), entry)
        return status, node, _string_list(buf, off)

    def drain_nodes(self, node_names, pods, pod_offset, policy=capi.KS_SCORE_LEFTOVER, flags=0):
        """Drain simulation over objects (ksh_drain_nodes): candidate d is the node named node_names[d] with pods
        [pod_offset[d], pod_offset[d+1]), each bound to that node.  Returns (placed[D], node_idx[P])."""
        pod_offset = np.ascontiguousarray(pod_offset, np.uint64).reshape(-1)
        d = len(node_names)
        if pod_offset.shape[0] != d + 1:
            raise ValueError(f"need len(pod_offset) == len(node_names) + 1 (got {pod_offset.shape[0]} and {d})")
        names = (C.c_char_p * max(d, 1))(*[n.encode() if isinstance(n, str) else n for n in node_names])
        p = int(pod_offset[-1])
        placed = np.empty(d, np.uint32)
        node = np.empty(p, np.int32)
        check(lib.ksh_drain_nodes(self._h, C.addressof(names), d, C.addressof(pods) if pods is not None else None,
                                  pod_offset.ctypes.data, int(policy), int(flags), placed.ctypes.data,
                                  node.ctypes.data), "ksh_drain_nodes")
        return placed, node

    def drain_fit_nodes(self, node_names, pods, pod_offset, group, n_groups, group_rules=None,
                        policy=capi.KS_SCORE_LEFTOVER, flags=0, want_refused=True):
        """Drain simulation under the full filter (ksh_drain_fit_nodes): drain_nodes with group [P] and group_rules
        [n_groups] as preempt_fit_pods takes them (None: no toleration and no term); the context's taints, the drained
        pods' extended resources and the pod limit apply.  Returns (placed[D], node_idx[P], refused[D, 4] or None)."""
        pod_offset = np.ascontiguousarray(pod_offset, np.uint64).reshape(-1)
        d = len(node_names)
        if pod_offset.shape[0] != d + 1:
            raise ValueError(f"need len(pod_offset) == len(node_names) + 1 (got {pod_offset.shape[0]} and {d})")
        p = int(pod_offset[-1])
        group = np.ascontiguousarray(group, np.int32).reshape(-1)
        if group.shape[0] != p:
            raise ValueError(f"group has {group.shape[0]} entries, pods {p}")
        nr = None
        if group_rules is not None:
            if len(group_rules) != n_groups:
                raise ValueError(f"group_rules has {len(group_rules)} entries, groups {n_groups}")
            nr = node_rules(group_rules)
        names = (C.c_char_p * max(d, 1))(*[n.encode() if isinstance(n, str) else n for n in node_names])
        placed = np.empty(d, np.uint32)
        node = np.empty(p, np.int32)
        refused = np.empty((d, 4), np.uint32) if want_refused else None
        check(lib.ksh_drain_fit_nodes(self._h, C.addressof(names), d, C.addressof(pods) if pods is not None else None,
                                      pod_offset.ctypes.data, group.ctypes.data, int(n_groups),
                                      None if nr is None else C.addressof(nr[0]), int(policy), int(flags),
                                      placed.ctypes.data, node.ctypes.data,
                                      None if refused is None else refused.ctypes.data), "ksh_drain_fit_nodes")
        return placed, node, refused

    def scaleup_estimate(self, templates, n_templates, max_nodes, pods, n_pods, overhead_pods=None, n_overhead=0,
                         want_nodes=True, want_reasons=True):
        """Node-group scale-up estimate over objects (ksh_scaleup_estimate): templates are Node objects, overhead_pods
        the DaemonSet pods charged to the template their spec.nodeName names, pods the pending pods.  Nothing is
        charged and the context is not changed.  Returns (rows, best, node, reasons) as Snapshot.scaleup_estimate."""
        max_nodes = np.ascontiguousarray(max_nodes, np.uint32).reshape(-1)
        if max_nodes.shape[0] != n_templates:
            raise ValueError(f"need {n_templates} max_nodes entries (got {max_nodes.shape[0]})")
        rows = np.zeros(n_templates, capi.SCALEUP_OPTION_DTYPE)
        best = C.c_int32(-1)
        node = np.empty((n_templates, n_pods), np.int32) if want_nodes else None
        why = np.empty((n_pods, 4), np.uint32) if want_reasons else None

        def ptr(a):
            return None if a is None else a.ctypes.data

        def obj(a):
            return C.addressof(a) if a is not None else None
        check(lib.ksh_scaleup_estimate(self._h, obj(templates), n_templates, ptr(max_nodes), obj(overhead_pods),
                                       n_overhead, obj(pods), n_pods, ptr(rows), C.addressof(best), ptr(node),
                                       ptr(why)), "ksh_scaleup_estimate")
        return rows, best.value, node, why

    def scaleup_fit_estimate(self, templates, n_templates, max_nodes, pods, n_pods, group, n_groups, group_rules=None,
                             template_taints=None, overhead_pods=None, n_overhead=0, want_nodes=True,
                             want_refused=True):
        """Scale-up estimate under the full filter over objects (ksh_scaleup_fit_estimate): scaleup_estimate with group
        [n_pods] and group_rules [n_groups] as drain_fit_nodes takes them, and template_taints, a list of n_templates
        lists of {"key", "value", "effect"} (None: no taint).  The pending pods' extended resources, the templates' pod
        limit, taints and required node affinity apply.  Returns (rows, best, node [T, P] or None, refused [P, 4] or
        None)."""
        max_nodes = np.ascontiguousarray(max_nodes, np.uint32).reshape(-1)
        if max_nodes.shape[0] != n_templates:
            raise ValueError(f"need {n_templates} max_nodes entries (got {max_nodes.shape[0]})")
        group = np.ascontiguousarray(group, np.int32).reshape(-1)
        if group.shape[0] != n_pods:
            raise ValueError(f"group has {group.shape[0]} entries, pods {n_pods}")
        nr = None
        if group_rules is not None:
            if len(group_rules) != n_groups:
                raise ValueError(f"group_rules has {len(group_rules)} entries, groups {n_groups}")
            nr = node_rules(group_rules)
        toff, taints = None, None
        if template_taints is not None:
            if len(template_taints) != n_templates:
                raise ValueError(f"template_taints has {len(template_taints)} entries, templates {n_templates}")
            flat = [t for ts in template_taints for t in ts]
            toff = np.zeros(n_templates + 1, np.uint64)
            np.cumsum([len(ts) for ts in template_taints], out=toff[1:])
            taints = (ksh_taint * max(len(flat), 1))(*[ksh_taint(_b(t["key"]), _b(t.get("value", "")),
                                                                 _b(t["effect"])) for t in flat])
        rows = np.zeros(n_templates, capi.SCALEUP_OPTION_DTYPE)
        best = C.c_int32(-1)
        node = np.empty((n_templates, n_pods), np.int32) if want_nodes else None
        refused = np.empty((n_pods, 4), np.uint32) if want_refused else None

        def ptr(a):
            return None if a is None else a.ctypes.data

        def obj(a):
            return C.addressof(a) if a is not None else None
        check(lib.ksh_scaleup_fit_estimate(self._h, obj(templates), n_templates, ptr(max_nodes), ptr(toff), obj(taints),
                                           obj(overhead_pods), n_overhead, obj(pods), n_pods, ptr(group), int(n_groups),
                                           None if nr is None else C.addressof(nr[0]), ptr(rows), C.addressof(best),
                                           ptr(node), ptr(refused)), "ksh_scaleup_fit_estimate")
        return rows, best.value, node, refused
