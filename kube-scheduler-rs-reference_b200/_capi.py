"""ctypes binding of include/ksched.h (+ ksched_host.h once built).  Fails loudly if the library is missing."""
import ctypes as C
import os
import re

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libksched.so")
INCLUDE_DIR = os.path.join(os.path.dirname(_HERE), "include")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(nvcc, sm_90a).  There is no Python/CPU fallback for the scheduling kernels."
    )
lib = C.CDLL(LIB_PATH)

KS_OK = 0
KS_MEM_HOST, KS_MEM_DEVICE = 0, 1
KS_SCORE_LEFTOVER, KS_SCORE_LEAST_ALLOCATED = 0, 1
KS_SCORE_MOST_ALLOCATED = 3  # bin-packing; 2 is reserved and rejected
KS_SCORE_LEAST_BALANCED = 4  # upstream's default profile: LeastAllocated + BalancedAllocation
KS_SELECT_AUTO, KS_SELECT_FORCE_DIRECT, KS_SELECT_FORCE_BITPAR, KS_SELECT_TIMING, KS_SELECT_NO_GRAPH = 0, 1, 2, 4, 8
KS_CELL_OK, KS_CELL_NOT_ENOUGH_RESOURCES, KS_CELL_NODE_SELECTOR_MISMATCH = 0, 1, 2
KS_ERR_NO_DEVICE = -8


class KsError(RuntimeError):
    def __init__(self, code, where):
        self.code = code
        msg = lib.ks_last_error().decode("utf-8", "replace")
        super().__init__(f"{where} failed with {code}: {msg}")


def check(rc, where):
    """Raise KsError for a negative return code of `where`; otherwise return the code (a count or a cell code for the
    calls that return one)."""
    if rc < 0:
        raise KsError(rc, where)
    return rc


class ks_pods(C.Structure):
    _fields_ = [("n", C.c_uint64), ("req_cpu", C.c_void_p), ("req_mem", C.c_void_p), ("sel", C.c_void_p),
                ("mem_space", C.c_int32)]


KS_MAX_PEERS = 15


class ks_exchange(C.Structure):
    _fields_ = [("world", C.c_uint32), ("rank", C.c_uint32), ("n_peers", C.c_uint32),
                ("peer_node_idx", C.c_void_p * KS_MAX_PEERS), ("peer_score", C.c_void_p * KS_MAX_PEERS),
                ("peer_flag", C.c_void_p * KS_MAX_PEERS), ("local_flags", C.c_void_p), ("local_state", C.c_void_p)]


class ks_bindings(C.Structure):
    _fields_ = [("node_idx", C.c_void_p), ("score", C.c_void_p), ("feasible_cnt", C.c_void_p),
                ("mem_space", C.c_int32), ("mask", C.c_void_p), ("mask_row_bytes", C.c_uint64),
                ("mask_space", C.c_int32), ("bindings_ready_event", C.c_void_p), ("exchange", C.POINTER(ks_exchange))]


class ks_pod_reasons(C.Structure):
    _fields_ = [("insufficient_cpu", C.c_uint32), ("insufficient_memory", C.c_uint32),
                ("not_enough_resources", C.c_uint32), ("node_selector_mismatch", C.c_uint32)]


def _proto(name, restype, *argtypes, optional=False):
    """Declare lib.name.  optional: a library built from the host layer and a device stand-in (tests/native) may lack
    the entry, which is then left undeclared."""
    if optional and not hasattr(lib, name):
        return None
    fn = getattr(lib, name)
    fn.restype = restype
    fn.argtypes = list(argtypes)
    return fn


_proto("ks_last_error", C.c_char_p)
_proto("ks_version", C.c_int)
_proto("ks_device_count", C.c_int)
_proto("ks_launch_count", C.c_uint64)
_proto("ks_mask_row_bytes", C.c_uint64, C.c_uint32)
_proto("ks_mask_row_bytes_aligned", C.c_uint64, C.c_uint32)
_proto("ks_snapshot_create", C.c_int, C.c_int, C.POINTER(C.c_void_p))
_proto("ks_snapshot_destroy", None, C.c_void_p)
_proto("ks_snapshot_set_nodes", C.c_int, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p)
_proto("ks_snapshot_set_bound", C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p)
_proto("ks_snapshot_apply_bind", C.c_int, C.c_void_p, C.c_int32, C.c_int64, C.c_int64)
_proto("ks_snapshot_get_free", C.c_int, C.c_void_p, C.c_void_p, C.c_void_p)
_proto("ks_snapshot_num_nodes", C.c_uint32, C.c_void_p)
_proto("ks_snapshot_label_words", C.c_uint32, C.c_void_p)
_proto("ks_check_cell", C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_uint32)
_proto("ks_check_cells", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p)
_proto("ks_select", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_int, C.c_uint32, C.POINTER(ks_bindings), C.c_void_p)
_proto("ks_last_timings", C.c_int, C.c_void_p, C.POINTER(C.c_float))
_proto("ks_last_path", C.c_char_p, C.c_void_p)
_proto("ks_last_trace", C.c_int, C.c_void_p, C.POINTER(C.c_uint64))
_proto("ks_snapshot_commit_claims", C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p)
_proto("ks_stream_bind", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_int, C.c_void_p, C.c_void_p,
       C.POINTER(C.c_uint32))

_proto("ks_stream_open", C.c_int, C.c_void_p, C.c_int, C.c_uint32, C.POINTER(C.c_void_p))
_proto("ks_stream_submit", C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p)
_proto("ks_stream_poll", C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64))
_proto("ks_stream_flush", C.c_int, C.c_void_p)
_proto("ks_stream_stats", C.c_int, C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64))
_proto("ks_stream_close", None, C.c_void_p)
_proto("ks_exchange_check", C.c_int, C.c_void_p)
_proto("ks_ipc_alloc", C.c_int, C.c_int, C.c_uint64, C.POINTER(C.c_void_p), C.c_char_p)
_proto("ks_ipc_open", C.c_int, C.c_int, C.c_char_p, C.POINTER(C.c_void_p))
_proto("ks_ipc_close", C.c_int, C.c_int, C.c_void_p)
_proto("ks_ipc_free", C.c_int, C.c_int, C.c_void_p)
_proto("ks_measure_write_bandwidth", C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.c_int, C.POINTER(C.c_double))
_proto("ks_device_read", C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64)
_proto("ks_select_sampling", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_uint32, C.c_uint64, C.c_uint64, C.c_void_p,
       C.c_void_p, C.c_void_p, C.c_void_p)
_proto("ks_explain", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.c_int32, C.c_void_p, optional=True)
_proto("ks_select_topk", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_int, C.c_uint32, C.c_void_p, C.c_void_p,
       C.c_void_p, C.c_int32, C.c_void_p, optional=True)
KS_TOPK_MAX = 32


class ks_bound_pods(C.Structure):
    _fields_ = [("n", C.c_uint64), ("node_idx", C.c_void_p), ("req_cpu", C.c_void_p), ("req_mem", C.c_void_p),
                ("priority", C.c_void_p)]


class ks_preemption(C.Structure):
    _fields_ = [("node_idx", C.c_int32), ("n_victims", C.c_uint32), ("candidates", C.c_uint32),
                ("feasible_cnt", C.c_uint32), ("max_victim_priority", C.c_int32), ("reserved", C.c_uint32),
                ("victim_priority_sum", C.c_int64)]


PREEMPTION_DTYPE = np.dtype(ks_preemption)  # the same row as a numpy record, for whole batches of rows
_proto("ks_preempt", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.POINTER(ks_bound_pods), C.c_uint32,
       C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, optional=True)
KS_PREEMPT_MAX_VICTIMS = 128


class ks_gangs(C.Structure):
    _fields_ = [("n", C.c_uint64), ("offset", C.c_void_p), ("min_member", C.c_void_p)]


_proto("ks_gang_bind", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.POINTER(ks_gangs), C.c_int, C.c_void_p, C.c_void_p,
       C.c_void_p, C.c_void_p, optional=True)
KS_GANG_MAX_SIZE = 1024


class ks_drain_candidates(C.Structure):
    _fields_ = [("n", C.c_uint64), ("node_idx", C.c_void_p), ("offset", C.c_void_p)]


_proto("ks_drain_check", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.POINTER(ks_drain_candidates), C.c_int, C.c_uint32,
       C.c_void_p, C.c_void_p, C.c_void_p, optional=True)
KS_DRAIN_MAX_PODS = 1024
KS_DRAIN_EXCLUDE_CANDIDATES = 1


class ks_node_templates(C.Structure):
    _fields_ = [("n", C.c_uint64), ("label_words", C.c_uint32), ("alloc_cpu", C.c_void_p), ("alloc_mem", C.c_void_p),
                ("free_cpu", C.c_void_p), ("free_mem", C.c_void_p), ("labels", C.c_void_p), ("max_nodes", C.c_void_p)]


class ks_scaleup_option(C.Structure):
    _fields_ = [("nodes", C.c_uint32), ("placed", C.c_uint32), ("eligible", C.c_uint32), ("utilization", C.c_int32),
                ("used_cpu", C.c_int64), ("used_mem", C.c_int64)]


SCALEUP_OPTION_DTYPE = np.dtype(ks_scaleup_option)  # the same row as a numpy record
_proto("ks_scaleup_estimate", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.POINTER(ks_node_templates), C.c_void_p,
       C.c_void_p, C.c_void_p, C.c_void_p, optional=True)
KS_SCALEUP_MAX_NODES = 1024
KS_SCALEUP_MAX_PODS = 65536
KS_SCALEUP_MAX_TEMPLATES = 4096


class ks_replica_plan(C.Structure):
    _fields_ = [("capacity", C.c_uint64), ("placed", C.c_uint32), ("nodes", C.c_uint32), ("feasible_cnt", C.c_uint32),
                ("max_per_node", C.c_uint32), ("last_score", C.c_int64)]


REPLICA_PLAN_DTYPE = np.dtype(ks_replica_plan)  # the same row as a numpy record
_proto("ks_place_replicas", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
       C.c_void_p, optional=True)
KS_REPLICAS_MAX_SPECS = 4096
KS_REPLICAS_MAX = 65536
KS_REPLICAS_MAX_TOTAL = 1 << 24


class ks_spread(C.Structure):
    _fields_ = [("n_domains", C.c_uint32), ("node_domain", C.c_void_p), ("max_skew", C.c_void_p),
                ("min_domains", C.c_void_p), ("existing", C.c_void_p)]


class ks_spread_plan(C.Structure):
    _fields_ = [("placed", C.c_uint32), ("nodes", C.c_uint32), ("max_per_node", C.c_uint32),
                ("eligible_domains", C.c_uint32), ("min_count", C.c_uint32), ("blocked_domain", C.c_int32),
                ("last_score", C.c_int64)]


SPREAD_PLAN_DTYPE = np.dtype(ks_spread_plan)  # the same row as a numpy record
_proto("ks_place_replicas_spread", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.POINTER(ks_spread), C.c_int,
       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, optional=True)
KS_SPREAD_MAX_DOMAINS = 1 << 20
KS_SPREAD_MAX_EXISTING = 1 << 24
KS_SPREAD_MAX_COUNTS = 1 << 26
KS_SPREAD_MAX_KEYS = 4


class ks_spread_multi(C.Structure):
    _fields_ = [("n_keys", C.c_uint32), ("n_domains", C.c_uint32 * KS_SPREAD_MAX_KEYS),
                ("node_domain", C.c_void_p * KS_SPREAD_MAX_KEYS), ("max_skew", C.c_void_p), ("min_domains", C.c_void_p),
                ("existing", C.c_void_p)]


_proto("ks_place_replicas_spread_multi", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p,
       C.POINTER(ks_spread_multi), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, optional=True)
_proto("ks_spread_bind", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.c_uint32, C.POINTER(ks_spread_multi),
       C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, optional=True)
KS_SPREAD_BIND_MAX_PODS = 65536
KS_SPREAD_BIND_MAX_GROUPS = 4096


class ks_pod_affinity(C.Structure):
    _fields_ = [("n_terms", C.c_uint32), ("owner", C.c_void_p), ("kind", C.c_void_p), ("key", C.c_void_p),
                ("target_offset", C.c_void_p), ("target", C.c_void_p), ("n_existing", C.c_uint64),
                ("existing_group", C.c_void_p), ("existing_node", C.c_void_p)]


_proto("ks_affinity_bind", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.c_uint32,
       C.POINTER(ks_spread_multi), C.POINTER(ks_pod_affinity), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
       C.c_void_p, optional=True)
KS_POD_AFFINITY, KS_POD_ANTI_AFFINITY = 0, 1
KS_POD_AFFINITY_PREFERRED, KS_POD_ANTI_AFFINITY_PREFERRED = 2, 3


class ks_bind_scoring(C.Structure):
    _fields_ = [("soft_skew", C.c_void_p), ("soft_all_keys", C.c_void_p), ("term_weight", C.c_void_p),
                ("hard_affinity_weight", C.c_uint32), ("weight_spread", C.c_uint32), ("weight_affinity", C.c_uint32)]


_proto("ks_profile_bind", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.c_uint32,
       C.POINTER(ks_spread_multi), C.POINTER(ks_pod_affinity), C.POINTER(ks_bind_scoring), C.c_int, C.c_void_p,
       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, optional=True)
KS_NODE_RULES_MAX_TAINTS = 64
KS_NODE_RULES_MAX_KEYS = 16
KS_NODE_RULES_MAX_PREFERRED = 4096
KS_NODE_RULES_MAX_WORDS = 1 << 26


class ks_node_rules(C.Structure):
    _fields_ = [("n_taints", C.c_uint32), ("node_taint_hard", C.c_void_p), ("node_taint_soft", C.c_void_p),
                ("tolerate_hard", C.c_void_p), ("tolerate_soft", C.c_void_p), ("n_keys", C.c_uint32),
                ("n_domains", C.c_uint32 * KS_NODE_RULES_MAX_KEYS), ("node_domain", C.c_void_p * KS_NODE_RULES_MAX_KEYS),
                ("n_exprs", C.c_uint32), ("expr_key", C.c_void_p), ("expr_set_offset", C.c_void_p),
                ("expr_set", C.c_void_p), ("n_terms", C.c_uint32), ("term_owner", C.c_void_p),
                ("term_weight", C.c_void_p), ("term_expr_offset", C.c_void_p), ("weight_taint", C.c_uint32),
                ("weight_node_affinity", C.c_uint32)]


_proto("ks_node_bind", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.c_uint32,
       C.POINTER(ks_spread_multi), C.POINTER(ks_pod_affinity), C.POINTER(ks_bind_scoring), C.POINTER(ks_node_rules),
       C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, optional=True)
KS_BIND_MAX_RESOURCES = 8


class ks_bind_resources(C.Structure):
    _fields_ = [("n_res", C.c_uint32), ("node_free", C.c_void_p), ("pod_req", C.c_void_p)]


_proto("ks_fit_bind", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.c_uint32,
       C.POINTER(ks_spread_multi), C.POINTER(ks_pod_affinity), C.POINTER(ks_bind_scoring), C.POINTER(ks_node_rules),
       C.POINTER(ks_bind_resources), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
       C.c_void_p, optional=True)
_proto("ks_gang_fit_bind", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.c_uint32,
       C.POINTER(ks_spread_multi), C.POINTER(ks_pod_affinity), C.POINTER(ks_bind_scoring), C.POINTER(ks_node_rules),
       C.POINTER(ks_bind_resources), C.POINTER(ks_gangs), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, optional=True)
_proto("ks_fit_preempt", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.c_uint32, C.POINTER(ks_node_rules),
       C.POINTER(ks_bind_resources), C.c_void_p, C.POINTER(ks_bound_pods), C.c_void_p, C.c_uint32, C.c_void_p,
       C.c_void_p, C.c_void_p, optional=True)
_proto("ks_fit_drain_check", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.c_uint32, C.POINTER(ks_node_rules),
       C.POINTER(ks_bind_resources), C.POINTER(ks_drain_candidates), C.c_int, C.c_uint32, C.c_void_p, C.c_void_p,
       C.c_void_p, C.c_void_p, optional=True)
_proto("ks_fit_scaleup_estimate", C.c_int, C.c_void_p, C.POINTER(ks_pods), C.c_void_p, C.c_uint32,
       C.POINTER(ks_node_rules), C.POINTER(ks_bind_resources), C.POINTER(ks_node_templates), C.c_void_p, C.c_void_p,
       C.c_void_p, C.c_void_p, C.c_void_p, optional=True)
KS_AFFINITY_MAX_TERMS = 16384
KS_AFFINITY_MAX_TARGETS = 1 << 22
KS_AFFINITY_MAX_EXISTING = 1 << 24
KS_AFFINITY_MAX_UPDATES = 1 << 24
KS_PREEMPT_MAX_ABS_SUM = 1 << 62
KS_ERR_INVALID, KS_ERR_PARSE, KS_ERR_RANGE = -1, -3, -5
KS_REFERENCE_ATTEMPTS = 5
_SAMPLING_MULT = 0xD1B54A32D192ED03


def sampling_stream(seed, p):
    """KS_SAMPLING_STREAM(seed, p) of include/ksched.h: start state of pod p's splitmix64 draw stream."""
    return (seed ^ (((p + 1) * _SAMPLING_MULT) & 0xFFFFFFFFFFFFFFFF)) & 0xFFFFFFFFFFFFFFFF


def declared_symbols():
    """Every function name declared in include/*.h (used by the CPU test that checks the export table)."""
    names = []
    for fn in sorted(os.listdir(INCLUDE_DIR)):
        if not fn.endswith(".h"):
            continue
        text = open(os.path.join(INCLUDE_DIR, fn)).read()
        text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
        names += re.findall(r"\b(ksh?_[a-z0-9_]+)\s*\(", text)
    return sorted(set(names))


def measure_write_bandwidth(device, dev_ptr, nbytes, iters=4):
    """GB/s of a store-only fill over a device buffer (its contents are overwritten)."""
    out = C.c_double()
    check(lib.ks_measure_write_bandwidth(int(device), C.c_void_p(int(dev_ptr)), int(nbytes), int(iters), C.byref(out)),
          "ks_measure_write_bandwidth")
    return float(out.value)


def mask_row_bytes(n_nodes):
    return int(lib.ks_mask_row_bytes(int(n_nodes)))


def mask_row_bytes_aligned(n_nodes):
    return int(lib.ks_mask_row_bytes_aligned(int(n_nodes)))


def device_count():
    return int(lib.ks_device_count())


def launch_count():
    return int(lib.ks_launch_count())
