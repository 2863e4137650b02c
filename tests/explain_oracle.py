"""CPU restatement of ks_explain's per-pod rejection counts for the tests, built on the oracle's own entry points:
the cell codes come from orc_run_packed / orc_run_faithful (fit first, then selector: src/predicates.rs:63-77), the
two halves of the fit (src/predicates.rs:42) from the same free / request values the oracle compares.
Columns: insufficient_cpu, insufficient_memory, not_enough_resources, node_selector_mismatch."""
import ctypes as C

import numpy as np


def _counts(codes, cpu_fail, mem_fail):
    out = np.empty((codes.shape[0], 4), np.uint32)
    out[:, 0] = cpu_fail.sum(axis=1)
    out[:, 1] = mem_fail.sum(axis=1)
    out[:, 2] = (codes == 1).sum(axis=1)  # ORC_CELL_NOT_ENOUGH_RESOURCES
    out[:, 3] = (codes == 2).sum(axis=1)  # ORC_CELL_NODE_SELECTOR_MISMATCH
    return out


def explain_packed(orc, free_cpu, free_mem, labels, req_cpu, req_mem, sel):
    """Packed form (cpu millicores, memory bytes, label words); free_* after the bound-pod subtraction."""
    fc, fm = np.asarray(free_cpu, np.int64), np.asarray(free_mem, np.int64)
    rc, rm = np.asarray(req_cpu, np.int64), np.asarray(req_mem, np.int64)
    codes = orc.run_packed(fc, fm, fc, fm, labels, rc, rm, sel, want_mask=False, want_codes=True)[4]
    return _counts(codes, rc[:, None] > fc[None, :], rm[:, None] > fm[None, :])


def explain_faithful(orc, cluster, pods, n_pods):
    """Object form on an orc.Cluster: every cell's code from orc_check_node_validity, free and requests in milli units
    from orc_node_available / orc_total_pod_resources."""
    codes = cluster.run(pods, n_pods, want_mask=False, want_codes=True)[4]
    avail = np.empty((cluster.n_nodes, 2), np.int64)
    for n in range(cluster.n_nodes):
        rc, avail[n] = cluster.available(n)
        assert rc == 0, rc
    req = np.empty((n_pods, 2), np.int64)
    for i in range(n_pods):
        out = (C.c_int64 * 2)()
        rc = orc.lib.orc_total_pod_resources(C.addressof(pods) + i * C.sizeof(pods._type_), out)
        assert rc == 0, rc
        req[i] = (out[0], out[1])
    return _counts(codes, req[:, :1] > avail[None, :, 0], req[:, 1:] > avail[None, :, 1])
