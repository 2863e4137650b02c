"""CPU restatement of gangs when binding (ks_gang_fit_bind, include/ksched.h; DESIGN.md 5s), from the definition.

Gang j is tried by running fit_bind_oracle.fit_bind_packed from the call's initial state over the pods of the gangs
committed so far followed by gang j's pods; the gang commits iff at least min_member[j] of its own pods bound there.
So no state is ever rolled back here: each try starts again from the inputs.  This is quadratic in the queue, which the
CPU sizes keep small, and shares no code with any rollback.  A committed gang's pods keep the outputs of the last run
(a run over a prefix binds as the longer run does); a rolled-back gang's pods get node -1, score 0, zero parts and the
refusal words of its own try."""
import numpy as np

from fit_bind_oracle import fit_bind_packed


def gangs_of(offset):
    """Gang j's pod indices, for the cut offset [n + 1]."""
    offset = [int(o) for o in np.asarray(offset).reshape(-1)]
    return [list(range(offset[j], offset[j + 1])) for j in range(len(offset) - 1)]


def gang_fit_bind_packed(free_cpu, free_mem, alloc_cpu, alloc_mem, labels, req_cpu, req_mem, sel, group, n_groups,
                         keys, node_labels, node_taints, group_rules, alloc, bound, pod_res, offset, min_member,
                         **kw):
    """Returns (node_idx [P], score [P], parts [P, 5], refused [P, 5], counts, soft_counts, usage, placed [n]) as
    Snapshot.gang_fit_bind with a NodeUsage in place of free_r; free_cpu / free_mem are charged in place with the
    committed gangs' pods.  kw are fit_bind_packed's keywords."""
    P = len(req_cpu)
    req_cpu, req_mem = np.asarray(req_cpu, np.int64).reshape(P), np.asarray(req_mem, np.int64).reshape(P)
    sel = np.asarray(sel, np.uint64).reshape(P, -1)
    group = np.asarray(group, np.int64).reshape(P)
    fc0, fm0 = np.array(free_cpu, np.int64), np.array(free_mem, np.int64)

    def walk(pods):
        fc, fm = fc0.copy(), fm0.copy()
        out = fit_bind_packed(fc, fm, alloc_cpu, alloc_mem, labels, req_cpu[pods], req_mem[pods], sel[pods],
                              group[pods], n_groups, keys, node_labels, node_taints, group_rules, alloc, bound,
                              [pod_res[p] for p in pods], **kw)
        return out, fc, fm

    node = np.full(P, -1, np.int32)
    score = np.zeros(P, np.int64)
    parts = np.zeros((P, 5), np.int64)
    refused = np.zeros((P, 5), np.uint32)
    gangs = gangs_of(offset)
    placed = np.zeros(len(gangs), np.uint32)
    committed = []
    for j, pods in enumerate(gangs):
        (tn, _, _, tref, _, _, _), _, _ = walk(committed + pods)
        own = tn[len(committed):]
        placed[j] = int((own >= 0).sum())
        refused[pods] = tref[len(committed):]
        if placed[j] >= int(min_member[j]):
            committed += pods
    (cn, cs, cp, cr, counts, soft, usage), fc, fm = walk(committed)
    node[committed], score[committed], parts[committed], refused[committed] = cn, cs, cp, cr
    free_cpu[:], free_mem[:] = fc, fm
    return node, score, parts, refused, counts, soft, usage, placed


def golden_inputs(case):
    """fit_bind_packed's arguments and keywords for one case of tests/golden/gv1_gang_fit_bind.json (without the
    gangs): nodes without labels, 1 GiB of memory per pod."""
    N, P = len(case["free_cpu"]), len(case["pods"]["cpu"])
    fc = np.array(case["free_cpu"], np.int64)
    fm = np.full(N, case["mem"], np.int64)
    ac, am = np.array(case["alloc_cpu"], np.int64), fm.copy()
    rc, rm = np.array(case["pods"]["cpu"], np.int64), np.full(P, 1 << 30, np.int64)
    group = np.array(case["pods"]["group"], np.int32)
    keys = [(np.array(k["domain"], np.int32), int(k["n"])) for k in case["keys"]]
    args = (fc, fm, ac, am, np.zeros((N, 1), np.uint64), rc, rm, np.zeros((P, 1), np.uint64), group, case["groups"],
            keys, [{}] * N, case["taints"], case["group_rules"], case["alloc"], [], case["pods"]["res"])
    kw = dict(terms=[(o, k, key, t) for o, k, key, t in case.get("terms", [])], policy=case["policy"])
    if "max_skew" in case:
        kw["max_skew"] = np.array(case["max_skew"], np.uint32)
    if "existing" in case:
        kw["existing"] = [np.array(e, np.uint32) for e in case["existing"]]
    return args, kw
