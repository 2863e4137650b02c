#!/usr/bin/env python
"""bench_fit_preempt.py — cost of ks_fit_preempt (preemption under the full filter: rule words, the victim index with
its request columns, k_fit_preempt_scan, k_fit_preempt_emit) on one H100, beside ks_preempt.

Workload:
  - bench_preempt.py's cluster: c3 (50k nodes, 500k bound pods) with bound-pod priorities drawn (seeded) from
    {0, 100, 1000, 10000}, plus one skewed node (node 0) holding 5 000 more small bound pods;
  - bench_fit_bind.py's GPU pool: 8 nvidia.com/gpu on every 20th node, tainted (bench_node_bind.py's rules: the
    control-plane and GPU-pool NoSchedule taints, the spot PreferNoSchedule taint and its required and preferred node
    affinity over 64 workloads); every pool node's 8 GPUs are held by two more bound pods of 4 GPUs at priority 0;
  - pods allocatable 110 on every node (minus the pods bound there);
  - 10 000 pending pods at priority 1000 in 64 workloads round robin, bench_preempt.py's first c3 pods with their
    requests raised until 90% of the cells fail on cpu or memory; the pods of every 8th workload (those that tolerate
    the pool) request 1-8 GPUs.
Host-space pods and outputs (ks_fit_preempt takes no other), max_victims 16.  Each figure is the median (and min / max)
of --steps calls after --warmup untimed ones, each timed by CUDA events recorded around the call, which returns after
its stream synchronise:
  - fit_preempt_ms: the whole call;
  - index_build_ms: a call with one pod (the rule words and the victim index plus a one-pod scan);
  - preempt_ms and fit_preempt_q1_ms: ks_preempt on the same cpu and memory inputs and ks_fit_preempt with rules and
    resources NULL and every pod in group -1 (identity Q1: the same rows), alternated call by call.
The GPU name, power limit and max SM clock are read in the same run.  Prints one JSON line; writes nothing."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_explain import gpu_info, spread  # noqa: E402
from bench_node_bind import rules_for  # noqa: E402

PODS, SKEW, WORKLOADS = 10_000, 5_000, 64
LEVELS = (0, 100, 1000, 10000)
POD_PRIORITY = 1000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-victims", type=int, default=16)
    args = ap.parse_args()
    import numpy as np
    import torch
    import ksched_pkg
    ks = ksched_pkg.load()
    if not torch.cuda.is_available() or ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_fit_preempt has no CPU fallback"}), flush=True)
        return 2
    from importlib import import_module
    snapshot_mod = import_module(ks.Snapshot.__module__)
    cl = ks.synth.config("c3")
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    N = len(ac)
    rng = np.random.default_rng(0xB2000003)
    bn = np.concatenate([bn, np.zeros(SKEW, np.int32)])  # the skewed node: node 0
    bc = np.concatenate([bc, np.full(SKEW, 1, np.int64)])
    bm = np.concatenate([bm, np.full(SKEW, 1 << 20, np.int64)])
    bp = rng.choice(np.array(LEVELS, np.int32), len(bn))
    pool = np.nonzero(np.arange(N) % 20 == 19)[0].astype(np.int32)
    B0 = len(bn)
    bn = np.concatenate([bn, np.repeat(pool, 2)])  # two 4-GPU batch pods on every pool node
    bc = np.concatenate([bc, np.full(2 * len(pool), 1000, np.int64)])
    bm = np.concatenate([bm, np.full(2 * len(pool), 1 << 30, np.int64)])
    bp = np.concatenate([bp, np.zeros(2 * len(pool), np.int32)])
    bgpu = np.concatenate([np.zeros(B0, np.int64), np.full(2 * len(pool), 4, np.int64)])
    bound_req = np.stack([np.ones(len(bn), np.int64), bgpu], axis=1)
    node_free = np.stack([110 - np.bincount(bn, minlength=N), np.where(np.arange(N) % 20 == 19, 8, 0)
                          - np.bincount(bn, weights=bgpu, minlength=N).astype(np.int64)]).astype(np.int64)
    rc, rm, sel = rc[:PODS].copy(), rm[:PODS].copy(), np.ascontiguousarray(sel[:PODS])
    group = (np.arange(PODS) % WORKLOADS).astype(np.int32)
    gpus = np.where(group % 8 == 0, 1 + (np.arange(PODS) // WORKLOADS) % 8, 0).astype(np.int64)
    pod_req = np.stack([np.ones(PODS, np.int64), gpus], axis=1)
    rules = rules_for(np, snapshot_mod, N, WORKLOADS)
    pp = np.full(PODS, POD_PRIORITY, np.int32)
    mv = args.max_victims
    stream = torch.cuda.current_stream()
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        fc, fm = snap.free()
        factor = 1
        for factor in range(1, 65):  # raise the requests until most nodes fail on resources
            fail = ~((rc[:200, None] * factor <= fc[None, :]) & (rm[:200, None] * factor <= fm[None, :]))
            if fail.mean() >= 0.9:
                break
        rc, rm = rc * factor, rm * factor
        ones = np.full(PODS, -1, np.int32)

        def fit(n):
            return lambda: snap.fit_preempt(rc[:n], rm[:n], sel[:n], pp[:n], group[:n], WORKLOADS, bn, bc, bm, bp, mv,
                                            rules=rules, node_free=node_free, pod_req=pod_req[:n], bound_req=bound_req)

        def q1():
            return snap.fit_preempt(rc, rm, sel, pp, ones, 0, bn, bc, bm, bp, mv)

        def preempt():
            return snap.preempt(rc, rm, sel, pp, bn, bc, bm, bp, mv)

        def timed(fns):
            """CUDA-event times of each function, alternated call by call; and the last results"""
            out = [None] * len(fns)
            for _ in range(max(args.warmup, 1)):
                for i, fn in enumerate(fns):
                    out[i] = fn()
            ms = [[] for _ in fns]
            for _ in range(args.steps):
                for i, fn in enumerate(fns):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(stream)
                    out[i] = fn()
                    b.record(stream)
                    b.synchronize()
                    ms[i].append(a.elapsed_time(b))
            return ms, out

        (f_ms,), ((rows, vic, unres),) = timed([fit(PODS)])
        (i_ms,), _ = timed([fit(1)])
        (p_ms, q_ms), (p_out, q_out) = timed([preempt, q1])
        assert all(np.array_equal(p_out[0][f], q_out[0][f]) for f in rows.dtype.names), "Q1: rows differ"
        assert np.array_equal(p_out[1], q_out[1]), "Q1: victims differ"
        assert np.array_equal(snap.free()[0], fc), "free[] changed"
    planned = rows["node_idx"] >= 0
    line = {"metric": "fit_preempt_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
            "workload": f"c3 nodes ({N}), {len(bn)} bound pods ({SKEW} on node 0, {2 * len(pool)} GPU batch pods on "
                        f"{len(pool)} tainted 8-GPU nodes), pods allocatable 110, {PODS} pods at priority "
                        f"{POD_PRIORITY} in {WORKLOADS} workloads ({int((gpus > 0).sum())} requesting 1-8 GPUs), "
                        f"requests x{factor}, max_victims {mv}",
            "fit_preempt_ms": spread(f_ms), "index_build_ms": spread(i_ms), "preempt_ms": spread(p_ms),
            "fit_preempt_q1_ms": spread(q_ms),
            "q1_vs_preempt": statistics.median(q_ms) / statistics.median(p_ms),
            "pods_with_plan": int(planned.sum()), "gpu_pods_with_plan": int((planned & (gpus > 0)).sum()),
            "gpu_pods_with_plan_ks_preempt": int(((p_out[0]["node_idx"] >= 0) & (gpus > 0)).sum()),
            "pods_feasible": int((rows["feasible_cnt"] > 0).sum()),
            "unresolvable_mean": float(unres.mean()), "victims": int(rows["n_victims"].sum()),
            "note": "host-space pods and outputs; CUDA events around each call (the call ends in a stream synchronise), "
                    "no L2 flush; index_build_ms is a one-pod call; preempt_ms and fit_preempt_q1_ms alternated call "
                    "by call"}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
