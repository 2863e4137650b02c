#!/usr/bin/env python
"""bench_node_bind.py — cost of ks_node_bind (ks_profile_bind with TaintToleration and NodeAffinity) on one H100, beside
ks_profile_bind on the same queue without rules in the same run, and the rule-word setup kernel alone.

Queue as bench_profile_bind.py: the c2 and c3 clusters, 64 workloads x 64 pods interleaved round robin (pod i of
workload i % 64, one seeded pod shape per workload), the system default soft spread (zone maxSkew 5, hostname 3,
ScheduleAnyway, soft_all_keys 0) on every workload.  Keys: zones3 (node n in zone n % 3) and hostname.  Rules:
  - taints: control-plane NoSchedule on nodes 0-2, a GPU pool NoSchedule on every 20th node (5%), PreferNoSchedule
    spot on every 5th node; every 8th workload tolerates the GPU pool, every 4th the spot taint;
  - node affinity over zone (z0-z2) and instance type (node n of type n % 7, t0-t6): every 4th workload requires zone
    In {z0, z1}, every 3rd type In {t0, t1, t2}; every workload prefers zone In {z2} (weight 30) and type In {t3}
    (weight 70).
Policies 1, 3 and 4; weights 3 (taint) and 2 (node affinity), the default profile's.  Every timed call starts from the
same free[] (set_bound, untimed).  call_ms = median / min / max of --steps calls after --warmup untimed ones (host-space
pods and outputs, wall clock; the call returns after its D2H copy), us_per_pod = median over the 4096 pods.  setup_us =
the device time of k_node_rules_setup per call from torch.profiler in a separate run of --steps calls (median / min /
max).  The GPU name, power limit and max SM clock are read in the same run.  Prints one JSON line; writes nothing else."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_explain import gpu_info, spread  # noqa: E402

WORKLOADS, PODS_PER_WORKLOAD = 64, 64


def rules_for(np, snapshot_mod, N, G):
    n = np.arange(N)
    hard = np.zeros(N, np.uint64)
    hard[:3] |= np.uint64(1)               # control-plane
    hard[n % 20 == 19] |= np.uint64(2)     # GPU pool
    soft = np.where(n % 5 == 4, np.uint64(4), np.uint64(0)).astype(np.uint64)  # spot
    w = np.arange(G)
    tol_h = np.where(w % 8 == 0, np.uint64(2), np.uint64(0)).astype(np.uint64)
    tol_s = np.where(w % 4 == 0, np.uint64(4), np.uint64(0)).astype(np.uint64)
    zone, itype = (n % 3).astype(np.int32), (n % 7).astype(np.int32)
    ns = snapshot_mod.node_set
    terms = []
    for g in range(G):
        if g % 4 == 0:
            terms.append((g, 0, [(0, ns(3, [0, 1]))]))
        if g % 3 == 0:
            terms.append((g, 0, [(1, ns(7, [0, 1, 2]))]))
        terms.append((g, 30, [(0, ns(3, [2]))]))
        terms.append((g, 70, [(1, ns(7, [3]))]))
    return dict(n_taints=3, taint_hard=hard, taint_soft=soft, tolerate_hard=tol_h, tolerate_soft=tol_s,
                rule_keys=[(zone, 3), (itype, 7)], node_terms=terms, weight_taint=3, weight_node_affinity=2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--configs", default="c2,c3")
    args = ap.parse_args()
    import numpy as np
    import ksched_pkg
    ks = ksched_pkg.load()
    if ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_node_bind has no CPU fallback"}), flush=True)
        return 2
    from importlib import import_module
    snapshot_mod = import_module(ks.Snapshot.__module__)
    line = {"metric": "node_bind_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup}
    policies = ((ks.KS_SCORE_LEAST_ALLOCATED, "least_allocated"),
                (ks.KS_SCORE_MOST_ALLOCATED, "most_allocated"), (ks.KS_SCORE_LEAST_BALANCED, "least_balanced"))
    P, G = WORKLOADS * PODS_PER_WORKLOAD, WORKLOADS
    group = (np.arange(P) % WORKLOADS).astype(np.int32)
    soft = np.tile([5, 3], (G, 1)).astype(np.uint32)
    sall = np.zeros(G, np.uint8)
    for cfg in args.configs.split(","):
        cl = ks.synth.config(cfg)
        ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
        N = len(ac)
        rng = np.random.default_rng(0x5B3)
        pick = np.sort(rng.choice(len(rc), WORKLOADS, replace=False))
        qc, qm, qs = rc[pick][group], rm[pick][group], np.ascontiguousarray(sel[pick][group])
        keys = [((np.arange(N) % 3).astype(np.int32), 3), (np.arange(N, dtype=np.int32), N)]
        rules = rules_for(np, snapshot_mod, N, G)
        out = {"nodes": N, "bound_pods": len(bn), "pods": P}
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)

            def timed(call):
                ms, res = [], None
                for s in range(args.warmup + args.steps):
                    snap.set_bound(bn, bc, bm)
                    t0 = time.perf_counter()
                    res = call()
                    if s >= args.warmup:
                        ms.append((time.perf_counter() - t0) * 1e3)
                return spread(ms), res

            for policy, pname in policies:
                for name, r in (("profile_bind_no_rules", None), ("node_bind", rules)):
                    if r is None:
                        call = lambda: snap.profile_bind(qc, qm, qs, group, G, keys, policy=policy, soft_skew=soft,
                                                         soft_all_keys=sall, want_counts=False)
                    else:
                        call = lambda: snap.node_bind(qc, qm, qs, group, G, keys, policy=policy, soft_skew=soft,
                                                      soft_all_keys=sall, rules=r, want_counts=False)
                    st, res = timed(call)
                    out[f"{name}/{pname}"] = {"call_ms": st, "us_per_pod": st["median"] * 1e3 / P,
                                              "placed": int((res[0] >= 0).sum()),
                                              "nodes_used": int(len(np.unique(res[0][res[0] >= 0])))}
                    if r is not None:
                        out[f"{name}/{pname}"]["refused_taint_node_affinity"] = [int(res[3][:, 0].sum()),
                                                                                 int(res[3][:, 1].sum())]
            # the setup kernel alone, in its own profiled run
            import torch
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    snap.set_bound(bn, bc, bm)
                    snap.node_bind(qc[:1], qm[:1], qs[:1], group[:1], G, keys, policy=4, soft_skew=soft,
                                   soft_all_keys=sall, rules=rules, want_counts=False)
                torch.cuda.synchronize()
            us = [e.device_time for e in prof.events() if "k_node_rules_setup" in e.name]
            out["setup_us"] = spread(us) if us else None
        line[cfg] = out
    line["note"] = ("host-space pods and outputs, wall clock per call from the same free[]; 64 workloads x 64 pods "
                    "interleaved round robin, one seeded pod shape per workload, default soft spread on zones3 and "
                    "hostname; baseline = ks_profile_bind on the same queue without rules; setup_us = "
                    "k_node_rules_setup device time from torch.profiler")
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
