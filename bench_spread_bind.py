#!/usr/bin/env python
"""bench_spread_bind.py — cost of ks_spread_bind (a mixed pod queue bound one pod at a time under each workload's topology
spread constraints) on one H100, beside ks_gang_bind with singleton groups (the same sequential reconcile without
spread) on the same queue in the same run.

Workloads: the c2 and c3 clusters (bench.py's nodes and bound pods, free[] after the bound pods).  The queue is 64
workloads x 64 pods, interleaved round robin (4096 pods; pod i belongs to workload i % 64); workload w's pods all carry
pod shape w, the 64 shapes drawn with a fixed seed from the cluster's pending pods.  Key sets: zones3 (node n in zone
n % 3, as bench_spread_multi.py) and zones3+hostname (one domain per node).  Constraint mixes, maxSkew 1 throughout:
  - none: every workload unconstrained (max_skew 0);
  - zone: every workload constrains the zone key only;
  - thirds (zones3+hostname only): workload w % 3 = 0 none, 1 zone, 2 zone and hostname.
Every policy.  Every timed call starts from the same free[] (set_bound, untimed).  Per workload: call_ms = median / min /
max of --steps calls after --warmup untimed ones (host-space pods and outputs, wall clock; the call returns after its
D2H copy), us_per_pod = median over the 4096 pods, the pods placed and the pods the spread rule refused (unbound with a
refusal).  baseline = ks_gang_bind with one singleton group per pod and min_member 0 on the same queue.  The GPU name,
power limit and max SM clock are read in the same run.  Prints one JSON line; writes nothing else."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--configs", default="c2,c3")
    args = ap.parse_args()
    import numpy as np
    import ksched_pkg
    ks = ksched_pkg.load()
    if ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_spread_bind has no CPU fallback"}), flush=True)
        return 2
    line = {"metric": "spread_bind_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup}
    policies = ((ks.KS_SCORE_LEFTOVER, "leftover"), (ks.KS_SCORE_LEAST_ALLOCATED, "least_allocated"),
                (ks.KS_SCORE_MOST_ALLOCATED, "most_allocated"), (ks.KS_SCORE_LEAST_BALANCED, "least_balanced"))
    P = WORKLOADS * PODS_PER_WORKLOAD
    group = (np.arange(P) % WORKLOADS).astype(np.int32)
    for cfg in args.configs.split(","):
        cl = ks.synth.config(cfg)
        ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
        N = len(ac)
        rng = np.random.default_rng(0x5B3)
        pick = np.sort(rng.choice(len(rc), WORKLOADS, replace=False))
        qc, qm, qs = rc[pick][group], rm[pick][group], np.ascontiguousarray(sel[pick][group])
        zones = ((np.arange(N) % 3).astype(np.int32), 3)
        host = (np.arange(N, dtype=np.int32), N)
        w = np.arange(WORKLOADS)
        runs = {"zones3/none": ([zones], np.zeros((WORKLOADS, 1))), "zones3/zone": ([zones], np.ones((WORKLOADS, 1))),
                "zones3+hostname/none": ([zones, host], np.zeros((WORKLOADS, 2))),
                "zones3+hostname/zone": ([zones, host], np.tile([1, 0], (WORKLOADS, 1))),
                "zones3+hostname/thirds": ([zones, host], np.stack([w % 3 >= 1, w % 3 == 2], 1))}
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
                st, res = timed(lambda: snap.gang_bind(qc, qm, qs, np.arange(P + 1), np.zeros(P), policy))
                out[f"baseline_gang_singletons/{pname}"] = {"call_ms": st, "us_per_pod": st["median"] * 1e3 / P,
                                                           "placed": int((res[0] >= 0).sum())}
                for rname, (keys, skew) in runs.items():
                    st, res = timed(lambda: snap.spread_bind(qc, qm, qs, group, keys, skew, policy=policy,
                                                             want_counts=False))
                    out[f"{rname}/{pname}"] = {"call_ms": st, "us_per_pod": st["median"] * 1e3 / P,
                                               "placed": int((res[0] >= 0).sum()),
                                               "refused_by_spread": int(((res[0] < 0) & (res[2] > 0)).sum())}
        line[cfg] = out
    line["note"] = ("host-space pods and outputs, wall clock per call from the same free[]; 64 workloads x 64 pods "
                    "interleaved round robin, one seeded pod shape per workload; zones3 = node n in zone n % 3, "
                    "hostname = one domain per node, maxSkew 1; baseline = ks_gang_bind with singleton groups")
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
