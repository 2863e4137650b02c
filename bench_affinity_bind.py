#!/usr/bin/env python
"""bench_affinity_bind.py — cost of ks_affinity_bind (a mixed pod queue bound one pod at a time under spread and required
inter-pod affinity / anti-affinity) on one H100, beside ks_spread_bind on the same queue in the same run.

Workloads, queue and key sets as bench_spread_bind.py: the c2 and c3 clusters, 64 workloads x 64 pods interleaved round
robin (pod i of workload i % 64, one seeded pod shape per workload), zones3 (node n in zone n % 3) and hostname (one
domain per node).  Mixes:
  - none: no terms, no spread (baseline: ks_spread_bind with every max_skew 0);
  - host-anti: every workload anti-affine to itself on hostname (at most one pod per node), no spread;
  - zone-affinity: every odd workload affine to the even one before it on zone, no spread;
  - zone-spread+host-anti: every workload zone spread maxSkew 1 and hostname self anti-affinity (baseline:
    ks_spread_bind with the zone spread alone).
Every policy.  Every timed call starts from the same free[] (set_bound, untimed).  call_ms = median / min / max of
--steps calls after --warmup untimed ones (host-space pods and outputs, wall clock; the call returns after its D2H copy),
us_per_pod = median over the 4096 pods, and the pods placed and refused by affinity.  The GPU name, power limit and max
SM clock are read in the same run.  Prints one JSON line; writes nothing else."""
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
        print(json.dumps({"error": "no CUDA device: ks_affinity_bind has no CPU fallback"}), flush=True)
        return 2
    line = {"metric": "affinity_bind_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup}
    policies = ((ks.KS_SCORE_LEFTOVER, "leftover"), (ks.KS_SCORE_LEAST_ALLOCATED, "least_allocated"),
                (ks.KS_SCORE_MOST_ALLOCATED, "most_allocated"), (ks.KS_SCORE_LEAST_BALANCED, "least_balanced"))
    P, G = WORKLOADS * PODS_PER_WORKLOAD, WORKLOADS
    group = (np.arange(P) % WORKLOADS).astype(np.int32)
    anti, aff = ks.capi.KS_POD_ANTI_AFFINITY, ks.capi.KS_POD_AFFINITY
    for cfg in args.configs.split(","):
        cl = ks.synth.config(cfg)
        ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
        N = len(ac)
        rng = np.random.default_rng(0x5B3)
        pick = np.sort(rng.choice(len(rc), WORKLOADS, replace=False))
        qc, qm, qs = rc[pick][group], rm[pick][group], np.ascontiguousarray(sel[pick][group])
        keys = [((np.arange(N) % 3).astype(np.int32), 3), (np.arange(N, dtype=np.int32), N)]
        host_anti = [(w, anti, 1, [w]) for w in range(G)]
        no_skew, zone_skew = np.zeros((G, 2), np.uint32), np.tile([1, 0], (G, 1)).astype(np.uint32)
        mixes = {"none": ([], None, no_skew), "host-anti": (host_anti, None, no_skew),
                 "zone-affinity": ([(w, aff, 0, [w - 1]) for w in range(1, G, 2)], None, no_skew),
                 "zone-spread+host-anti": (host_anti, zone_skew, zone_skew)}
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
                for mname, (terms, skew, base_skew) in mixes.items():
                    st, res = timed(lambda: snap.spread_bind(qc, qm, qs, group, keys, base_skew, policy=policy,
                                                             want_counts=False))
                    out[f"{mname}/baseline_spread_bind/{pname}"] = {"call_ms": st, "us_per_pod": st["median"] * 1e3 / P,
                                                                    "placed": int((res[0] >= 0).sum())}
                    st, res = timed(lambda: snap.affinity_bind(qc, qm, qs, group, G, keys, terms, None, skew,
                                                               policy=policy, want_counts=False))
                    out[f"{mname}/{pname}"] = {"call_ms": st, "us_per_pod": st["median"] * 1e3 / P,
                                               "placed": int((res[0] >= 0).sum()),
                                               "refused_by_affinity": int(((res[0] < 0) & (res[2][:, 1] > 0)).sum())}
        line[cfg] = out
    line["note"] = ("host-space pods and outputs, wall clock per call from the same free[]; 64 workloads x 64 pods "
                    "interleaved round robin, one seeded pod shape per workload; zones3 = node n in zone n % 3, "
                    "hostname = one domain per node; baseline = ks_spread_bind on the same queue (every max_skew 0, or "
                    "the zone spread of the mix)")
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
