#!/usr/bin/env python
"""bench_profile_bind.py — cost of ks_profile_bind (a mixed pod queue bound one pod at a time, scored with soft topology
spread and preferred inter-pod affinity as the default profile scores) on one H100, beside ks_affinity_bind on the same
queue in the same run.

Workloads and queue as bench_spread_bind.py: the c2 and c3 clusters, 64 workloads x 64 pods interleaved round robin
(pod i of workload i % 64, one seeded pod shape per workload).  Keys: zones3 (node n in zone n % 3), hostname (one domain
per node) and rack (node n in rack n // 3: thousands of domains of three nodes, so distinct domains are counted through
the domain bitmaps rather than by node count).  Mixes:
  - none: no soft term;
  - default-spread: the system default constraints, zone maxSkew 5 and hostname 3, ScheduleAnyway, soft_all_keys 0;
  - rack-spread: zone 5 and rack 3 (the bitmap path for the rack key);
  - zone+host-anti-pref: zone soft maxSkew 1 and preferred hostname self anti-affinity of weight 100;
  - zone-affinity-pref: every odd workload preferred-affine (weight 100) to the even one before it on zone.
The baseline is ks_affinity_bind with no term on the same queue, once per cluster and policy.  Policies 1, 3 and 4;
weights 2 and 2, hard_affinity_weight 1.  Every timed call starts from the same free[] (set_bound, untimed).  call_ms =
median / min / max of --steps calls after --warmup untimed ones (host-space pods and outputs, wall clock; the call returns
after its D2H copy), us_per_pod = median over the 4096 pods, the pods placed and the distinct nodes they used.  The GPU
name, power limit and max SM clock are read in the same run.  Prints one JSON line; writes nothing else."""
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
        print(json.dumps({"error": "no CUDA device: ks_profile_bind has no CPU fallback"}), flush=True)
        return 2
    line = {"metric": "profile_bind_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup}
    policies = ((ks.KS_SCORE_LEAST_ALLOCATED, "least_allocated"),
                (ks.KS_SCORE_MOST_ALLOCATED, "most_allocated"), (ks.KS_SCORE_LEAST_BALANCED, "least_balanced"))
    P, G = WORKLOADS * PODS_PER_WORKLOAD, WORKLOADS
    group = (np.arange(P) % WORKLOADS).astype(np.int32)
    anti, aff = ks.capi.KS_POD_ANTI_AFFINITY_PREFERRED, ks.capi.KS_POD_AFFINITY_PREFERRED
    for cfg in args.configs.split(","):
        cl = ks.synth.config(cfg)
        ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
        N = len(ac)
        rng = np.random.default_rng(0x5B3)
        pick = np.sort(rng.choice(len(rc), WORKLOADS, replace=False))
        qc, qm, qs = rc[pick][group], rm[pick][group], np.ascontiguousarray(sel[pick][group])
        keys = [((np.arange(N) % 3).astype(np.int32), 3), (np.arange(N, dtype=np.int32), N),
                ((np.arange(N) // 3).astype(np.int32), (N + 2) // 3)]
        host_anti = [(w, anti, 1, [w]) for w in range(G)]
        zone_aff = [(w, aff, 0, [w - 1]) for w in range(1, G, 2)]
        mixes = {"none": ([], None, None), "default-spread": ([], np.tile([5, 3, 0], (G, 1)).astype(np.uint32), 0),
                 "rack-spread": ([], np.tile([5, 0, 3], (G, 1)).astype(np.uint32), 0),
                 "zone+host-anti-pref": (host_anti, np.tile([1, 0, 0], (G, 1)).astype(np.uint32), 1),
                 "zone-affinity-pref": (zone_aff, None, 1)}
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
                st, res = timed(lambda: snap.affinity_bind(qc, qm, qs, group, G, keys, policy=policy,
                                                           want_counts=False))
                out[f"baseline_affinity_bind/{pname}"] = {
                    "call_ms": st, "us_per_pod": st["median"] * 1e3 / P, "placed": int((res[0] >= 0).sum()),
                    "nodes_used": int(len(np.unique(res[0][res[0] >= 0])))}
                for mname, (terms, soft, soft_all) in mixes.items():
                    sa = None if soft_all is None else np.full(G, soft_all, np.uint8)
                    tw = [100] * len(terms) if terms else None
                    st, res = timed(lambda: snap.profile_bind(qc, qm, qs, group, G, keys, terms, policy=policy,
                                                              soft_skew=soft, soft_all_keys=sa, term_weight=tw,
                                                              want_counts=False))
                    out[f"{mname}/{pname}"] = {"call_ms": st, "us_per_pod": st["median"] * 1e3 / P,
                                               "placed": int((res[0] >= 0).sum()),
                                               "nodes_used": int(len(np.unique(res[0][res[0] >= 0])))}
        line[cfg] = out
    line["note"] = ("host-space pods and outputs, wall clock per call from the same free[]; 64 workloads x 64 pods "
                    "interleaved round robin, one seeded pod shape per workload; zones3 = node n in zone n % 3, "
                    "hostname = one domain per node, rack = node n // 3; baseline = ks_affinity_bind on the same queue "
                    "with no term")
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
