#!/usr/bin/env python
"""bench_fit_bind.py — cost of ks_fit_bind (ks_node_bind with the pod count and scalar resources of NodeResourcesFit)
on one H100, beside ks_node_bind on the same queue, the two calls alternated call by call in one run.

Queue and rules as bench_node_bind.py: the c2 and c3 clusters, 64 workloads x 64 pods interleaved round robin, the
default soft spread on zones3 and hostname, its taints and node affinity.  Resources (R = 2):
  - pods: allocatable 110 per node, minus the pods the cluster already binds there;
  - nvidia.com/gpu: 8 on every 20th node (the tainted GPU pool of bench_node_bind.py), 0 elsewhere; every 8th workload
    (the ones that tolerate the pool) requests 1-4 GPUs per pod, the others none.
Policies 1, 3 and 4.  Every timed call starts from the same free[] (set_bound, untimed).  us_per_pod = median / min /
max over --steps calls after --warmup untimed ones of wall-clock call time / 4096 pods (host-space pods and outputs;
the call returns after its D2H copy).  The GPU name, power limit and max SM clock are read in the same run.  Prints one
JSON line; writes nothing else."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_explain import gpu_info, spread  # noqa: E402
from bench_node_bind import PODS_PER_WORKLOAD, WORKLOADS, rules_for  # noqa: E402


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
        print(json.dumps({"error": "no CUDA device: ks_fit_bind has no CPU fallback"}), flush=True)
        return 2
    from importlib import import_module
    snapshot_mod = import_module(ks.Snapshot.__module__)
    line = {"metric": "fit_bind_us_per_pod", "unit": "us", "gpu": gpu_info(), "steps": args.steps,
            "warmup": args.warmup}
    policies = ((ks.KS_SCORE_LEAST_ALLOCATED, "least_allocated"),
                (ks.KS_SCORE_MOST_ALLOCATED, "most_allocated"), (ks.KS_SCORE_LEAST_BALANCED, "least_balanced"))
    P, G = WORKLOADS * PODS_PER_WORKLOAD, WORKLOADS
    group = (np.arange(P) % WORKLOADS).astype(np.int32)
    soft = np.tile([5, 3], (G, 1)).astype(np.uint32)
    sall = np.zeros(G, np.uint8)
    gpus = np.where(np.arange(G) % 8 == 0, 1 + (np.arange(G) // 8) % 4, 0)
    pod_req = np.stack([np.ones(P, np.int64), gpus[group].astype(np.int64)], axis=1)
    for cfg in args.configs.split(","):
        cl = ks.synth.config(cfg)
        ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
        N = len(ac)
        rng = np.random.default_rng(0x5B3)
        pick = np.sort(rng.choice(len(rc), WORKLOADS, replace=False))
        qc, qm, qs = rc[pick][group], rm[pick][group], np.ascontiguousarray(sel[pick][group])
        keys = [((np.arange(N) % 3).astype(np.int32), 3), (np.arange(N, dtype=np.int32), N)]
        rules = rules_for(np, snapshot_mod, N, G)
        node_free = np.stack([110 - np.bincount(bn, minlength=N),
                              np.where(np.arange(N) % 20 == 19, 8, 0)]).astype(np.int64)
        out = {"nodes": N, "bound_pods": len(bn), "pods": P, "gpu_pods": int((pod_req[:, 1] > 0).sum())}
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            calls = {
                "node_bind": lambda policy: snap.node_bind(qc, qm, qs, group, G, keys, policy=policy, soft_skew=soft,
                                                           soft_all_keys=sall, rules=rules, want_counts=False),
                "fit_bind": lambda policy: snap.fit_bind(qc, qm, qs, group, G, keys, policy=policy, soft_skew=soft,
                                                         soft_all_keys=sall, rules=rules, node_free=node_free,
                                                         pod_req=pod_req, want_counts=False),
            }
            for policy, pname in policies:
                us = {name: [] for name in calls}
                res = {}
                for s in range(args.warmup + args.steps):
                    for name, call in calls.items():  # alternated call by call
                        snap.set_bound(bn, bc, bm)
                        t0 = time.perf_counter()
                        res[name] = call(policy)
                        if s >= args.warmup:
                            us[name].append((time.perf_counter() - t0) * 1e6 / P)
                for name in calls:
                    r = res[name]
                    out[f"{name}/{pname}"] = {"us_per_pod": spread(us[name]), "placed": int((r[0] >= 0).sum())}
                out[f"fit_bind/{pname}"]["refused_resources"] = int(res["fit_bind"][3][:, 0].sum())
                out[f"fit_bind/{pname}"]["gpu_pods_placed"] = int(((res["fit_bind"][0] >= 0) &
                                                                   (pod_req[:, 1] > 0)).sum())
        line[cfg] = out
    line["note"] = ("host-space pods and outputs, wall clock per call / 4096 pods from the same free[]; ks_fit_bind "
                    "and ks_node_bind alternated call by call on bench_node_bind.py's queue and rules; resources: "
                    "pods 110 per node, 8 GPUs on every 20th node, every 8th workload requesting 1-4 GPUs per pod")
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
