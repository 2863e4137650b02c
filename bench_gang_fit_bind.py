#!/usr/bin/env python
"""bench_gang_fit_bind.py — cost of ks_gang_fit_bind (ks_fit_bind with gangs placed all or nothing) on one H100.

Queue, rules and resources as bench_fit_bind.py: the c2 and c3 clusters, 64 workloads x 64 pods interleaved round
robin, the default soft spread on zones3 and hostname, bench_node_bind.py's taints and node affinity, pods 110 per node
and 8 GPUs on every 20th node.  Policy 4 (the default profile).  Two measurements:
  - committed: the queue cut into gangs of 64 pods with min_member 0, so every gang commits and the outputs are
    ks_fit_bind's (M1); ks_gang_fit_bind and ks_fit_bind alternated call by call;
  - rollback: one workload spread over hostnames at maxSkew 1, queued as one gang of S pods (S = 8 to 4,096) whose
    last pod fits no node, so the gang binds S - 1 pods and rolls them back.  The rollback's cost is the call's time
    less that of the same queue with min_member 0 (the gang commits), the two alternated call by call.
Every timed call starts from the same free[] (set_bound, untimed).  Times are medians / min / max over --steps calls
after --warmup untimed ones of the wall-clock call time (host-space pods and outputs; the call returns after its D2H
copy).  The GPU name, power limit and max SM clock are read in the same run.  Prints one JSON line; writes nothing
else."""
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

SIZES = (8, 64, 512, 4096)


def timed(snap, bound, calls, steps, warmup):
    """Wall-clock us of each call, alternated call by call, every call from the same free[]"""
    us = {name: [] for name in calls}
    res = {}
    for s in range(warmup + steps):
        for name, call in calls.items():
            snap.set_bound(*bound)
            t0 = time.perf_counter()
            res[name] = call()
            if s >= warmup:
                us[name].append((time.perf_counter() - t0) * 1e6)
    return us, res


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
        print(json.dumps({"error": "no CUDA device: ks_gang_fit_bind has no CPU fallback"}), flush=True)
        return 2
    from importlib import import_module
    snapshot_mod = import_module(ks.Snapshot.__module__)
    line = {"metric": "gang_fit_bind_us", "unit": "us", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup}
    policy = ks.KS_SCORE_LEAST_BALANCED
    P, G = WORKLOADS * PODS_PER_WORKLOAD, WORKLOADS
    group = (np.arange(P) % WORKLOADS).astype(np.int32)
    soft = np.tile([5, 3], (G, 1)).astype(np.uint32)
    sall = np.zeros(G, np.uint8)
    gpus = np.where(np.arange(G) % 8 == 0, 1 + (np.arange(G) // 8) % 4, 0)
    pod_req = np.stack([np.ones(P, np.int64), gpus[group].astype(np.int64)], axis=1)
    offset = np.arange(0, P + 1, 64, dtype=np.uint64)
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
        out = {"nodes": N, "bound_pods": len(bn), "pods": P}
        common = dict(policy=policy, soft_skew=soft, soft_all_keys=sall, rules=rules, node_free=node_free,
                      want_counts=False)
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            mm0 = np.zeros(len(offset) - 1, np.uint32)
            calls = {
                "fit_bind": lambda: snap.fit_bind(qc, qm, qs, group, G, keys, pod_req=pod_req, **common),
                "gang_fit_bind": lambda: snap.gang_fit_bind(qc, qm, qs, group, G, keys, offset, mm0, pod_req=pod_req,
                                                            **common),
            }
            us, res = timed(snap, (bn, bc, bm), calls, args.steps, args.warmup)
            same = all(np.array_equal(a, b) for a, b in zip(res["fit_bind"][:4], res["gang_fit_bind"][:4]))
            out["committed"] = {name: {"us_per_pod": spread([u / P for u in us[name]]),
                                       "placed": int((res[name][0] >= 0).sum())} for name in calls}
            out["committed"]["same_outputs"] = bool(same)
            # one hostname-spread workload as one gang whose last pod fits no node
            wl = 1  # a workload that does not ask for GPUs
            for S in SIZES:
                gc = np.full(S, qc[wl], np.int64)
                gc[-1] = 1 << 36
                gm, gs = np.full(S, qm[wl], np.int64), np.ascontiguousarray(np.repeat(qs[wl:wl + 1], S, axis=0))
                gg = np.zeros(S, np.int32)
                skew = np.array([[0, 1]], np.uint32)
                req = np.stack([np.ones(S, np.int64), np.zeros(S, np.int64)], axis=1)
                off = np.array([0, S], np.uint64)
                kw = dict(max_skew=skew, pod_req=req, policy=policy, node_free=node_free, want_counts=False)
                calls = {
                    "commit": lambda: snap.gang_fit_bind(gc, gm, gs, gg, 1, keys, off, [0], **kw),
                    "rollback": lambda: snap.gang_fit_bind(gc, gm, gs, gg, 1, keys, off, [S], **kw),
                }
                us, res = timed(snap, (bn, bc, bm), calls, args.steps, args.warmup)
                c, r = np.median(us["commit"]), np.median(us["rollback"])
                out[f"rollback/{S}"] = {"commit_us": spread(us["commit"]), "rollback_us": spread(us["rollback"]),
                                        "placed": int(res["rollback"][7][0]),
                                        "rollback_cost_us": round(float(r - c), 1),
                                        "rolled_back": bool((res["rollback"][0] < 0).all())}
        line[cfg] = out
    line["note"] = ("host-space pods and outputs, wall clock per call from the same free[]; committed: "
                    "bench_fit_bind.py's queue in gangs of 64 with min_member 0, alternated call by call with "
                    "ks_fit_bind; rollback: one hostname-spread gang of S pods whose last pod fits no node, against "
                    "the same gang with min_member 0")
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
