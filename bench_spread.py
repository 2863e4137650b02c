#!/usr/bin/env python
"""bench_spread.py — cost of ks_place_replicas_spread (replica placement under a topology spread constraint) on one H100.

Workloads: the c2 and c3 clusters (bench.py's nodes and bound pods, free[] after the bound pods), each with two
topology keys: three zones (node n in zone n % 3) and the hostname key (node n its own domain, D = N).  On each, under
every policy and with maxSkew 1:
  - batch: 256 pod shapes drawn with a fixed seed from the cluster's pending pods (their requests and selectors), each
    asking for 1 000 copies: the scale-out of many Deployments at once;
  - one: one shape asking for 65 536 copies (the per-spec limit): the cost of one long sequential plan.
Per workload: call_ms = median / min / max of --steps calls after --warmup untimed ones (host-space specs and outputs,
the copy list and domain counts returned; wall clock, the call returns after its D2H copy), the copies placed, and
us_per_copy = median call over the copies of the longest spec (copies are placed one at a time per spec, so that spec
bounds the call).  The GPU name, power limit and max SM clock are read in the same run.  Prints one JSON line; writes
nothing else."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_explain import gpu_info, spread  # noqa: E402

SHAPES = 256
BATCH_REPLICAS = 1000
ONE_REPLICAS = 65536


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
        print(json.dumps({"error": "no CUDA device: ks_place_replicas_spread has no CPU fallback"}), flush=True)
        return 2
    line = {"metric": "place_replicas_spread_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps,
            "warmup": args.warmup, "max_skew": 1}
    policies = ((ks.KS_SCORE_LEFTOVER, "leftover"), (ks.KS_SCORE_LEAST_ALLOCATED, "least_allocated"),
                (ks.KS_SCORE_MOST_ALLOCATED, "most_allocated"), (ks.KS_SCORE_LEAST_BALANCED, "least_balanced"))
    for cfg in args.configs.split(","):
        cl = ks.synth.config(cfg)
        ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
        N = len(ac)
        rng = np.random.default_rng(0x5B2)
        pick = np.sort(rng.choice(len(rc), SHAPES, replace=False))
        rc, rm, sel = rc[pick], rm[pick], np.ascontiguousarray(sel[pick])
        keys = {"zones3": ((np.arange(N) % 3).astype(np.int32), 3), "hostname": (np.arange(N, dtype=np.int32), N)}
        work = {"batch": (rc, rm, sel, np.full(SHAPES, BATCH_REPLICAS, np.uint32)),
                "one": (rc[:1], rm[:1], sel[:1], np.array([ONE_REPLICAS], np.uint32))}
        out = {"nodes": N, "bound_pods": len(bn)}
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            snap.set_bound(bn, bc, bm)
            for kname, (dom, D) in keys.items():
                for wname, (wrc, wrm, wsel, R) in work.items():
                    skew = np.ones(len(R), np.uint32)
                    for policy, pname in policies:
                        ms = []
                        for s in range(args.warmup + args.steps):
                            t0 = time.perf_counter()
                            rows = snap.place_replicas_spread(wrc, wrm, wsel, R, dom, D, skew, policy=policy)[0]
                            if s >= args.warmup:
                                ms.append((time.perf_counter() - t0) * 1e3)
                        st = spread(ms)
                        longest = int(rows["placed"].max(initial=0))
                        out[f"{kname}/{wname}/{pname}"] = {
                            "call_ms": st, "placed": int(rows["placed"].sum()), "longest_spec": longest,
                            "us_per_copy": st["median"] * 1e3 / longest if longest else None,
                            "blocked_specs": int((rows["blocked_domain"] >= 0).sum())}
        line[cfg] = out
    line["note"] = ("host-space specs and outputs, wall clock per call; batch = 256 seeded pod shapes x 1000 copies, "
                    "one = one shape x 65536 copies; zones3 = node n in zone n % 3, hostname = one domain per node")
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
