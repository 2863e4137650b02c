#!/usr/bin/env python
"""bench_spread_multi.py — cost of ks_place_replicas_spread_multi (replica placement under one topology spread
constraint per key, every constraint binding at once) on one H100, beside the single-key call in the same run.

Workloads: the c2 and c3 clusters (bench.py's nodes and bound pods, free[] after the bound pods) with bench_spread.py's
shapes: batch = 256 pod shapes drawn with a fixed seed from the cluster's pending pods, each asking for 1 000 copies;
one = one shape asking for 65 536 copies.  Key sets, under every policy:
  - zones3 (single key, ks_place_replicas_spread, maxSkew 1): the baseline, measured in the same run;
  - zones3+hostname with maxSkew 1/1 and 1/2 (zones3 = node n in zone n % 3, hostname = one domain per node);
  - hostname+zones3, the same two keys in swapped order (the primary is still zones3: it has fewer domains).
Per workload: call_ms = median / min / max of --steps calls after --warmup untimed ones (host-space specs and outputs,
the copy list and domain counts returned; wall clock, the call returns after its D2H copy), the copies placed,
us_per_copy = median call over the copies of the longest spec, and the specs with a blocked domain on some key.  The GPU
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
from bench_spread import BATCH_REPLICAS, ONE_REPLICAS, SHAPES  # noqa: E402


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
        print(json.dumps({"error": "no CUDA device: ks_place_replicas_spread_multi has no CPU fallback"}), flush=True)
        return 2
    line = {"metric": "place_replicas_spread_multi_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps,
            "warmup": args.warmup}
    policies = ((ks.KS_SCORE_LEFTOVER, "leftover"), (ks.KS_SCORE_LEAST_ALLOCATED, "least_allocated"),
                (ks.KS_SCORE_MOST_ALLOCATED, "most_allocated"), (ks.KS_SCORE_LEAST_BALANCED, "least_balanced"))
    for cfg in args.configs.split(","):
        cl = ks.synth.config(cfg)
        ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
        N = len(ac)
        rng = np.random.default_rng(0x5B2)
        pick = np.sort(rng.choice(len(rc), SHAPES, replace=False))
        rc, rm, sel = rc[pick], rm[pick], np.ascontiguousarray(sel[pick])
        zones = ((np.arange(N) % 3).astype(np.int32), 3)
        host = (np.arange(N, dtype=np.int32), N)
        key_sets = {"zones3": ([zones], (1,)), "zones3+hostname/1-1": ([zones, host], (1, 1)),
                    "zones3+hostname/1-2": ([zones, host], (1, 2)), "hostname+zones3/1-1": ([host, zones], (1, 1)),
                    "hostname+zones3/2-1": ([host, zones], (2, 1))}
        work = {"batch": (rc, rm, sel, np.full(SHAPES, BATCH_REPLICAS, np.uint32)),
                "one": (rc[:1], rm[:1], sel[:1], np.array([ONE_REPLICAS], np.uint32))}
        out = {"nodes": N, "bound_pods": len(bn)}
        with ks.Snapshot(0) as snap:
            snap.set_nodes(ac, am, lab)
            snap.set_bound(bn, bc, bm)
            for kname, (keys, skews) in key_sets.items():
                for wname, (wrc, wrm, wsel, R) in work.items():
                    skew = np.tile(np.array(skews, np.uint32), (len(R), 1))
                    for policy, pname in policies:
                        ms = []
                        for s in range(args.warmup + args.steps):
                            t0 = time.perf_counter()
                            if len(keys) == 1:
                                rows = snap.place_replicas_spread(wrc, wrm, wsel, R, *keys[0], skew[:, 0],
                                                                  policy=policy)[0][:, None]
                            else:
                                rows = snap.place_replicas_spread_multi(wrc, wrm, wsel, R, keys, skew,
                                                                        policy=policy)[0]
                            if s >= args.warmup:
                                ms.append((time.perf_counter() - t0) * 1e3)
                        st = spread(ms)
                        longest = int(rows["placed"][:, 0].max(initial=0))
                        out[f"{kname}/{wname}/{pname}"] = {
                            "call_ms": st, "placed": int(rows["placed"][:, 0].sum()), "longest_spec": longest,
                            "us_per_copy": st["median"] * 1e3 / longest if longest else None,
                            "blocked_specs": int((rows["blocked_domain"] >= 0).any(axis=1).sum())}
        line[cfg] = out
    line["note"] = ("host-space specs and outputs, wall clock per call; batch = 256 seeded pod shapes x 1000 copies, "
                    "one = one shape x 65536 copies; zones3 = node n in zone n % 3 (single key, the baseline), "
                    "hostname = one domain per node; a/b = maxSkew of the first / second key")
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
