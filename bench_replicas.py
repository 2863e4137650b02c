#!/usr/bin/env python
"""bench_replicas.py — cost of ks_place_replicas (replica placement) on one H100.

Workload: the c3 cluster (bench.py's nodes and bound pods, free[] after the bound pods) and 256 pod shapes drawn with a
fixed seed from its pending pods, keeping their requests and selectors, each asking for R = 10 000 copies.  This is the
question a controller asks when a Deployment, ReplicaSet or Job scales out, and capacity dashboards ask for every
workload shape.  Specs and outputs are host memory, as ks_place_replicas takes them.
  - call_ms per policy: the whole call, median / min / max of --steps calls after --warmup untimed ones, with the copy
    list (out_node and out_score) and without it (the capacity query);
  - one_shape_with_copies: for the 4 shapes of the gang comparison, a plan call with that one shape alone (median per
    shape, its copies checked equal to the batched plan's), so the method is compared without the batching;
  - gang: the exact one-copy-at-a-time answer the library had before, ks_gang_bind with 10 000 singleton groups, for 4
    of the shapes under each policy, each on a freshly loaded snapshot (the call charges free[]); its nodes and scores
    are checked equal to the plan's, and gang_ms is the median call;
  - placed: copies placed over all shapes, and shapes whose capacity is below R.
The GPU name, power limit and max SM clock are read in the same run.  Prints one JSON line; writes nothing else."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_explain import gpu_info, spread  # noqa: E402

SHAPES = 256
REPLICAS = 10000
GANG_SHAPES = 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import numpy as np
    import ksched_pkg
    ks = ksched_pkg.load()
    if ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_place_replicas has no CPU fallback"}), flush=True)
        return 2
    cl = ks.synth.config("c3")
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    rng = np.random.default_rng(0x2E9)
    pick = np.sort(rng.choice(len(rc), SHAPES, replace=False))
    rc, rm, sel = rc[pick], rm[pick], np.ascontiguousarray(sel[pick])
    R = np.full(SHAPES, REPLICAS, np.uint32)
    line = {"metric": "place_replicas_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
            "workload": f"c3 cluster ({len(ac)} nodes, {len(bn)} bound pods), {SHAPES} seeded c3 pod shapes x "
                        f"R = {REPLICAS}"}
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        for policy, name in ((ks.KS_SCORE_LEFTOVER, "leftover"), (ks.KS_SCORE_LEAST_ALLOCATED, "least_allocated")):
            res = {}
            for want, key in ((True, "with_copies"), (False, "capacity_only")):
                ms = []
                for s in range(args.warmup + args.steps):
                    t = time.perf_counter()
                    out = snap.place_replicas(rc, rm, sel, R, policy, want_nodes=want)
                    if s >= args.warmup:
                        ms.append((time.perf_counter() - t) * 1e3)
                    if want:
                        plan = out
                res[key] = spread(ms)
            rows, node, score, off = plan
            one_ms = []  # the same shapes as the gang calls, one shape per plan call
            for t in range(GANG_SHAPES):
                ms = []
                for s in range(args.warmup + args.steps):
                    t0 = time.perf_counter()
                    one = snap.place_replicas(rc[t:t + 1], rm[t:t + 1], sel[t:t + 1], R[t:t + 1], policy)
                    if s >= args.warmup:
                        ms.append((time.perf_counter() - t0) * 1e3)
                a, b = int(off[t]), int(off[t + 1])
                assert np.array_equal(one[1], node[a:b]) and np.array_equal(one[2], score[a:b]), f"{name} shape {t}"
                one_ms.append(statistics.median(ms))
            res["one_shape_with_copies"] = {"shapes": GANG_SHAPES, "call_ms": spread(one_ms)}
            gang_ms = []
            for t in range(GANG_SHAPES):
                with ks.Snapshot(0) as g:
                    g.set_nodes(ac, am, lab)
                    g.set_bound(bn, bc, bm)
                    t0 = time.perf_counter()
                    gi, gs, _, _ = g.gang_bind(np.repeat(rc[t:t + 1], REPLICAS), np.repeat(rm[t:t + 1], REPLICAS),
                                               np.repeat(sel[t:t + 1], REPLICAS, axis=0),
                                               np.arange(REPLICAS + 1, dtype=np.uint64), np.zeros(REPLICAS, np.uint32),
                                               policy)
                    gang_ms.append((time.perf_counter() - t0) * 1e3)
                a, b = int(off[t]), int(off[t + 1])
                assert np.array_equal(gi, node[a:b]) and np.array_equal(gs, score[a:b]), f"{name} shape {t}: gang differs"
            res["gang_singletons"] = {"shapes": GANG_SHAPES, "call_ms": spread(gang_ms), "checked_equal": True}
            res["gang_over_one_shape_plan"] = statistics.median(gang_ms) / statistics.median(one_ms)
            res["gang_over_plan_per_shape"] = statistics.median(gang_ms) / (res["with_copies"]["median"] / SHAPES)
            res["placed"] = int(rows["placed"].sum())
            res["shapes_below_R"] = int((rows["capacity"] < REPLICAS).sum())
            line[name] = res
    line["note"] = ("host-space specs and outputs, wall clock per call (the call returns after its D2H copy); "
                    "gang_over_one_shape_plan = one gang call over a plan call for that one shape (the method alone); "
                    "gang_over_plan_per_shape = one gang call over 1/256 of the batched plan call (method and batching)")
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
