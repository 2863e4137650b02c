#!/usr/bin/env python
"""bench_drain.py — cost of ks_drain_check (drain simulation: k_drain_scan + k_drain_commit per round) on one H100.

Workload: the c3 node table of bench.py (50k nodes, seed 0xB2000003) and its 500k bound pods.  Every node is a candidate
and its pods are its bound pods; bound pod i carries c3 pending pod j's selector, j drawn with a fixed seed, so the
selector path runs.  This is the sweep a scale-down or consolidation controller would like to run every loop: one
candidate per node.  Pods and outputs are host memory, as ks_drain_check takes them.
  - drain_ms: the whole ks_drain_check call (one H2D copy, two kernels per round, one D2H copy), median / min / max of
    --steps calls after --warmup untimed ones;
  - cells_per_s: sum over rounds of (pods evaluated x N) over the median call time;
  - us_per_candidate: the median call time over the number of candidates;
  - drainable: candidates whose every pod found a destination; rounds: the largest candidate's pod count.
  - cpu: the restatement (tests/drain_oracle.py, the oracle's per-pod argmax) on a seeded sample of candidates, on the
    usable host cores, extrapolated to every candidate; kind = "port" as bench.py's CPU figures.
The GPU name, power limit and max SM clock are read in the same run.  Prints one JSON line; writes nothing."""
import argparse
import json
import os
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_explain import gpu_info, spread  # noqa: E402

CPU_SAMPLE = 64  # candidates the CPU restatement runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import numpy as np
    import ksched_pkg
    from drain_oracle import bound_candidates, drain_packed
    from oracle import orc
    ks = ksched_pkg.load()
    if ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_drain_check has no CPU fallback"}), flush=True)
        return 2
    cl = ks.synth.config("c3")
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    N = len(ac)
    order, node, off = bound_candidates(bn, N)
    rng = np.random.default_rng(0xB2000003)
    prc, prm = bc[order], bm[order]
    psel = np.ascontiguousarray(sel[rng.integers(0, len(rc), len(order))])
    size = np.diff(off).astype(np.int64)
    rounds = int(size.max())
    evaluated = int(size.sum())  # upper bound: a candidate that stops skips its later rounds
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        fc, fm = snap.free()
        ms = []
        for s in range(args.warmup + args.steps):
            t = time.perf_counter()
            placed, idx, score = snap.drain_check(prc, prm, psel, node, off)
            if s >= args.warmup:
                ms.append((time.perf_counter() - t) * 1e3)
    # pods evaluated: each candidate evaluates its placed pods and the one it stops at
    evaluated = int(np.minimum(placed.astype(np.int64) + 1, size).sum())
    med = statistics.median(ms)
    # CPU restatement on a seeded sample, candidates spread over the host cores
    cores = len(os.sched_getaffinity(0))
    sample = sorted(rng.choice(N, CPU_SAMPLE, replace=False).tolist())
    t = time.perf_counter()
    with ThreadPoolExecutor(cores) as ex:
        parts = list(ex.map(lambda d: drain_packed(orc, fc, fm, ac, am, lab, prc, prm, psel, node, off, 0, False, [d]),
                            sample))
    cpu_s = time.perf_counter() - t
    for d, (pl, ix, sc) in zip(sample, parts):
        a, b = int(off[d]), int(off[d + 1])
        assert pl[d] == placed[d] and np.array_equal(ix[a:b], idx[a:b]) and np.array_equal(sc[a:b], score[a:b]), \
            f"candidate {d}: ks_drain_check and the restatement disagree"
    cpu_ms = cpu_s * 1e3 * N / CPU_SAMPLE
    line = {"metric": "drain_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
            "workload": f"c3 nodes ({N}), {len(bn)} bound pods; every node a candidate with its bound pods "
                        f"({len(order)} pods), LEFTOVER",
            "drain_ms": spread(ms), "cells_per_s": evaluated * N / (med / 1e3), "us_per_candidate": med * 1e3 / N,
            "drainable": int((placed == size).sum()), "candidates": N, "rounds": rounds, "pods_evaluated": evaluated,
            "cpu": {"ms": cpu_ms, "kind": "port", "cores": cores,
                    "sample": f"{CPU_SAMPLE} seeded candidates ({cpu_s:.2f} s), extrapolated to {N}",
                    "note": "restatement: per pod the oracle's argmax over every node (oracle/, multi-threaded)"},
            "gpu_vs_cpu": cpu_ms / med,
            "note": "host-space pods and outputs, wall clock per call (the call returns after its D2H copy)"}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
