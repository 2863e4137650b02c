#!/usr/bin/env python
"""bench_gang.py — cost of ks_gang_bind (pod groups, all or nothing: k_gang_batch) on one H100.

Workload: the c3 node table of bench.py (50k nodes, seed 0xB2000003, 500k bound pods) and 2 000 groups of 8 to 256 pods
(seeded), taken in order from the c3 pods, every group all or nothing (min_member = its size).  Requests are multiplied
by the factor at which the groups ask for about 1.7x the cluster's free cpu, so a sizeable share rolls back.  Pods and
outputs are host memory, as ks_gang_bind takes them.  Every timed call starts from the same free[] (set_bound, untimed).
  - gang_ms: the whole ks_gang_bind call (one H2D copy, one cooperative launch over every group, one D2H copy);
  - per_group_us: gang_ms over the number of groups;
  - host_loop_ms: what a controller does without it: ks_stream_bind per group, then for a group that falls short one
    ks_snapshot_apply_bind with the negated request per placed pod.  Its bindings and free[] must equal ks_gang_bind's.
Each figure is the median (and min / max) of --steps calls after --warmup untimed ones (the host loop runs at most 3
timed steps).  The GPU name, power limit and max SM clock are read in the same run.  Prints one JSON line; writes
nothing."""
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

GROUPS, SIZE_MIN, SIZE_MAX = 2000, 8, 256
DEMAND = 1.7  # requested cpu over free cpu


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import numpy as np
    import ksched_pkg
    ks = ksched_pkg.load()
    if ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_gang_bind has no CPU fallback"}), flush=True)
        return 2
    cl = ks.synth.config("c3")
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    N = len(ac)
    rng = np.random.default_rng(0xB2000003)
    sizes = rng.integers(SIZE_MIN, SIZE_MAX + 1, GROUPS)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    P = int(off[-1])
    rc, rm, sel = rc[:P].copy(), rm[:P].copy(), np.ascontiguousarray(sel[:P])
    mm = sizes.astype(np.uint32)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        fc0, _ = snap.free()
        factor = max(1, int(round(DEMAND * float(np.maximum(fc0, 0).sum()) / float(rc.sum()))))
        rc, rm = rc * factor, rm * factor

        def gang():
            return snap.gang_bind(rc, rm, sel, off, mm)

        def host_loop():
            idx = np.full(P, -1, np.int32)
            for g in range(GROUPS):
                a, b = int(off[g]), int(off[g + 1])
                i, _, _ = snap.stream_bind(rc[a:b], rm[a:b], sel[a:b])
                if (i >= 0).sum() >= mm[g]:
                    idx[a:b] = i
                    continue
                for k in np.nonzero(i >= 0)[0]:  # undo, pod by pod
                    snap.apply_bind(int(i[k]), -int(rc[a + k]), -int(rm[a + k]))
            return idx

        def timed(fn, steps):
            ms, out = [], None
            for s in range(max(args.warmup, 1) + steps):
                snap.set_bound(bn, bc, bm)
                t = time.perf_counter()
                out = fn()
                if s >= max(args.warmup, 1):
                    ms.append((time.perf_counter() - t) * 1e3)
            return ms, out, snap.free()

        g_ms, (idx, score, placed, rounds), g_free = timed(gang, args.steps)
        h_ms, h_idx, h_free = timed(host_loop, min(args.steps, 3))
    assert np.array_equal(idx, h_idx), "ks_gang_bind and the per-group host loop disagree on the bindings"
    assert all(np.array_equal(a, b) for a, b in zip(g_free, h_free)), "ks_gang_bind and the host loop disagree on free[]"
    committed = placed >= mm
    line = {"metric": "gang_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
            "workload": f"c3 nodes ({N}), {len(bn)} bound pods, {GROUPS} groups of {SIZE_MIN}-{SIZE_MAX} pods "
                        f"({P} pods), min_member = size, requests x{factor}",
            "gang_ms": spread(g_ms), "per_group_us": statistics.median(g_ms) * 1e3 / GROUPS,
            "host_loop_ms": spread(h_ms), "host_loop_vs_gang": statistics.median(h_ms) / statistics.median(g_ms),
            "rounds": {"total": int(rounds.sum()), "mean": float(rounds.mean()), "max": int(rounds.max())},
            "groups_committed": int(committed.sum()), "groups_rolled_back": int((~committed).sum()),
            "pods_bound": int((idx >= 0).sum()),
            "note": "host-space pods and outputs, wall clock per call (the call returns after its D2H copy); host loop = "
                    "ks_stream_bind per group + ks_snapshot_apply_bind(-request) per placed pod of a rolled-back group"}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
