#!/usr/bin/env python
"""bench_fit_drain.py — cost of ks_fit_drain_check (drain simulation under the full filter: k_node_rules_setup, then
k_fit_drain_scan + k_fit_drain_commit per round) on one H100, beside ks_drain_check.

Workload: bench_drain.py's c3 sweep - the c3 node table (50k nodes) and its 500k bound pods, every node a candidate with
its bound pods, each carrying a seeded c3 pending pod's selector - plus bench_fit_preempt.py's GPU pool: 8
nvidia.com/gpu on every 20th node, tainted (bench_node_bind.py's rules over 64 workloads), with two 4-GPU pods bound on
every pool node in workloads that tolerate the pool (every 8th); every other bound pod is in workload (index % 64).
pods allocatable 110 on every node.  Resources: the pod count and nvidia.com/gpu.  Host-space pods and outputs, policy
LEFTOVER.  Each figure is the median (and min / max) of --steps calls after --warmup untimed ones, each timed by CUDA
events recorded around the call, which returns after its stream synchronise:
  - fit_drain_ms: the whole call with out_refused;
  - fit_drain_no_refused_ms: the same without out_refused (the cost of the refusal words is the difference);
  - drain_ms and fit_drain_d1_ms: ks_drain_check and ks_fit_drain_check with rules and resources NULL (identity D1: the
    same outputs, checked in the run), alternated call by call;
  - drainable_lost: the candidates ks_drain_check calls drainable that this call does not.
The GPU name, power limit and max SM clock are read in the same run.  Prints one JSON line; writes nothing."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_explain import gpu_info, spread  # noqa: E402
from bench_node_bind import rules_for  # noqa: E402

WORKLOADS = 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import numpy as np
    import torch
    import ksched_pkg
    from drain_oracle import bound_candidates
    ks = ksched_pkg.load()
    if not torch.cuda.is_available() or ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_fit_drain_check has no CPU fallback"}), flush=True)
        return 2
    from importlib import import_module
    snapshot_mod = import_module(ks.Snapshot.__module__)
    cl = ks.synth.config("c3")
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    N = len(ac)
    rng = np.random.default_rng(0xB2000003)
    pool = np.nonzero(np.arange(N) % 20 == 19)[0].astype(np.int32)
    B0 = len(bn)
    bn = np.concatenate([bn, np.repeat(pool, 2)])  # two 4-GPU pods on every pool node
    bc = np.concatenate([bc, np.full(2 * len(pool), 1000, np.int64)])
    bm = np.concatenate([bm, np.full(2 * len(pool), 1 << 30, np.int64)])
    bgpu = np.concatenate([np.zeros(B0, np.int64), np.full(2 * len(pool), 4, np.int64)])
    bgroup = np.concatenate([(np.arange(B0) % WORKLOADS), 8 * (np.arange(2 * len(pool)) % 8)]).astype(np.int32)
    order, node, off = bound_candidates(bn, N)
    psel = np.ascontiguousarray(sel[rng.integers(0, len(rc), len(order))])
    psel[B0 <= order] = 0  # the GPU pods carry no selector
    prc, prm, pgroup = bc[order], bm[order], bgroup[order]
    node_free = np.stack([110 - np.bincount(bn, minlength=N), np.where(np.arange(N) % 20 == 19, 8, 0)
                          - np.bincount(bn, weights=bgpu, minlength=N).astype(np.int64)]).astype(np.int64)
    pod_req = np.ascontiguousarray(np.stack([np.ones(len(order), np.int64), bgpu[order]], axis=1))
    rules = rules_for(np, snapshot_mod, N, WORKLOADS)
    none = np.full(len(order), -1, np.int32)
    size = np.diff(off).astype(np.int64)
    stream = torch.cuda.current_stream()
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        fc, fm = snap.free()

        def fit(refused):
            return lambda: snap.fit_drain_check(prc, prm, psel, pgroup, WORKLOADS, node, off, rules=rules,
                                                node_free=node_free, pod_req=pod_req, want_refused=refused)

        def d1():
            return snap.fit_drain_check(prc, prm, psel, none, 0, node, off, want_refused=False)

        def drain():
            return snap.drain_check(prc, prm, psel, node, off)

        def timed(fns):
            """CUDA-event times of each function, alternated call by call; and the last results"""
            out = [None] * len(fns)
            for _ in range(max(args.warmup, 1)):
                for i, fn in enumerate(fns):
                    out[i] = fn()
            ms = [[] for _ in fns]
            for _ in range(args.steps):
                for i, fn in enumerate(fns):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(stream)
                    out[i] = fn()
                    b.record(stream)
                    b.synchronize()
                    ms[i].append(a.elapsed_time(b))
            return ms, out

        (f_ms, n_ms), (full, bare) = timed([fit(True), fit(False)])
        assert all(np.array_equal(a, b) for a, b in zip(full[:3], bare[:3])), "out_refused changed the placement"
        (p_ms, q_ms), (p_out, q_out) = timed([drain, d1])
        assert all(np.array_equal(a, b) for a, b in zip(p_out, q_out[:3])), "D1: outputs differ"
        assert all(np.array_equal(a, b) for a, b in zip(snap.free(), (fc, fm))), "free[] changed"
    placed, refused = full[0], full[3]
    ok, ok_drain = placed == size, p_out[0] == size
    stopped = ~ok
    line = {"metric": "fit_drain_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
            "workload": f"c3 nodes ({N}), {len(bn)} bound pods ({2 * len(pool)} 4-GPU pods on {len(pool)} tainted "
                        f"8-GPU nodes), pods allocatable 110; every node a candidate with its bound pods "
                        f"({len(order)} pods, {WORKLOADS} workloads), resources pods and nvidia.com/gpu, LEFTOVER",
            "fit_drain_ms": spread(f_ms), "fit_drain_no_refused_ms": spread(n_ms),
            "refused_cost_ms": statistics.median(f_ms) - statistics.median(n_ms),
            "drain_ms": spread(p_ms), "fit_drain_d1_ms": spread(q_ms),
            "d1_vs_drain": statistics.median(q_ms) / statistics.median(p_ms),
            "fit_vs_drain": statistics.median(f_ms) / statistics.median(p_ms),
            "candidates": N, "drainable": int(ok.sum()), "drainable_ks_drain_check": int(ok_drain.sum()),
            "drainable_lost": int((ok_drain & ~ok).sum()),
            "stopped_by_word": [int((stopped & (refused[:, w] > 0)).sum()) for w in range(4)],
            "note": "host-space pods and outputs; CUDA events around each call (the call ends in a stream synchronise), "
                    "no L2 flush; drain_ms and fit_drain_d1_ms alternated call by call, as fit_drain_ms and "
                    "fit_drain_no_refused_ms"}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
