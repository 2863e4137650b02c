#!/usr/bin/env python
"""bench_topk.py — rate of ks_select_topk (the k best feasible nodes per pod, k_select_topk) on one H100.

For the one-GPU workloads of bench.py (c2 = 100k pods x 10k nodes, c3 = 1M x 50k, same seeds), the whole batch is
ranked with k in {1, 8, 32} under both score policies, pods and outputs held on the device.  Each figure is the median
(and min / max) of --steps CUDA-event timed calls after --warmup untimed ones, with the per-cell select kernel
(ks_select --path direct, bindings and counts, no mask) timed on the same pods and policy next to it.  Entry 0 of every
row and the feasible counts are checked against that select pass.  The GPU name, power limit and max SM clock are read
in the same run.  Prints one JSON line; writes nothing."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_explain import gpu_info, spread  # noqa: E402


def workload(ks, torch, name, ks_list, steps, warmup):
    import numpy as np
    P, N = ks.synth.SHAPES[name]
    cl = ks.synth.make(P, N, ks.synth.SEEDS[name])
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream()
    d_rc, d_rm = torch.from_numpy(rc).to(dev), torch.from_numpy(rm).to(dev)
    d_sel = torch.from_numpy(np.ascontiguousarray(sel).view(np.int64)).to(dev)
    idx = torch.empty(P, dtype=torch.int32, device=dev)
    score = torch.empty(P, dtype=torch.int64, device=dev)
    cnt = torch.empty(P, dtype=torch.int32, device=dev)
    k_max = max(ks_list)
    t_idx = torch.empty(P * k_max, dtype=torch.int32, device=dev)
    t_score = torch.empty(P * k_max, dtype=torch.int64, device=dev)
    t_cnt = torch.empty(P, dtype=torch.int32, device=dev)

    def timed(fn):
        for _ in range(max(warmup, 1)):
            fn()
        stream.synchronize()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for a, b in ev:
            a.record(stream)
            fn()
            b.record(stream)
        stream.synchronize()
        return [a.elapsed_time(b) for a, b in ev]

    res = {"workload": f"{name}: {P} pods x {N} nodes", "cells": P * N}
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        for policy, pname in ((ks.KS_SCORE_LEFTOVER, "leftover"), (ks.KS_SCORE_LEAST_ALLOCATED, "least_allocated")):
            def direct():
                snap.select_raw(P, d_rc, d_rm, d_sel, ks.KS_MEM_DEVICE, idx, score, cnt, ks.KS_MEM_DEVICE, policy=policy,
                                flags=ks.KS_SELECT_FORCE_DIRECT, stream=stream.cuda_stream)

            d_ms = timed(direct)
            out = {"direct_select_ms": spread(d_ms)}
            for k in ks_list:
                def topk():
                    snap.select_topk_raw(P, d_rc, d_rm, d_sel, ks.KS_MEM_DEVICE, k, t_idx, t_score, t_cnt,
                                         ks.KS_MEM_DEVICE, policy=policy, stream=stream.cuda_stream)

                ms = timed(topk)
                rows_i = t_idx[:P * k].view(P, k)
                rows_s = t_score[:P * k].view(P, k)
                assert torch.equal(rows_i[:, 0], idx) and torch.equal(rows_s[:, 0], score), f"entry 0 ({pname}, k={k})"
                assert torch.equal(t_cnt, cnt), f"feasible count ({pname}, k={k})"
                med = statistics.median(ms)
                out[f"k{k}"] = {"ms": spread(ms), "cells_per_s": P * N / (med * 1e-3),
                                "vs_direct_select": med / statistics.median(d_ms)}
            res[pname] = out
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workload", default="all", choices=["all", "c2", "c3"])
    args = ap.parse_args()
    import torch
    import ksched_pkg
    ks = ksched_pkg.load()
    if not torch.cuda.is_available() or ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_select_topk has no CPU fallback"}), flush=True)
        return 2
    line = {"metric": "topk_cells_per_sec", "unit": "cells/s", "gpu": gpu_info(), "steps": args.steps,
            "warmup": args.warmup,
            "note": "whole batch ranked, pods and outputs on the device, CUDA events per call, no L2 flush; "
                    "direct_select = ks_select --path direct on the same pods and policy"}
    for name in (("c2", "c3") if args.workload == "all" else (args.workload,)):
        line[name] = workload(ks, torch, name, (1, 8, 32), args.steps, args.warmup)
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
