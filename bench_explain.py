#!/usr/bin/env python
"""bench_explain.py — rate of ks_explain (per-pod rejection counts, k_explain_counts) on one H100.

For each one-GPU workload of bench.py (c3 = 1M pods x 50k nodes, c2 = 100k x 10k, same seeds): one ks_select pass finds
the NoNodeFound pods, then ks_explain counts why for exactly those pods, pods and counts held on the device.  For c2 the
whole batch (1e9 cells) is explained as well.  Each figure is the median (and min / max) of --steps CUDA-event timed
calls after --warmup untimed ones, with the per-cell select kernel (ks_select --path direct, bindings and counts only)
timed on the same pods next to it.  The counts are checked against the select pass:
not_enough_resources + node_selector_mismatch + feasible_cnt == N for every explained pod.
Prints one JSON line; writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def spread(xs):
    xs = sorted(xs)
    return {"min": xs[0], "median": statistics.median(xs), "max": xs[-1]}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:
        return {"error": str(e)[:200]}


def measure(ks, torch, snap, d_rc, d_rm, d_sel, rows, cnt, N, stream, steps, warmup):
    n = int(len(rows))
    if n == 0:
        return {"pods": 0, "cells": 0}
    dev = d_rc.device
    ix = torch.from_numpy(np.asarray(rows, np.int64)).to(dev)
    s_rc, s_rm, s_sel = d_rc[ix].contiguous(), d_rm[ix].contiguous(), d_sel[ix].contiguous()
    out = torch.empty((n, 4), dtype=torch.int32, device=dev)
    idx = torch.empty(n, dtype=torch.int32, device=dev)
    score = torch.empty(n, dtype=torch.int64, device=dev)
    dcnt = torch.empty(n, dtype=torch.int32, device=dev)

    def explain():
        snap.explain_raw(n, s_rc, s_rm, s_sel, ks.KS_MEM_DEVICE, out, ks.KS_MEM_DEVICE, stream=stream.cuda_stream)

    def direct():
        snap.select_raw(n, s_rc, s_rm, s_sel, ks.KS_MEM_DEVICE, idx, score, dcnt, ks.KS_MEM_DEVICE,
                        flags=ks.KS_SELECT_FORCE_DIRECT, stream=stream.cuda_stream)

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

    ms = timed(explain)
    why = out.cpu().numpy().view(np.uint32).astype(np.int64)
    assert np.array_equal(why[:, 2] + why[:, 3] + cnt[rows].astype(np.int64), np.full(n, N)), "explain invariant"
    assert np.all(np.maximum(why[:, 0], why[:, 1]) <= why[:, 2]) and np.all(why[:, 2] <= why[:, 0] + why[:, 1])
    d_ms = timed(direct)
    med, d_med = statistics.median(ms), statistics.median(d_ms)
    return {"pods": n, "cells": n * N, "ms": spread(ms), "cells_per_s": n * N / (med * 1e-3),
            "direct_select_ms": spread(d_ms), "direct_select_cells_per_s": n * N / (d_med * 1e-3)}


def workload(ks, torch, name, steps, warmup):
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
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        snap.select_raw(P, d_rc, d_rm, d_sel, ks.KS_MEM_DEVICE, idx, score, cnt, ks.KS_MEM_DEVICE, stream=stream.cuda_stream)
        stream.synchronize()
        h_idx, h_cnt = idx.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)
        assert np.array_equal(h_idx < 0, h_cnt == 0)
        res = {"workload": f"{name}: {P} pods x {N} nodes",
               "no_node_found": measure(ks, torch, snap, d_rc, d_rm, d_sel, np.nonzero(h_idx < 0)[0], h_cnt, N, stream,
                                        steps, warmup)}
        if name == "c2":
            res["all_pods"] = measure(ks, torch, snap, d_rc, d_rm, d_sel, np.arange(P), h_cnt, N, stream, steps, warmup)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workload", default="all", choices=["all", "c2", "c3"])
    args = ap.parse_args()
    import torch
    import ksched_pkg
    ks = ksched_pkg.load()
    if not torch.cuda.is_available() or ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_explain has no CPU fallback"}), flush=True)
        return 2
    line = {"metric": "explain_cells_per_sec", "unit": "cells/s", "gpu": gpu_info(), "steps": args.steps,
            "warmup": args.warmup,
            "note": "pods and counts on the device, CUDA events per call, no L2 flush (the node table is a few MB); "
                    "direct_select = ks_select --path direct on the same pods"}
    for name in (("c3", "c2") if args.workload == "all" else (args.workload,)):
        line[name] = workload(ks, torch, name, args.steps, args.warmup)
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
