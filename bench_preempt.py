#!/usr/bin/env python
"""bench_preempt.py — cost of ks_preempt (priority preemption: the victim index, k_preempt_scan, k_preempt_emit) on one
H100.

Workload: the c3 cluster of bench.py (50k nodes, seed 0xB2000003, 500k bound pods) with bound-pod priorities drawn
(seeded) from {0, 100, 1000, 10000}, plus one skewed node that holds 5 000 more small bound pods of those priorities.
The pending batch is the first 10 000 c3 pods at priority 1000, their requests multiplied by the smallest factor at which
at least 90% of the (pod, node) cells fail on resources.  Pods and outputs are on the device; the bound list is host
memory, as ks_preempt takes it.  Each figure is the median (and min / max) of --steps CUDA-event timed calls after
--warmup untimed ones:
  - preempt_ms: the whole call (upload of the bound list, victim index, scan, emit);
  - index_build_ms: a call with one pod, i.e. the upload and the victim index plus a one-pod scan;
  - explain_ms: ks_explain on the same pods, for scale.
It also reports how many pods got a plan and how many cells reached the exact walk (counted with torch from the
definition, outside the timed calls).  The GPU name, power limit and max SM clock are read in the same run.  Prints one
JSON line; writes nothing."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_explain import gpu_info, spread  # noqa: E402

PODS, SKEW = 10_000, 5_000
LEVELS = (0, 100, 1000, 10000)
POD_PRIORITY = 1000


def walk_cells(torch, fc, fm, lab, rc, rm, sel, bn, bc, bm, bp, pi):
    """Cells that reach the exact walk: fail on resources, selector matches, a lower-priority pod on the node, and the
    room check passes (one priority for the whole batch, so the lower set's sums are one vector)."""
    dev = torch.device("cuda", 0)
    N = fc.shape[0]
    low = bp < pi
    sum_c = torch.zeros(N, dtype=torch.int64, device=dev).index_add_(0, bn[low].long(), bc[low])
    sum_m = torch.zeros(N, dtype=torch.int64, device=dev).index_add_(0, bn[low].long(), bm[low])
    has_low = torch.zeros(N, dtype=torch.bool, device=dev)
    has_low[bn[low].long()] = True
    total = 0
    for a in range(0, rc.shape[0], 500):
        c, m, s = rc[a:a + 500, None], rm[a:a + 500, None], sel[a:a + 500]
        fit = (c <= fc) & (m <= fm)
        match = torch.ones_like(fit)
        for w in range(lab.shape[1]):
            match &= (s[:, w:w + 1] & ~lab[:, w][None, :]) == 0
        room = (c <= fc + sum_c) & (m <= fm + sum_m)
        total += int((~fit & match & has_low & room).sum())
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-victims", type=int, default=16)
    args = ap.parse_args()
    import numpy as np
    import torch
    import ksched_pkg
    ks = ksched_pkg.load()
    if not torch.cuda.is_available() or ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_preempt has no CPU fallback"}), flush=True)
        return 2
    cl = ks.synth.config("c3")
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    N = len(ac)
    rng = np.random.default_rng(0xB2000003)
    bn = np.concatenate([bn, np.zeros(SKEW, np.int32)])  # the skewed node: node 0
    bc = np.concatenate([bc, np.full(SKEW, 1, np.int64)])
    bm = np.concatenate([bm, np.full(SKEW, 1 << 20, np.int64)])
    bp = rng.choice(np.array(LEVELS, np.int32), len(bn))
    rc, rm, sel = rc[:PODS].copy(), rm[:PODS].copy(), np.ascontiguousarray(sel[:PODS])
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream()
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        fc, fm = snap.free()
        d_fc, d_fm = torch.from_numpy(fc).to(dev), torch.from_numpy(fm).to(dev)
        d_lab = torch.from_numpy(np.ascontiguousarray(lab).view(np.int64)).to(dev)
        factor = 1
        for factor in range(1, 65):  # raise the requests until most nodes fail on resources
            c = torch.from_numpy(rc[:200] * factor).to(dev)[:, None]
            m = torch.from_numpy(rm[:200] * factor).to(dev)[:, None]
            if float((~((c <= d_fc) & (m <= d_fm))).float().mean()) >= 0.9:
                break
        rc, rm = rc * factor, rm * factor
        pp = np.full(PODS, POD_PRIORITY, np.int32)
        d_rc, d_rm = torch.from_numpy(rc).to(dev), torch.from_numpy(rm).to(dev)
        d_sel = torch.from_numpy(sel.view(np.int64)).to(dev)
        d_pp = torch.from_numpy(pp).to(dev)
        out = torch.empty((PODS, 4), dtype=torch.int64, device=dev)
        vic = torch.empty((PODS, args.max_victims), dtype=torch.int32, device=dev)
        why = torch.empty((PODS, 4), dtype=torch.int32, device=dev)
        bound = (bn, bc, bm, bp)

        def timed(fn):
            for _ in range(max(args.warmup, 1)):
                fn()
            stream.synchronize()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
            for a, b in ev:
                a.record(stream)
                fn()
                b.record(stream)
            stream.synchronize()
            return [a.elapsed_time(b) for a, b in ev]

        def preempt(n):
            return lambda: snap.preempt_raw(n, d_rc, d_rm, d_sel, ks.KS_MEM_DEVICE, d_pp, bound, args.max_victims, out,
                                            vic, ks.KS_MEM_DEVICE, stream=stream.cuda_stream)

        def explain():
            snap.explain_raw(PODS, d_rc, d_rm, d_sel, ks.KS_MEM_DEVICE, why, ks.KS_MEM_DEVICE, stream=stream.cuda_stream)

        p_ms = timed(preempt(PODS))
        rows = out.cpu().numpy().view(ks.capi.PREEMPTION_DTYPE).reshape(PODS)
        i_ms = timed(preempt(1))
        e_ms = timed(explain)
        # the same pods through the host-space entry point: the rows must not change
        h_rows, _ = snap.preempt(rc, rm, sel, pp, bn, bc, bm, bp, args.max_victims)
        assert np.array_equal(h_rows, rows), "device- and host-space calls disagree"
        walked = walk_cells(torch, d_fc, d_fm, d_lab, d_rc, d_rm, d_sel, torch.from_numpy(bn).to(dev),
                            torch.from_numpy(bc).to(dev), torch.from_numpy(bm).to(dev), torch.from_numpy(bp).to(dev),
                            POD_PRIORITY)
    line = {"metric": "preempt_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
            "workload": f"c3 nodes ({N}), {len(bn)} bound pods ({SKEW} on node 0), {PODS} pods at priority "
                        f"{POD_PRIORITY}, requests x{factor}, max_victims {args.max_victims}",
            "preempt_ms": spread(p_ms), "index_build_ms": spread(i_ms), "explain_ms": spread(e_ms),
            "preempt_vs_explain": statistics.median(p_ms) / statistics.median(e_ms),
            "pods_with_plan": int((rows["node_idx"] >= 0).sum()),
            "pods_feasible": int((rows["feasible_cnt"] > 0).sum()),
            "cells": PODS * N, "cells_walked": walked,
            "note": "pods, priorities and outputs on the device, bound list in host memory; CUDA events per call, no L2 "
                    "flush; index_build_ms is a one-pod call (bound-list upload + victim index + one-pod scan)"}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
