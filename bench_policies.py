#!/usr/bin/env python
"""bench_policies.py — the score policies of tests/policy_oracle.py on one H100: --policy 3 = KS_SCORE_MOST_ALLOCATED
(bin-packing), next to LEFTOVER and LEAST_ALLOCATED; --policy 4 = KS_SCORE_LEAST_BALANCED (upstream's default resource
scoring), next to LEAST_ALLOCATED.

For the one-GPU workloads of bench.py (c2 = 100k pods x 10k nodes, c3 = 1M x 50k, same seeds), pods and outputs on the
device, no mask:
  * the ks_select step under the policy on both kernel paths (the bit-parallel k_most_alloc / k_least_balanced behind
    k_mask_rows, and the per-cell kernel) and under AUTO, and the other policies under AUTO and on the per-cell kernel;
  * ks_select_topk (k = 8) under the policy on the same pods;
  * on the c2 cluster under the policy: ks_stream_bind of 1024 pods, ks_drain_check with the bound pods of 512 nodes as
    candidates, and ks_place_replicas (host-staged calls, host clock around the synchronous call; the snapshot's free[]
    is reset before each ks_stream_bind).  The replica section follows the algorithm: policy 3 fills nodes whole in one
    threshold search, timed on 256 pod specs x 1000 copies; policy 4 places one copy at a time, timed on one pod spec
    at 1, 1000 and 65 536 copies, with the cost per copy.
Each figure is the median (and min / max) of --steps timed calls after --warmup untimed ones.  Before timing, the
bindings of 256 seeded pods of each workload are checked against the CPU restatement of tests/policy_oracle.py,
and top-k entry 0 against the select.  The GPU name, power limit and max SM clock are read in the same run.  Prints one
JSON line; writes nothing."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_explain import gpu_info, spread  # noqa: E402


def timed_events(torch, stream, fn, steps, warmup):
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


def timed_host(fn, steps, warmup, before=None):
    ms = []
    for i in range(max(warmup, 1) + steps):
        if before:
            before()
        t0 = time.perf_counter()
        fn()
        if i >= max(warmup, 1):
            ms.append((time.perf_counter() - t0) * 1e3)
    return ms


NAME = {3: "most_allocated", 4: "least_balanced"}
OTHERS = {3: ((0, "leftover"), (1, "least_allocated")), 4: ((1, "least_allocated"),)}


def workload(ks, torch, o, name, steps, warmup, MA, others):
    import numpy as np
    from drain_oracle import bound_candidates
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
    res = {"workload": f"{name}: {P} pods x {N} nodes", "cells": P * N, "select_ms": {}}
    fc, fm = o.free_reduce(ac, am, bn, bc, bm)
    sample = np.random.default_rng(0x3A).choice(P, 256, replace=False)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        runs = [(MA, NAME[MA], f, fname) for f, fname in ((ks.KS_SELECT_FORCE_BITPAR, "bitpar"),
                                                         (ks.KS_SELECT_AUTO, "auto"), (ks.KS_SELECT_FORCE_DIRECT, "direct"))]
        for pol, pname in OTHERS[MA]:
            runs += [(pol, pname, ks.KS_SELECT_AUTO, "auto"), (pol, pname, ks.KS_SELECT_FORCE_DIRECT, "direct")]
        for pol, pname, flags, fname in runs:
            if pol != MA and not others:
                continue

            def select():
                snap.select_raw(P, d_rc, d_rm, d_sel, ks.KS_MEM_DEVICE, idx, score, cnt, ks.KS_MEM_DEVICE, policy=pol,
                                flags=flags, stream=stream.cuda_stream)

            ms = timed_events(torch, stream, select, steps, warmup)
            res["select_ms"][f"{pname}/{fname}"] = dict(spread(ms), path=snap.last_path())
            if pol == MA:
                w = o.run_packed(fc, fm, ac, am, lab, rc[sample], rm[sample], sel[sample], MA, want_mask=False)
                got_i, got_s = idx.cpu().numpy()[sample], score.cpu().numpy()[sample]
                assert np.array_equal(got_i, w[0]) and np.array_equal(got_s, w[1]), f"{name}: select vs restatement"
                if fname == "bitpar":
                    s_idx, s_score = idx.clone(), score.clone()
                else:  # every path binds every pod as the bit-parallel one did
                    assert torch.equal(idx, s_idx) and torch.equal(score, s_score), f"{name}: {fname} vs bitpar"
        k = 8
        t_idx = torch.empty(P * k, dtype=torch.int32, device=dev)
        t_score = torch.empty(P * k, dtype=torch.int64, device=dev)
        t_cnt = torch.empty(P, dtype=torch.int32, device=dev)

        def topk():
            snap.select_topk_raw(P, d_rc, d_rm, d_sel, ks.KS_MEM_DEVICE, k, t_idx, t_score, t_cnt, ks.KS_MEM_DEVICE,
                                 policy=MA, stream=stream.cuda_stream)

        res["topk8_ms"] = spread(timed_events(torch, stream, topk, steps, warmup))
        assert torch.equal(t_idx.view(P, k)[:, 0], s_idx) and torch.equal(t_score.view(P, k)[:, 0], s_score), "top-k entry 0"
        if name == "c2":
            sp = slice(0, 1024)

            def reset():
                snap.set_bound(bn, bc, bm)

            res["stream_bind_1024_ms"] = spread(timed_host(lambda: snap.stream_bind(rc[sp], rm[sp], sel[sp], MA), steps,
                                                           warmup, reset))
            reset()
            got = snap.stream_bind(rc[sp], rm[sp], sel[sp], MA)
            want = o.stream_bind_packed(fc.copy(), fm.copy(), ac, am, lab, rc[sp], rm[sp], sel[sp], MA)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), "stream_bind vs restatement"
            reset()
            order, node, off = bound_candidates(bn, N)
            D = 512
            po = order[:int(off[D])]
            args = (bc[po], bm[po], np.ascontiguousarray(sel[np.arange(len(po)) % P]), node[:D], off[:D + 1])
            res["drain_512_ms"] = spread(timed_host(lambda: snap.drain_check(*args, MA), steps, warmup))
            if MA == 3:
                T, R = 256, np.full(256, 1000, np.uint32)
                rargs = (rc[:T] + 1, rm[:T] + 1, np.ascontiguousarray(sel[:T]), R)
                res["replicas_256x1000_ms"] = spread(timed_host(lambda: snap.place_replicas(*rargs, MA), steps, warmup))
                return res
            from policy_oracle import heap_packed
            t = int(np.nonzero((rc > 0) & (sel == 0).all(axis=1))[0][0])  # a spec with a request and no selector
            for R in (1, 1000, 65536):
                rargs = (rc[t:t + 1], rm[t:t + 1], np.ascontiguousarray(sel[t:t + 1]), np.array([R], np.uint32))
                ms = spread(timed_host(lambda: snap.place_replicas(*rargs, MA), steps, warmup))
                got = snap.place_replicas(*rargs, MA)
                placed = int(got[0]["placed"][0])
                if R <= 1000:  # the heap restatement at 65 536 copies takes minutes in Python
                    want = heap_packed(fc, fm, ac, am, lab, *rargs)
                    assert all(np.array_equal(a, b) for a, b in zip(got[1:3], want[1:3])), "replicas vs restatement"
                res[f"replicas_1x{R}_ms"] = dict(ms, placed=placed, us_per_copy=round(ms["median"] * 1e3 / max(placed, 1), 3))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workload", default="all", choices=["all", "c2", "c3"])
    ap.add_argument("--policy", type=int, required=True, choices=sorted(NAME))
    ap.add_argument("--policy-only", action="store_true", help="time the policy only, not the others")
    args = ap.parse_args()
    import torch
    import ksched_pkg
    ks = ksched_pkg.load()
    if not torch.cuda.is_available() or ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: the scheduling kernels have no CPU fallback"}), flush=True)
        return 2
    from oracle import orc
    from policy_oracle import Oracle
    line = {"metric": f"{NAME[args.policy]}_step_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps,
            "warmup": args.warmup,
            "note": "ks_select: pods and outputs on the device, no mask, CUDA events per call; host-staged calls: host "
                    "clock around the synchronous call"}
    for name in (("c2", "c3") if args.workload == "all" else (args.workload,)):
        line[name] = workload(ks, torch, Oracle(orc), name, args.steps, args.warmup, args.policy, not args.policy_only)
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
