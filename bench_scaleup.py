#!/usr/bin/env python
"""bench_scaleup.py — cost of ks_scaleup_estimate (scale-up estimate: k_scaleup_pack + k_scaleup_reasons) on one H100.

Workload: 20 000 c3 pending pods (bench.py's c3 pods, seed 0xB2000003), drawn with a fixed seed, keeping their requests
and selectors.  Templates: the 36 synth node shapes (NODE_CPU_CORES x NODE_MEM_GIB) x 8 seeded label variants (one
value per label key, as synth nodes carry), 288 templates, capacity = allocatable, max_nodes = 1024.  This is the
question cluster-autoscaler's binpacking estimator asks for every node group on every loop.  Pods and outputs are host
memory, as ks_scaleup_estimate takes them; out_node and out_reasons are requested.
  - call_ms: the whole call (one H2D copy, two kernels, one D2H copy, the best-template pick), median / min / max of
    --steps calls after --warmup untimed ones;
  - cells_per_s: templates x pods over the median call time;  us_per_template: the median over the templates;
  - best: the picked template's placed pods and nodes;
  - cpu: the restatement (tests/scaleup_oracle.py) on a seeded sample of templates, one worker process per template on
    the usable host cores (the restatement's loop holds the GIL, so threads would not run in parallel), extrapolated to
    every template; kind = "port" as bench.py's CPU figures.  The sampled rows are checked.
  - --profile DIR: one more call under torch.profiler; the trace goes to DIR/scaleup_trace.json and the per-kernel
    device times into the line ("kernels_us").
The GPU name, power limit and max SM clock are read in the same run.  Prints one JSON line; writes nothing else."""
import argparse
import json
import os
import statistics
import sys
import time
import multiprocessing
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_explain import gpu_info, spread  # noqa: E402

PODS = 20000
VARIANTS = 8
MAX_NODES = 1024
CPU_SAMPLE = 16  # templates the CPU restatement packs


def templates(cl, seed):
    """The 36 node shapes x VARIANTS label variants: (alloc_cpu, alloc_mem, labels[T, W])."""
    import numpy as np
    from ksched_pkg import load
    synth = load().synth
    rng = np.random.default_rng(seed)
    shapes = [(c * 1000, m << 30) for c in synth.NODE_CPU_CORES.tolist() for m in synth.NODE_MEM_GIB.tolist()]
    vals = np.stack([rng.integers(0, cl.n_vals(k), VARIANTS) for k in range(cl.n_keys)], axis=1)  # [VARIANTS, keys]
    lab = np.zeros((VARIANTS, cl.label_words), np.uint64)
    for v in range(VARIANTS):
        for k in range(cl.n_keys):
            b = int(cl.pair_bit(k, vals[v, k]))
            lab[v, b // 64] |= np.uint64(1) << np.uint64(b % 64)
    ac = np.array([s[0] for s in shapes for _ in range(VARIANTS)], np.int64)
    am = np.array([s[1] for s in shapes for _ in range(VARIANTS)], np.int64)
    return ac, am, np.ascontiguousarray(np.tile(lab, (len(shapes), 1)))


def _restate_one(args):
    """One template through the restatement, in a worker process (the first-fit loop holds the GIL)."""
    from oracle import orc
    from scaleup_oracle import scaleup_packed
    ac, am, lab, mx, rc, rm, sel = args
    return scaleup_packed(orc, ac, am, ac, am, lab, mx, rc, rm, sel)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", default=None, help="directory for a torch.profiler trace of one more call")
    args = ap.parse_args()
    import numpy as np
    import ksched_pkg
    from oracle import orc
    from explain_oracle import explain_packed
    ks = ksched_pkg.load()
    if ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_scaleup_estimate has no CPU fallback"}), flush=True)
        return 2
    cl = ks.synth.config("c3")
    _, _, _, _, _, _, rc, rm, sel = cl.packed()
    rng = np.random.default_rng(0x5CA1E)
    pick = np.sort(rng.choice(len(rc), PODS, replace=False))
    rc, rm, sel = rc[pick], rm[pick], np.ascontiguousarray(sel[pick])
    ac, am, lab = templates(cl, 0x5CA1E)
    T = len(ac)
    mx = np.full(T, MAX_NODES, np.uint32)
    kernels_us = None
    with ks.Snapshot(0) as snap:
        ms = []
        for s in range(args.warmup + args.steps):
            t = time.perf_counter()
            rows, best, node, why = snap.scaleup_estimate(rc, rm, sel, ac, am, ac, am, lab, mx)
            if s >= args.warmup:
                ms.append((time.perf_counter() - t) * 1e3)
        if args.profile:
            import torch
            from torch.profiler import ProfilerActivity, profile
            os.makedirs(args.profile, exist_ok=True)
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                snap.scaleup_estimate(rc, rm, sel, ac, am, ac, am, lab, mx)
                torch.cuda.synchronize()
            prof.export_chrome_trace(os.path.join(args.profile, "scaleup_trace.json"))
            kernels_us = {}
            for ev in prof.events():
                if getattr(ev, "device_type", None) is not None and "k_scaleup" in ev.name:
                    name = "k_scaleup_pack" if "k_scaleup_pack" in ev.name else "k_scaleup_reasons"
                    kernels_us[name] = kernels_us.get(name, 0.0) + ev.device_time
    med = statistics.median(ms)
    cores = len(os.sched_getaffinity(0))
    sample = sorted(rng.choice(T, CPU_SAMPLE, replace=False).tolist())
    t = time.perf_counter()
    with ProcessPoolExecutor(min(cores, CPU_SAMPLE), mp_context=multiprocessing.get_context("spawn")) as ex:
        parts = list(ex.map(_restate_one, [(ac[i:i + 1], am[i:i + 1], lab[i:i + 1], mx[i:i + 1], rc, rm, sel)
                                           for i in sample]))
    cpu_s = time.perf_counter() - t
    for i, (w_rows, _, w_node, _) in zip(sample, parts):
        assert w_rows[0] == rows[i] and np.array_equal(w_node[0], node[i]), f"template {i}: call and restatement disagree"
    assert np.array_equal(explain_packed(orc, ac, am, lab, rc, rm, sel), why), "reasons: call and restatement disagree"
    cpu_ms = cpu_s * 1e3 * T / CPU_SAMPLE
    line = {"metric": "scaleup_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
            "workload": f"{PODS} seeded c3 pods (requests and selectors), {T} templates (36 shapes x {VARIANTS} label "
                        f"variants), max_nodes {MAX_NODES}, out_node and out_reasons requested",
            "call_ms": spread(ms), "cells_per_s": T * PODS / (med / 1e3), "us_per_template": med * 1e3 / T,
            "best": {"template": best, "placed": int(rows["placed"][best]) if best >= 0 else 0,
                     "nodes": int(rows["nodes"][best]) if best >= 0 else 0},
            "eligible_total": int(rows["eligible"].sum()), "nodes_max": int(rows["nodes"].max()),
            "cpu": {"ms": cpu_ms, "kind": "port", "cores": min(cores, CPU_SAMPLE), "workers": "processes",
                    "sample": f"{CPU_SAMPLE} seeded templates ({cpu_s:.2f} s), extrapolated to {T}",
                    "note": "restatement: oracle cell codes, then Python sort and numpy first fit per template"},
            "gpu_vs_cpu": cpu_ms / med,
            "note": "host-space pods and outputs, wall clock per call (the call returns after its D2H copy)"}
    if kernels_us is not None:
        line["kernels_us"] = kernels_us
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
