#!/usr/bin/env python
"""bench_fit_scaleup.py — cost of ks_fit_scaleup_estimate (the scale-up estimate under the full filter:
k_node_rules_setup + k_fit_scaleup_pack + k_fit_scaleup_reasons) on one H100.

Workload: bench_scaleup.py's (20 000 seeded c3 pending pods, 288 templates of 36 shapes x 8 label variants, max_nodes
1024) with what makes the full filter decide on a GPU cluster:
  - every template's pod limit is 110 ("pods" allocatable; node_free = 110, each pod requests 1);
  - 32 more templates of 96 cores, 1152 GiB and 8 GPUs, tainted nvidia.com/gpu=present:NoSchedule;
  - a seeded 5 % of the pods request 1-8 GPUs and belong to a group that tolerates the taint;
  - a seeded 10 % of the others carry a required node-affinity term `instance-type In {6 of the 37 types}` (16 groups).
Pods and outputs are host memory.
  - call_ms: the whole call with out_node and out_refused, median / min / max of --steps calls after --warmup;
  - e1: the E1 configuration (rules and resources NULL) and ks_scaleup_estimate on the same pods and templates,
    alternated call by call in one run, each median / min / max, their ratio, and the outputs checked equal (E1);
  - kernels_us: per-kernel device time of one full call under torch.profiler (--profile DIR also keeps the trace);
  - misplaced: pods ks_scaleup_estimate calls placeable (eligible for some template) that no template accepts under
    the full filter, and how the best template's placed pods and nodes differ between the two calls.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_explain import gpu_info, spread  # noqa: E402
from bench_scaleup import MAX_NODES, PODS, templates  # noqa: E402

GPU_TEMPLATES = 32
AFF_GROUPS = 16


def workload(np, ks):
    cl = ks.synth.config("c3")
    _, _, _, _, _, _, rc, rm, sel = cl.packed()
    rng = np.random.default_rng(0x5CA1E)
    pick = np.sort(rng.choice(len(rc), PODS, replace=False))
    rc, rm, sel = rc[pick], rm[pick], np.ascontiguousarray(sel[pick])
    ac, am, lab = templates(cl, 0x5CA1E)
    n_shapes = len(ac) // 8
    rng = np.random.default_rng(0xF17)
    gl = lab[rng.integers(0, len(ac), GPU_TEMPLATES)]
    ac = np.concatenate([ac, np.full(GPU_TEMPLATES, 96000, np.int64)])
    am = np.concatenate([am, np.full(GPU_TEMPLATES, 1152 << 30, np.int64)])
    lab = np.ascontiguousarray(np.concatenate([lab, gl]))
    T, P = len(ac), PODS
    itype = np.concatenate([np.repeat(np.arange(n_shapes), 8), np.full(GPU_TEMPLATES, n_shapes)]).astype(np.int32)
    D = n_shapes + 1
    gpu = np.zeros(T, bool)
    gpu[-GPU_TEMPLATES:] = True
    # groups: 0 tolerates the GPU taint; 1..AFF_GROUPS each require instance-type In a seeded set of 6 types
    group = np.full(P, -1, np.int32)
    gp = rng.random(P) < 0.05
    group[gp] = 0
    ap = ~gp & (rng.random(P) < 0.10)
    group[ap] = rng.integers(1, AFF_GROUPS + 1, int(ap.sum()))
    terms = []
    for g in range(1, AFF_GROUPS + 1):
        w = np.zeros((D + 64) // 64, np.uint64)
        for d in rng.choice(D, 6, replace=False):
            w[d // 64] |= np.uint64(1) << np.uint64(d % 64)
        terms.append((g, 0, [(0, w)]))
    rules = dict(n_taints=1, taint_hard=gpu.astype(np.uint64), tolerate_hard=np.array([1] + [0] * AFF_GROUPS, np.uint64),
                 rule_keys=[(itype, D)], node_terms=terms)
    node_free = np.stack([np.full(T, 110, np.int64), np.where(gpu, 8, 0).astype(np.int64)])
    pod_req = np.zeros((P, 2), np.int64)
    pod_req[:, 0] = 1
    pod_req[gp, 1] = rng.integers(1, 9, int(gp.sum()))
    return rc, rm, sel, ac, am, lab, np.full(T, MAX_NODES, np.uint32), group, AFF_GROUPS + 1, rules, node_free, pod_req


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", default=None, help="directory for the torch.profiler trace of the profiled call")
    args = ap.parse_args()
    import numpy as np
    import ksched_pkg
    ks = ksched_pkg.load()
    if ks.device_count() == 0:
        print(json.dumps({"error": "no CUDA device: ks_fit_scaleup_estimate has no CPU fallback"}), flush=True)
        return 2
    rc, rm, sel, ac, am, lab, mx, group, G, rules, node_free, pod_req = workload(np, ks)
    T, P = len(ac), len(rc)
    none = np.full(P, -1, np.int32)
    with ks.Snapshot(0) as snap:
        def full():
            return snap.fit_scaleup_estimate(rc, rm, sel, ac, am, ac, am, lab, mx, group, G, rules=rules,
                                             node_free=node_free, pod_req=pod_req)

        def e1():
            return snap.fit_scaleup_estimate(rc, rm, sel, ac, am, ac, am, lab, mx, none, 0)

        def old():
            return snap.scaleup_estimate(rc, rm, sel, ac, am, ac, am, lab, mx)

        def timed(f, into, keep):
            t = time.perf_counter()
            r = f()
            if keep:
                into.append((time.perf_counter() - t) * 1e3)
            return r
        ms, ms_e1, ms_old = [], [], []
        for s in range(args.warmup + args.steps):
            got = timed(full, ms, s >= args.warmup)
        for s in range(args.warmup + args.steps):  # alternated call by call
            r_e1 = timed(e1, ms_e1, s >= args.warmup)
            r_old = timed(old, ms_old, s >= args.warmup)
        assert np.array_equal(r_e1[0], r_old[0]) and r_e1[1] == r_old[1] and np.array_equal(r_e1[2], r_old[2]), "E1"
        assert np.array_equal(r_e1[3][:, 0], r_old[3][:, 2] + r_old[3][:, 3]) and not r_e1[3][:, 1:].any(), "E1 words"
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            full()
            torch.cuda.synchronize()
        if args.profile:
            os.makedirs(args.profile, exist_ok=True)
            prof.export_chrome_trace(os.path.join(args.profile, "fit_scaleup_trace.json"))
        kernels_us = {}
        for ev in prof.events():
            if getattr(ev, "device_type", None) is not None and ev.device_type == torch.autograd.DeviceType.CUDA:
                for k in ("k_fit_scaleup_pack", "k_fit_scaleup_reasons", "k_node_rules_setup"):
                    if k in ev.name:
                        kernels_us[k] = kernels_us.get(k, 0.0) + ev.device_time
    rows, best, node, refused, used = got
    orow, obest, _, why = r_old
    old_elig = T - why[:, 2].astype(np.int64) - why[:, 3]
    new_elig = T - refused.sum(axis=1).astype(np.int64)
    line = {"metric": "fit_scaleup_ms", "unit": "ms", "gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
            "workload": f"{P} seeded c3 pods, {T} templates (bench_scaleup's 288 + {GPU_TEMPLATES} tainted 8-GPU), "
                        f"max_nodes {MAX_NODES}, pods 110 each; 5% GPU pods (1-8 GPUs, tolerating), 10% required "
                        f"instance-type In (16 groups); out_node and out_refused requested",
            "call_ms": spread(ms),
            "e1": {"fit_scaleup_ms": spread(ms_e1), "scaleup_ms": spread(ms_old),
                   "ratio": statistics.median(ms_e1) / statistics.median(ms_old), "outputs": "equal (E1)"},
            "kernels_us": kernels_us,
            "best": {"template": best, "placed": int(rows["placed"][best]) if best >= 0 else 0,
                     "nodes": int(rows["nodes"][best]) if best >= 0 else 0,
                     "gpus_used": int(used[best, 1]) if best >= 0 else 0},
            "old_best": {"template": obest, "placed": int(orow["placed"][obest]) if obest >= 0 else 0,
                         "nodes": int(orow["nodes"][obest]) if obest >= 0 else 0},
            "misplaced": {"placeable_by_old_not_under_full_filter": int(((old_elig > 0) & (new_elig == 0)).sum()),
                          "gpu_pods": int((pod_req[:, 1] > 0).sum()),
                          "refused_totals": refused.sum(axis=0).tolist()},
            "eligible_total": int(rows["eligible"].sum()), "nodes_max": int(rows["nodes"].max()),
            "note": "host-space pods and outputs, wall clock per call (the call returns after its D2H copy)"}
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
