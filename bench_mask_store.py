"""Store-pattern table of the mask pass on one GPU (BASELINE.md, "Mask pass: store patterns").

Part 1 compiles examples/mask_store_probe.cu (nvcc, sm_90a, into a temporary directory: the source tree may be read-only)
and runs its patterns on one 1M x 6400-byte buffer of its own, alternated, several repetitions each: P0 = a plain
128-bit-store fill, P1 = k_mask_rows' store shape, P2-P5 = P1 with one thing changed (whole-line store order, longer
column blocks, count atomics, record loads), P6 = P5 with the records staged in a shared-memory ring by bulk copies.  Part 2 times k_mask_rows itself on workload c3 through Snapshot.select_raw
with parts of its work switched off (counts NULL, mask NULL, the minimal row pitch), alternated the same way.
Prints one JSON line with min / median / max per row, the card's name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def spread(xs):
    xs = sorted(xs)
    return {"min": round(xs[0], 4), "median": round(statistics.median(xs), 4), "max": round(xs[-1], 4), "n": len(xs)}


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:
        return {"error": str(e)[:200]}


def probe(rows, pitch, reps):
    build = tempfile.mkdtemp(prefix="ks_mask_store_")
    exe = os.path.join(build, "mask_store_probe")
    try:
        nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        os.path.join(ROOT, "examples", "mask_store_probe.cu"), "-o", exe], check=True)
        out = subprocess.run([exe, str(rows), str(pitch), str(reps)], check=True, capture_output=True, text=True).stdout
    finally:
        shutil.rmtree(build, ignore_errors=True)
    res = json.loads(out)
    res["gbs"] = {k: spread(v) for k, v in res["gbs"].items()}
    return res


def ablations(reps):
    """k_mask_rows on c3 with parts of its work removed; every variant alternated, L2 flushed before every call."""
    import torch
    import ksched_pkg
    ks = ksched_pkg.load()
    dev = torch.device("cuda", 0)
    P, N = ks.synth.SHAPES["c3"]
    cl = ks.synth.make(P, N, ks.synth.SEEDS["c3"])
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    snap = ks.Snapshot(0)
    snap.set_nodes(ac, am, lab)
    snap.set_bound(bn, bc, bm)
    stream = torch.cuda.Stream()
    d_rc, d_rm = torch.from_numpy(rc).to(dev), torch.from_numpy(rm).to(dev)
    d_sel = torch.from_numpy(np.ascontiguousarray(sel).view(np.int64)).to(dev)
    d_cnt = torch.empty(P, dtype=torch.int32, device=dev)
    d_bind = torch.empty(P * 12, dtype=torch.uint8, device=dev)
    p_score, p_idx = d_bind.data_ptr(), d_bind.data_ptr() + 8 * P
    row_a, row_m = ks.mask_row_bytes_aligned(N), ks.mask_row_bytes(N)
    d_mask = torch.empty((P, row_a), dtype=torch.uint8, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    variants = {  # name: (mask row bytes or 0 = no mask, counts on)
        "as_bench": (row_a, True),
        "cnt_null": (row_a, False),
        "mask_null": (0, True),
        "pitch_minimal": (row_m, True),
    }

    def call(row, cnt, timing):
        snap.select_raw(P, d_rc, d_rm, d_sel, ks.KS_MEM_DEVICE, p_idx, p_score, d_cnt if cnt else None, ks.KS_MEM_DEVICE,
                        mask=d_mask if row else None, mask_row_bytes=row, mask_space=ks.KS_MEM_DEVICE,
                        policy=ks.KS_SCORE_LEFTOVER, flags=ks.KS_SELECT_AUTO | (ks.KS_SELECT_TIMING if timing else 0),
                        stream=stream.cuda_stream)

    for row, cnt in variants.values():  # warm-up: index build, graph capture of every variant
        for timing in (False, True, False):
            call(row, cnt, timing)
    stream.synchronize()
    k2 = {k: [] for k in variants}
    step = {k: [] for k in variants}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(reps):
        for name, (row, cnt) in variants.items():
            with torch.cuda.stream(stream):
                flush.fill_(1)
                e0.record(stream)
            call(row, cnt, False)
            with torch.cuda.stream(stream):
                e1.record(stream)
            stream.synchronize()
            step[name].append(e0.elapsed_time(e1))
            with torch.cuda.stream(stream):
                flush.fill_(2)
            call(row, cnt, True)
            stream.synchronize()
            k2[name].append(snap.last_timings()[0])
    snap.close()
    return {name: {"k2_ms": spread(k2[name]), "call_ms": spread(step[name]), "mask_row_bytes": variants[name][0],
                   "counts": variants[name][1]} for name in variants}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--pitch", type=int, default=6400)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--no-ablations", action="store_true")
    args = ap.parse_args()
    import bench
    sampler = bench.ClockSampler(0)
    try:  # the sampler's nvidia-smi child is stopped on every path
        line = {"card": card(), "probe": probe(args.rows, args.pitch, args.reps)}
        if not args.no_ablations:
            line["k_mask_rows_c3"] = ablations(args.reps)
    finally:
        clocks = sampler.stop()
    line["clocks"] = clocks
    print(json.dumps(line), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
