"""The staging set shared by every call that synchronises before it returns (-m gpu): the host-staged calls
(ks_scaleup_estimate, ks_gang_bind, ks_drain_check, ks_stream_bind's device loop, ks_place_replicas and
ks_place_replicas_spread) and the host-space pods and results of select, explain, top-k, preempt, check_cells, sampling,
commit_claims and apply_bind stage through one device in/work/out set per snapshot.  One snapshot runs a sequence of those calls that grows and shrinks the set, so each call
finds contents a larger call of another kind left behind.  Every result, and free[] after the committing calls, must
equal the same call on a fresh snapshot; cached-graph selects in between, with device-space buffers and with pinned host
pods, outputs and mask (a graph that points into the shared set), keep returning the oracle's bindings."""
from dataclasses import astuple

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, P = 2000, 6000


@pytest.fixture(scope="module")
def cluster(ks):
    cl = ks.synth.make(P, N, seed=0x57A6, bound_per_node=3)
    return cl.packed()


def _same(a, b):
    if isinstance(a, tuple):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        if a.dtype != b.dtype or a.shape != b.shape:
            return False
        if a.dtype.names:
            return all(np.array_equal(a[f], b[f]) for f in a.dtype.names)
        return np.array_equal(a, b)
    return a == b


def _templates(rng, T):
    ac = rng.choice([2000, 4000, 8000, 16000, 32000, 64000], T).astype(np.int64)
    am = rng.choice([8, 16, 32, 64, 128, 256], T).astype(np.int64) << 30
    fc, fm = ac - rng.integers(0, 500, T), am - rng.integers(0, 1 << 30, T)
    lab = rng.integers(0, 1 << 62, (T, 1)).astype(np.uint64) | np.uint64(0xFF)
    return ac, am, fc, fm, lab, rng.integers(1, 40, T).astype(np.uint32)


def _candidates(rng, D, pods_max):
    node = rng.integers(0, N, D).astype(np.int32)
    off = np.concatenate([[0], np.cumsum(rng.integers(0, pods_max + 1, D))]).astype(np.uint64)
    return node, off, rng.integers(0, P, int(off[-1]))


def test_shared_staging_across_call_kinds(ks, orc, cluster):
    import torch
    ac, am, lab, bn, bc, bm, rc, rm, sel = cluster
    rng = np.random.default_rng(0x57A6)
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    Q = 3000  # pods of the cached-graph selects
    o_idx, o_score, o_cnt, o_mask = orc.run_packed(fc, fm, ac, am, lab, rc[:Q], rm[:Q], sel[:Q])[:4]
    dev = torch.device("cuda:0")
    t = [torch.from_numpy(np.ascontiguousarray(x[:Q]).view(np.int64)).to(dev) for x in (rc, rm, sel)]
    idx = torch.empty(Q, dtype=torch.int32, device=dev)
    score = torch.empty(Q, dtype=torch.int64, device=dev)
    cnt = torch.empty(Q, dtype=torch.int32, device=dev)
    row = ks.capi.mask_row_bytes(N)
    h_pods = [x.cpu().pin_memory() for x in t]
    h_idx, h_score, h_cnt = (torch.empty(Q, dtype=d).pin_memory() for d in (torch.int32, torch.int64, torch.int32))
    h_mask = torch.empty((Q, row), dtype=torch.uint8).pin_memory()
    bprio = rng.integers(-100, 100, len(bn)).astype(np.int32)
    pprio = rng.integers(-100, 200, P).astype(np.int32)

    def fresh(call):
        with ks.Snapshot(0) as ref:
            ref.set_nodes(ac, am, lab)
            ref.set_bound(bn, bc, bm)
            return call(ref), ref.free()

    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)

        def run(what, call, commits=False):
            snap.set_bound(bn, bc, bm)  # committing calls start from the bound list's free[]; so does the select below
            got = call(snap)
            want, want_free = fresh(call)
            assert _same(got, want), what
            if commits:
                assert _same(snap.free(), want_free), f"free[] after {what}"
                snap.set_bound(bn, bc, bm)
            for rep in range(2):  # capture (or replay), then a replay of the cached graph
                idx.fill_(-7)
                cnt.fill_(-7)
                torch.cuda.synchronize()
                snap.select_raw(Q, t[0], t[1], t[2], ks.KS_MEM_DEVICE, idx, score, cnt, ks.KS_MEM_DEVICE)
                torch.cuda.synchronize()
                assert np.array_equal(idx.cpu().numpy(), o_idx), (what, rep)
                assert np.array_equal(score.cpu().numpy(), o_score), (what, rep)
                assert np.array_equal(cnt.cpu().numpy().view(np.uint32), o_cnt), (what, rep)
            for rep in range(2):  # the same select from pinned host memory: its graph points into d_in / d_out
                for b in (h_idx, h_cnt):
                    b.fill_(-7)
                h_mask.fill_(0x5A)
                snap.select_raw(Q, *h_pods, ks.KS_MEM_HOST, h_idx, h_score, h_cnt, ks.KS_MEM_HOST, mask=h_mask,
                                mask_row_bytes=row, mask_space=ks.KS_MEM_HOST)
                assert np.array_equal(h_idx.numpy(), o_idx), (what, "host", rep)
                assert np.array_equal(h_score.numpy(), o_score), (what, "host", rep)
                assert np.array_equal(h_cnt.numpy().view(np.uint32), o_cnt), (what, "host", rep)
                assert np.array_equal(h_mask.numpy(), o_mask), (what, "host mask", rep)

        big = _templates(rng, 256)
        run("scaleup T=256 P=4096 with out_node", lambda s: s.scaleup_estimate(rc[:4096], rm[:4096], sel[:4096], *big))
        off = np.array([0, 3, 5, 12], np.uint64)
        run("gang P=12 G=3", lambda s: s.gang_bind(rc[:12], rm[:12], sel[:12], off, np.array([3, 1, 7], np.uint32)),
            commits=True)
        run("select_topk", lambda s: s.select_topk(rc[:500], rm[:500], sel[:500], 8))
        node, doff, pick = _candidates(rng, 300, 12)
        first = len(pick)
        run("drain D=300 excluding candidates",
            lambda s: s.drain_check(rc[pick], rm[pick], sel[pick], node, doff, 0, ks.capi.KS_DRAIN_EXCLUDE_CANDIDATES))
        run("preempt", lambda s: s.preempt(rc[:400], rm[:400], sel[:400], pprio[:400], bn, bc, bm, bprio, 16))
        run("stream 1 pod", lambda s: s.stream_bind(rc[:1], rm[:1], sel[:1]), commits=True)
        run("stream 1024 pods", lambda s: s.stream_bind(rc[:1024], rm[:1024], sel[:1024]), commits=True)
        reps = rng.integers(0, 60, 200).astype(np.uint32)
        run("place_replicas T=200 with copies", lambda s: s.place_replicas(rc[:200], rm[:200], sel[:200], reps, 1))
        small = _templates(rng, 8)
        run("scaleup T=8 P=100 without out_node",
            lambda s: s.scaleup_estimate(rc[:100], rm[:100], sel[:100], *small, want_nodes=False))
        zone = (np.arange(N) % 4 - 1).astype(np.int32)  # -1 (no key), 0, 1, 2, ...
        ex = rng.integers(0, 5, (100, 3)).astype(np.uint32)
        run("place_replicas_spread T=100 with existing counts",
            lambda s: s.place_replicas_spread(rc[:100], rm[:100], sel[:100], reps[:100], zone, 3, np.full(100, 2),
                                              existing=ex))
        node, doff, pick = _candidates(rng, 900, 16)
        assert len(pick) > first
        run("drain D=900 policy 1", lambda s: s.drain_check(rc[pick], rm[pick], sel[pick], node, doff, 1))
        run("select with mask, all pods", lambda s: astuple(s.select(rc, rm, sel, want_mask=True)))
        run("explain", lambda s: s.explain(rc, rm, sel))
        # P x N bytes of codes: d_out grows past every earlier step (scale-up's out_node took 256 x 4096 x 4)
        run("check_cells", lambda s: s.check_cells(rc, rm, sel))
        run("select_sampling", lambda s: s.select_sampling(rc[:1000], rm[:1000], sel[:1000], seed=7))
        run("commit_claims", lambda s: s.commit_claims(o_idx, rc[:Q], rm[:Q]), commits=True)
        run("apply_bind", lambda s: s.apply_bind(int(o_idx[o_idx >= 0][0]), 100, 1 << 20), commits=True)
