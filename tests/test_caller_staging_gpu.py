"""Caller-space staging (-m gpu): the calls whose caller says, per array, whether it is in host or device memory.  Each
space combination must return, bit for bit, what the same call returns with every array in device memory on the same
snapshot, and what the CPU oracle returns where the size is small.  Covers the two-chunk host pipeline of ks_select,
mixed mask / binding spaces, the host / device combinations of ks_select_topk and ks_preempt with each optional result
absent and present, and a caller stream for every call that takes one."""
import functools
import itertools

import numpy as np
import pytest

from preempt_oracle import crowded, preempt_packed
from topk_oracle import topk_packed

pytestmark = pytest.mark.gpu

N = 2000
PIPE_P = 262144 + 17  # the smallest batch ks_select pipelines in two pod chunks, plus an odd tail
H, D = 0, 1  # the spaces, as ks.KS_MEM_HOST / ks.KS_MEM_DEVICE


@functools.lru_cache(maxsize=2)
def _cluster(ks, P, seed):
    cl = ks.synth.make(P, N, seed=seed, bound_per_node=3)
    return cl.packed()


def _dev(x):
    import torch
    x = np.ascontiguousarray(x)
    return torch.from_numpy(x.view(np.int64) if x.dtype == np.uint64 else x).to("cuda:0")


def _pods(ks, space, rc, rm, sel):
    """(req_cpu, req_mem, sel, space) in the given space: numpy (pageable) for host, torch on cuda:0 for device."""
    if space == H:
        return rc, rm, np.ascontiguousarray(sel), ks.KS_MEM_HOST
    return _dev(rc), _dev(rm), _dev(sel), ks.KS_MEM_DEVICE


def _buf(space, shape, dtype, fill):
    """A result buffer filled with garbage: numpy for host, torch on cuda:0 for device."""
    a = np.full(shape, fill, dtype)
    return a if space == H else _dev(a)


def _host(a):
    return a if a is None or isinstance(a, np.ndarray) else a.cpu().numpy()


def _stream(use):
    import torch
    return torch.cuda.Stream() if use else None


def _sync(st):
    import torch
    (st.synchronize if st is not None else torch.cuda.synchronize)()


def _select(ks, snap, pods, n, policy, flags, out_space, mask_space=None, cnt=True, st=None):
    """ks_select through select_raw; returns (idx, score, cnt or None, mask or None) on the host."""
    mem = ks.KS_MEM_HOST if out_space == H else ks.KS_MEM_DEVICE
    idx = _buf(out_space, n, np.int32, -7)
    score = _buf(out_space, n, np.int64, -7)
    c = _buf(out_space, n, np.int32, -7) if cnt else None
    row = ks.capi.mask_row_bytes(N)
    mask = None if mask_space is None else _buf(mask_space, (n, row), np.uint8, 0x5A)
    snap.select_raw(n, *pods, idx, score, c, mem, mask=mask, mask_row_bytes=row if mask is not None else 0,
                    mask_space=ks.KS_MEM_HOST if mask_space == H else ks.KS_MEM_DEVICE, policy=policy, flags=flags,
                    stream=st.cuda_stream if st is not None else None)
    _sync(st)
    return _host(idx), _host(score), None if c is None else _host(c).view(np.uint32), _host(mask)


@pytest.mark.parametrize("policy", [0, 1])
def test_select_two_chunk_pipeline(ks, orc, policy):
    """Host pods and host bindings on the bit-parallel path at P >= 262144 run as two pod chunks; pageable memory, then
    pinned memory twice (capture, then replay of the cached graph)."""
    import torch
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, PIPE_P, 0xCA11)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        want = _select(ks, snap, _pods(ks, D, rc, rm, sel), PIPE_P, policy, ks.KS_SELECT_FORCE_DIRECT, D)[:3]
        s = np.unique(np.linspace(0, PIPE_P - 1, 300).astype(np.int64))
        fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
        o = orc.run_packed(fc, fm, ac, am, lab, rc[s], rm[s], sel[s], policy=policy, want_mask=False)[:3]
        for a, b in zip(want, o):
            assert np.array_equal(a[s], b)
        got = _select(ks, snap, _pods(ks, H, rc, rm, sel), PIPE_P, policy, ks.KS_SELECT_FORCE_BITPAR, H)[:3]
        assert snap.last_path() == "bitpar"
        for a, b in zip(got, want):
            assert np.array_equal(a, b), "pageable"
        pinned = [torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).pin_memory() for x in (rc, rm, sel)]
        outs = [torch.empty(PIPE_P, dtype=d).pin_memory() for d in (torch.int32, torch.int64, torch.int32)]
        for rep in range(2):
            for o_ in outs:
                o_.fill_(-7)
            snap.select_raw(PIPE_P, *pinned, ks.KS_MEM_HOST, *outs, ks.KS_MEM_HOST, policy=policy,
                            flags=ks.KS_SELECT_FORCE_BITPAR)
            got = [o_.numpy() for o_ in outs]
            got[2] = got[2].view(np.uint32)
            for a, b in zip(got, want):
                assert np.array_equal(a, b), ("pinned", rep)


@pytest.mark.parametrize("flags", ["FORCE_DIRECT", "FORCE_BITPAR"])
@pytest.mark.parametrize("pods_space", [H, D])
def test_select_mixed_spaces(ks, orc, flags, pods_space):
    """A host mask with device bindings, a device mask with host bindings, host bindings without a count, each on a
    caller stream and on the snapshot's."""
    P = 3000
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, P, 0x5E1)
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    o_idx, o_score, o_cnt, o_mask = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel)[:4]
    f = getattr(ks, "KS_SELECT_" + flags)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        pods = _pods(ks, pods_space, rc, rm, sel)
        want = _select(ks, snap, _pods(ks, D, rc, rm, sel), P, 0, f, D, mask_space=D)
        for a, b in zip(want, (o_idx, o_score, o_cnt, o_mask)):
            assert np.array_equal(a, b)
        for use_stream in (False, True):
            cases = {"host mask, device bindings": dict(out_space=D, mask_space=H),
                     "device mask, host bindings": dict(out_space=H, mask_space=D),
                     "host bindings, no count": dict(out_space=H, cnt=False)}
            for what, kw in cases.items():
                got = _select(ks, snap, pods, P, 0, f, st=_stream(use_stream), **kw)
                for a, b in zip(got, want):
                    assert a is None or np.array_equal(a, b), (what, use_stream)


@pytest.mark.parametrize("pods_space,out_space", list(itertools.product([H, D], [H, D])))
def test_topk_spaces(ks, orc, pods_space, out_space):
    """Every pods / results space pair, with score and count absent and present, on the snapshot's stream and a caller's;
    P small enough that the node dimension is split (partials in use)."""
    P, k = 700, 5
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, P, 0x70F)
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    o = topk_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, k, 1)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        pods = _pods(ks, pods_space, rc, rm, sel)
        mem = ks.KS_MEM_HOST if out_space == H else ks.KS_MEM_DEVICE
        for use_stream, optional in itertools.product((False, True), (False, True)):
            st = _stream(use_stream)
            idx = _buf(out_space, (P, k), np.int32, -7)
            score = _buf(out_space, (P, k), np.int64, -7) if optional else None
            cnt = _buf(out_space, P, np.int32, -7) if optional else None
            snap.select_topk_raw(P, *pods, k, idx, score, cnt, mem, policy=1,
                                 stream=st.cuda_stream if st is not None else None)
            _sync(st)
            assert np.array_equal(_host(idx), o[0]), (use_stream, optional)
            if optional:
                assert np.array_equal(_host(score), o[1]) and np.array_equal(_host(cnt).view(np.uint32), o[2])


@pytest.mark.parametrize("pods_space,out_space", list(itertools.product([H, D], [H, D])))
def test_preempt_spaces(ks, orc, pods_space, out_space):
    """Every pods / results space pair (priorities in the pods' space), with victims absent and present, on the snapshot's
    stream and a caller's."""
    P, mv = 600, 3
    ac, am, lab, bn, bc, bm, bp, rc, rm, sel, pp = crowded(ks, P, 700, 0x9E)
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    o_rows, o_vic = preempt_packed(orc, fc, fm, ac, am, lab, rc, rm, sel, pp, bn, bc, bm, bp, mv)
    assert (o_rows["node_idx"] >= 0).any(), "the workload must produce plans"
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        pods = _pods(ks, pods_space, rc, rm, sel)
        prio = pp if pods_space == H else _dev(pp)
        mem = ks.KS_MEM_HOST if out_space == H else ks.KS_MEM_DEVICE
        for use_stream, victims in itertools.product((False, True), (False, True)):
            st = _stream(use_stream)
            out = _buf(out_space, (P, 4), np.int64, -7)  # 32 bytes per row
            vic = _buf(out_space, (P, mv), np.int32, -7) if victims else None
            snap.preempt_raw(P, *pods, prio, (bn, bc, bm, bp), mv, out, vic, mem,
                             stream=st.cuda_stream if st is not None else None)
            _sync(st)
            rows = np.ascontiguousarray(_host(out)).view(ks.capi.PREEMPTION_DTYPE).reshape(P)
            for f in o_rows.dtype.names:
                assert np.array_equal(rows[f], o_rows[f]), (f, use_stream, victims)
            if victims:
                assert np.array_equal(_host(vic), o_vic), (use_stream, victims)


@pytest.mark.parametrize("pods_space,out_space", list(itertools.product([H, D], [H, D])))
def test_explain_spaces(ks, pods_space, out_space):
    """Every pods / results space pair on a caller stream, against the all-device call on the snapshot's stream."""
    P = 3000
    ac, am, lab, bn, bc, bm, rc, rm, sel = _cluster(ks, P, 0x5E1)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        want = _buf(D, (P, 4), np.int32, -7)
        snap.explain_raw(P, *_pods(ks, D, rc, rm, sel), want, ks.KS_MEM_DEVICE)
        _sync(None)
        want = _host(want)
        assert np.array_equal(want.view(np.uint32), snap.explain(rc, rm, sel))
        st = _stream(True)
        out = _buf(out_space, (P, 4), np.int32, -7)
        snap.explain_raw(P, *_pods(ks, pods_space, rc, rm, sel), out,
                         ks.KS_MEM_HOST if out_space == H else ks.KS_MEM_DEVICE, stream=st.cuda_stream)
        _sync(st)
        assert np.array_equal(_host(out), want)
