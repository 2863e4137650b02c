"""KS_SCORE_LEAST_BALANCED with the fused all-gather of the bindings (ks_exchange): two ranks on the bit-parallel path,
where k_least_balanced stores every binding into both ranks' gather buffers.  Every rank must end with every rank's
bindings, and its own counts and mask, bit for bit against the CPU restatement of the unsharded batch."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _worker(rank, world, port, P, N, steps, q):
    try:
        sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
        import torch
        import torch.distributed as dist
        import ksched_pkg
        ks = ksched_pkg.load()
        from oracle import orc
        from least_balanced_oracle import LEAST_BALANCED, Oracle
        o = Oracle(orc)
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        device = rank % max(1, torch.cuda.device_count())
        torch.cuda.set_device(device)
        dev = torch.device("cuda", device)
        cl = ks.synth.make(P, N, seed=7070 + N, bound_per_node=4)
        ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
        lo, hi = ks.multigpu.shard_bounds(P, world, rank)
        cap = ks.multigpu.shard_capacity(P, world)
        n = hi - lo
        snap = ks.Snapshot(device)
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        xch = ks.multigpu.PeerExchange(device, world, rank, max(cap, 1))
        t = [torch.from_numpy(np.ascontiguousarray(x[lo:hi]).view(np.int64).copy()).to(dev) for x in (rc, rm, sel)]
        cnt = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        row = ks.mask_row_bytes(N)
        mask = torch.zeros((max(n, 1), row), dtype=torch.uint8, device=dev)
        st = torch.cuda.Stream()
        fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
        ok = True
        for step in range(steps):
            rc_it = rc + 50 * step  # new requests every step: stale data in a gather buffer would be detected
            t[0].copy_(torch.from_numpy(np.ascontiguousarray(rc_it[lo:hi])))
            torch.cuda.synchronize()
            dist.barrier()
            snap.select_raw(n, t[0], t[1], t[2], ks.KS_MEM_DEVICE, xch.node_idx_ptr, xch.score_ptr, cnt, ks.KS_MEM_DEVICE,
                            mask=mask, mask_row_bytes=row, mask_space=ks.KS_MEM_DEVICE, policy=LEAST_BALANCED,
                            flags=ks.KS_SELECT_FORCE_BITPAR, stream=st.cuda_stream, exchange=xch)
            st.synchronize()
            snap.exchange_check()
            ok &= n == 0 or snap.last_path() == "bitpar"  # an empty shard only takes part in the exchange
            g_idx, g_score = xch.read()
            fi, fs, fcn, fmask, _ = o.run_packed(fc, fm, ac, am, lab, rc_it, rm, sel, LEAST_BALANCED, want_mask=True)
            for r in range(world):
                a, b = ks.multigpu.shard_bounds(P, world, r)
                ok &= np.array_equal(g_idx[r, :b - a], fi[a:b]) and np.array_equal(g_score[r, :b - a], fs[a:b])
            ok &= np.array_equal(cnt.cpu().numpy()[:n].view(np.uint32), fcn[lo:hi])
            ok &= np.array_equal(mask.cpu().numpy()[:n], fmask[lo:hi])
            dist.barrier()
        xch.close()
        snap.close()
        q.put((rank, bool(ok), n, ""))
        dist.destroy_process_group()
    except Exception as e:  # report instead of hanging the parent
        import traceback
        q.put((rank, False, -1, traceback.format_exc()[-1500:] + str(e)))


@pytest.mark.parametrize("P,N,steps", [(20000, 3000, 3), (1, 5000, 2)])
def test_least_balanced_exchange_two_ranks(P, N, steps):
    """P = 1 leaves rank 1 with an empty shard."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 37000 + (os.getpid() % 2000) + P % 7
    procs = [ctx.Process(target=_worker, args=(r, 2, port, P, N, steps, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(r[0] for r in res) == [0, 1], res
    assert all(r[1] for r in res), res
    assert sum(r[2] for r in res) == P
