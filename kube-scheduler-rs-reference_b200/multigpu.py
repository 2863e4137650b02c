"""Pods-dimension sharding across ranks (SURVEY.md §8e): the node snapshot is replicated on every GPU, rank r
evaluates pods [lo_r, hi_r) and ONE all-gather of the packed per-pod bindings makes every rank hold all
bindings.  torch.distributed is plumbing only (NCCL on GPUs, gloo in the CPU tests)."""
import numpy as np

BYTES_PER_POD = 16  # score i64 | node_idx i32 | feasible_cnt u32


def shard_bounds(n_total, world, rank):
    """Contiguous, balanced split: the first (n_total % world) ranks get one extra pod."""
    base, extra = divmod(int(n_total), int(world))
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_capacity(n_total, world):
    return (int(n_total) + world - 1) // world


def binding_offsets(capacity):
    """Byte offsets of (score, node_idx, feasible_cnt) inside one shard buffer of `capacity` pods."""
    return 0, 8 * capacity, 12 * capacity


def pack_bindings(capacity, node_idx, score, cnt):
    """numpy helper (tests / CPU): build the shard buffer the GPU kernels write in place."""
    buf = np.zeros(capacity * BYTES_PER_POD, np.uint8)
    o_s, o_i, o_c = binding_offsets(capacity)
    n = len(node_idx)
    buf[o_s:o_s + 8 * n] = np.ascontiguousarray(score, np.int64).view(np.uint8)
    buf[o_i:o_i + 4 * n] = np.ascontiguousarray(node_idx, np.int32).view(np.uint8)
    buf[o_c:o_c + 4 * n] = np.ascontiguousarray(cnt, np.uint32).view(np.uint8)
    return buf


def unpack_bindings(gathered, n_total, world):
    """gathered: uint8 array of world * capacity * 16 bytes -> (node_idx, score, cnt) in global pod order."""
    cap = shard_capacity(n_total, world)
    g = np.asarray(gathered, np.uint8).reshape(world, cap * BYTES_PER_POD)
    o_s, o_i, o_c = binding_offsets(cap)
    idx, score, cnt = [], [], []
    for r in range(world):
        lo, hi = shard_bounds(n_total, world, r)
        n = hi - lo
        score.append(g[r, o_s:o_s + 8 * n].view(np.int64))
        idx.append(g[r, o_i:o_i + 4 * n].view(np.int32))
        cnt.append(g[r, o_c:o_c + 4 * n].view(np.uint32))
    return np.concatenate(idx), np.concatenate(score), np.concatenate(cnt)


def all_gather_bindings(local_buf, out_buf=None):
    """One collective: every rank contributes its shard buffer (torch uint8 tensor, equal sizes)."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size()
    if out_buf is None:
        out_buf = torch.empty(world * local_buf.numel(), dtype=torch.uint8, device=local_buf.device)
    dist.all_gather_into_tensor(out_buf, local_buf)
    return out_buf


class PeerExchange:
    """Gather buffers for the fused all-gather of the bindings (include/ksched.h, ks_exchange).

    Every rank owns one CUDA-IPC allocation  [score i64: world x cap | node_idx i32: world x cap | flags | state];
    rank r's argmax kernels store its shard's bindings into slot r of EVERY rank's buffer over NVLink and release one
    flag per destination; ks_select returns (stream-wise) once this rank's buffer holds every shard.
    torch.distributed only carries the 64-byte IPC handles at set-up time."""

    def __init__(self, device, world, rank, capacity, group=None):
        import ctypes as C
        import torch.distributed as dist
        from . import _capi as capi
        self.device, self.world, self.rank, self.cap = int(device), int(world), int(rank), int(capacity)
        self._capi, self._C = capi, C
        self.off_score = 0
        self.off_idx = self.world * self.cap * 8
        self.off_flags = (self.world * self.cap * 12 + 255) // 256 * 256
        self.off_state = self.off_flags + 256
        self.bytes = self.off_state + 256
        base = C.c_void_p()
        handle = C.create_string_buffer(64)
        capi.check(capi.lib.ks_ipc_alloc(self.device, self.bytes, C.byref(base), handle), "ks_ipc_alloc")
        self.base = base.value
        handles = [None] * self.world
        dist.all_gather_object(handles, handle.raw, group=group)
        self.peer_base = {}
        for r in range(self.world):
            if r == self.rank:
                continue
            p = C.c_void_p()
            capi.check(capi.lib.ks_ipc_open(self.device, handles[r], C.byref(p)), f"ks_ipc_open(rank {r})")
            self.peer_base[r] = p.value
        d = capi.ks_exchange()
        d.world, d.rank, d.n_peers = self.world, self.rank, self.world - 1
        for k, r in enumerate(sorted(self.peer_base)):
            d.peer_node_idx[k] = self.peer_base[r] + self.off_idx + self.rank * self.cap * 4
            d.peer_score[k] = self.peer_base[r] + self.off_score + self.rank * self.cap * 8
            d.peer_flag[k] = self.peer_base[r] + self.off_flags + self.rank * 4
        d.local_flags = self.base + self.off_flags
        d.local_state = self.base + self.off_state
        self.desc = d

    @property
    def node_idx_ptr(self):  # this rank's own slot: pass as ks_bindings.node_idx
        return self.base + self.off_idx + self.rank * self.cap * 4

    @property
    def score_ptr(self):
        return self.base + self.off_score + self.rank * self.cap * 8

    def read(self):
        """(node_idx [world, cap] int32, score [world, cap] int64) of everything gathered so far (synchronises)."""
        buf = np.empty(self.world * self.cap * 12, np.uint8)
        self._capi.check(self._capi.lib.ks_device_read(self.device, self.base, buf.ctypes.data, buf.nbytes),
                         "ks_device_read")
        score = buf[:self.off_idx].view(np.int64).reshape(self.world, self.cap)
        idx = buf[self.off_idx:self.off_idx + self.world * self.cap * 4].view(np.int32).reshape(self.world, self.cap)
        return idx, score

    def trace_ns(self):
        """Device-clock stamps (ns, %globaltimer of this rank's GPU) of the last exchange step:
        {"argmax1_start", "argmax2_start", "flags_published", "wait_started", "wait_done"}
        (ks_exchange.local_state words 2..11; synchronises)."""
        st = np.zeros(6, np.uint64)
        self._capi.check(self._capi.lib.ks_device_read(self.device, self.base + self.off_state, st.ctypes.data,
                                                       st.nbytes), "ks_device_read")
        names = ("argmax1_start", "flags_published", "wait_started", "wait_done", "argmax2_start")
        return {k: int(st[1 + i]) for i, k in enumerate(names)}

    def close(self):
        lib = self._capi.lib
        for p in self.peer_base.values():
            lib.ks_ipc_close(self.device, p)
        self.peer_base = {}
        if self.base:
            lib.ks_ipc_free(self.device, self.base)
            self.base = None


def stream_bind_distributed(snap, req_cpu, req_mem, sel, arrival, policy=0, max_rounds=64, done=True):
    """Streaming micro-batch on `world` replicas (config C5 on several GPUs).  Every rank holds a full replica of
    the snapshot and its own arrivals (`arrival` = globally unique, ordered ids).  Per round: local select (claims
    against the replica's free[]), ONE all-gather of the claims, and every rank commits the identical union in
    global arrival order (ks_snapshot_commit_claims) -> replicas stay bit-identical, capacity never over-commits.
    All ranks must call this in lockstep (a rank without arrivals passes empty arrays); `done` says that this rank
    has no further arrivals.  Returns (node_idx, rounds, all_ranks_done).
    `snap` needs .select(...)/.commit_claims(...) (ks.Snapshot; tests substitute an oracle-backed stand-in)."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size()
    n = len(req_cpu)
    req_cpu = np.asarray(req_cpu, np.int64)
    req_mem = np.asarray(req_mem, np.int64)
    sel = np.asarray(sel, np.uint64)
    sel = sel.reshape(n, sel.shape[-1] if sel.ndim > 1 else 1)
    arrival = np.asarray(arrival, np.int64)
    out_idx = np.full(n, -1, np.int32)
    pending = np.arange(n)
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
    rounds = 0
    all_done = False
    while rounds < max_rounds:
        m = len(pending)
        head = torch.tensor([m, 0 if done else 1], dtype=torch.int64, device=dev)
        dist.all_reduce(head, op=dist.ReduceOp.MAX)
        cap, all_done = int(head[0].item()), int(head[1].item()) == 0
        if cap == 0:
            break
        if m:
            r = snap.select(req_cpu[pending], req_mem[pending], sel[pending], policy=policy, flags=1)  # per-cell kernel
            idx = r.node_idx
        else:
            idx = np.zeros(0, np.int32)
        claim = np.full((cap, 4), -1, np.int64)  # [arrival, node, cpu, mem]; arrival -1 = padding
        claim[:m, 0] = arrival[pending]
        claim[:m, 1] = idx
        claim[:m, 2] = req_cpu[pending]
        claim[:m, 3] = req_mem[pending]
        mine = torch.from_numpy(claim).to(dev)
        allc = torch.empty((world * cap, 4), dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(allc, mine)
        allc = allc.cpu().numpy()
        allc = allc[allc[:, 0] >= 0]
        order = np.argsort(allc[:, 0], kind="stable")  # global arrival order
        allc = allc[order]
        acc = snap.commit_claims(allc[:, 1].astype(np.int32), allc[:, 2], allc[:, 3])
        accepted = dict(zip(allc[:, 0].tolist(), acc.tolist()))
        keep = []
        for k, p in enumerate(pending):
            if idx[k] < 0:
                continue
            if accepted[int(arrival[p])]:
                out_idx[p] = idx[k]
            else:
                keep.append(p)
        pending = np.asarray(keep, dtype=np.int64)
        rounds += 1
    return out_idx, rounds, all_done
