"""GPU parity tests (-m gpu): the CUDA path through the C ABI vs the CPU oracle, bit-exact
(integer / bit work: no tolerance).  Small sizes compare everything; BASELINE.json's full sizes use a full
packed-oracle comparison where the CPU finishes in seconds (C2) and size-independent properties + sampled
rows beyond that (C3)."""
import numpy as np
import pytest

from helpers import load_golden, mask_bits, pack_by_dictionary, rows_to_str

pytestmark = pytest.mark.gpu

import os

_ALL_PATHS = {"direct": 1, "bitpar": 2}  # KS_SELECT_FORCE_DIRECT / KS_SELECT_FORCE_BITPAR
PATHS = {k: v for k, v in _ALL_PATHS.items() if k in os.environ.get("KS_TEST_PATHS", "direct,bitpar").split(",")}


def _oracle(orc, cl, policy, want_codes=False):
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    return orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, policy=policy, want_codes=want_codes)


# The policies whose bit-parallel argmax walks a bound order with an early exit: k_least_alloc (1) and bound_walk's
# k_most_alloc (3) and k_least_balanced (4).  LEAST_ALLOCATED's cases keep their ids.
BOUND_ORDERED = {1: "", 3: "-most_allocated", 4: "-least_balanced"}


def _with_policies(cases):
    return [pytest.param(*c, q, id="-".join(map(str, c)) + sfx) for c in cases for q, sfx in BOUND_ORDERED.items()]


def _snapshot(ks, cl):
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    snap = ks.Snapshot(0)
    snap.set_nodes(ac, am, lab)
    snap.set_bound(bn, bc, bm)
    return snap, (rc, rm, sel)


def _assert_same(r, o, tag):
    oidx, oscore, ocnt, omask, _ = o
    assert np.array_equal(r.feasible_cnt, ocnt), f"{tag}: feasible_cnt"
    assert np.array_equal(r.mask, omask), f"{tag}: mask"
    assert np.array_equal(r.node_idx, oidx), f"{tag}: node_idx"
    assert np.array_equal(r.score, oscore), f"{tag}: score"


def test_gv1_config_c1_through_abi(ks, orc):
    """BASELINE.json configs[0]: 10 pods x 5 nodes, resource_fits only — golden vector GV-1."""
    g = load_golden("gv1.json")
    names = [n["name"] for n in g["nodes"]]
    alloc = [(4000, 8589934592), (2000, 4294967296), (8000, 17179869184), (1000, 1073741824), (0, 0)]
    bound = [(1, 500, 1073741824), (2, 2000, 4294967296), (2, 500, 536870912), (3, 1000, 1073741824), (4, 100, 1)]
    labels, sel = pack_by_dictionary([n["labels"] for n in g["nodes"]], [None] * 10)
    assert names == ["n0", "n1", "n2", "n3", "n4"]
    with ks.Snapshot(0) as snap:
        snap.set_nodes([a[0] for a in alloc], [a[1] for a in alloc], labels)
        snap.set_bound([b[0] for b in bound], [b[1] for b in bound], [b[2] for b in bound])
        fc, fm = snap.free()
        assert list(fc) == g["expected_free_cpu_milli"] and list(fm) == g["expected_free_mem_bytes"]
        rc, rm = g["expected_req_cpu_milli"], g["expected_req_mem_bytes"]
        codes = snap.check_cells(rc, rm, sel)
        assert rows_to_str(codes == 0) == g["expected_feasible_rows"]
        assert set(np.unique(codes)) <= {0, 1}
        for name, flag in PATHS.items():
            r = snap.select(rc, rm, sel, flags=flag, want_mask=True)
            assert rows_to_str(mask_bits(r.mask, 5)) == g["expected_feasible_rows"], name
            assert list(r.node_idx) == g["expected_node_idx_leftover"], name
            assert list(r.feasible_cnt) == [s.count("1") for s in g["expected_feasible_rows"]], name
        for p in range(10):
            for n in range(5):
                assert snap.check_cell(rc[p], rm[p], sel[p], n) == codes[p, n]


def test_gv1_objects_vs_faithful_oracle(ks, orc):
    """Same GV-1 objects through the faithful (string-parsing) oracle and through the GPU reason codes."""
    g = load_golden("gv1.json")
    arena = ks.objects.ObjectArena()
    nodes, allp, pods = arena.nodes(g["nodes"]), arena.pods(g["bound_pods"]), arena.pods(g["pods"])
    oc = orc.Cluster(nodes, 5, allp, len(g["bound_pods"]))
    _, _, _, _, ocodes = oc.run(pods, 10, want_codes=True)
    labels, sel = pack_by_dictionary([n["labels"] for n in g["nodes"]], [None] * 10)
    with ks.Snapshot(0) as snap:
        snap.set_nodes([4000, 2000, 8000, 1000, 0], [8589934592, 4294967296, 17179869184, 1073741824, 0], labels)
        snap.set_bound([1, 2, 2, 3, 4], [500, 2000, 500, 1000, 100], [1073741824, 4294967296, 536870912, 1073741824, 1])
        codes = snap.check_cells(g["expected_req_cpu_milli"], g["expected_req_mem_bytes"], sel)
    assert np.array_equal(codes, ocodes)


SHAPES = [
    (1, 1, 8), (5, 31, 8), (33, 32, 8), (100, 1024, 8), (257, 1025, 8), (1000, 3000, 8), (300, 2049, 16),
    (64, 2500, 32), (40, 1300, 64), (2000, 256, 8), (3, 20000, 8),
    (300, 150_000, 8),  # more column blocks than SMs: every CTA walks several column blocks
]


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("P,N,keys", SHAPES)
def test_random_clusters_leftover(ks, orc, path, P, N, keys):
    cl = ks.synth.make(P, N, seed=1000 + P + N, n_keys=keys, bound_per_node=4)
    snap, (rc, rm, sel) = _snapshot(ks, cl)
    with snap:
        fc, fm = snap.free()
        cfc, cfm = cl.free()
        assert np.array_equal(fc, cfc) and np.array_equal(fm, cfm)  # K0 vs numpy
        r = snap.select(rc, rm, sel, policy=ks.KS_SCORE_LEFTOVER, flags=PATHS[path], want_mask=True)
        assert r.path == path
        _assert_same(r, _oracle(orc, cl, 0), f"{path} {P}x{N} W={cl.label_words}")


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("P,N,keys", [(5, 31, 8), (257, 1025, 8), (500, 3000, 8), (64, 2500, 32), (3, 20000, 8), (4000, 9000, 8),
                                      (300, 150_000, 8),
                                      (300, 2049, 16),  # one tile past a column block: the last block holds one real tile
                                      (40, 1300, 64)])  # W = 8: k_least_alloc<8> reads the bound-order pair columns through L1/L2
def test_random_clusters_least_allocated(ks, orc, path, P, N, keys):
    """KS_SCORE_LEAST_ALLOCATED (not separable): the per-cell kernel and the bit-parallel path (bound-ordered scan with
    early exit, k_least_alloc) against the oracle - node, score, count and mask."""
    cl = ks.synth.make(P, N, seed=2000 + P + N, n_keys=keys, bound_per_node=4)
    snap, (rc, rm, sel) = _snapshot(ks, cl)
    with snap:
        r = snap.select(rc, rm, sel, policy=ks.KS_SCORE_LEAST_ALLOCATED, flags=PATHS[path], want_mask=True)
        assert r.path == path
        _assert_same(r, _oracle(orc, cl, 1), f"least-allocated {path} {P}x{N}")
        assert r.score.min() >= 0 and r.score.max() <= 100
        auto = snap.select(rc, rm, sel, policy=ks.KS_SCORE_LEAST_ALLOCATED)
        assert auto.path == ("bitpar" if P * N >= 1 << 24 else "direct") and np.array_equal(auto.node_idx, r.node_idx)


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("seed,P,N,policy", _with_policies([(11, 3000, 6000), (12, 700, 40_000)]))
def test_least_allocated_near_ties(ks, orc, path, seed, P, N, policy):
    """Homogeneous clusters: thousands of nodes whose LeastAllocated scores lie within a point or two of each other
    (and many exact ties), so the single-precision pre-filter of k_least_alloc keeps whole tiles of candidates and the
    winner is decided by the exact integer score and then the lowest node index - vs the oracle, every pod.  Under
    policies 3 and 4 the same near ties sit at bound_walk's early exit."""
    from policy_oracle import Oracle
    rng = np.random.default_rng(seed)
    ac = rng.choice(np.array([64000, 64000, 64001, 63999, 32000], np.int64), N)
    am = rng.choice(np.array([1 << 38, (1 << 38) + 4096, 1 << 37], np.int64), N)
    lab = np.zeros((N, 1), np.uint64)
    lab[:, 0] = rng.choice(np.array([1, 3, 7], np.uint64), N)
    B = 2 * N  # bound pods leave every node about half full, within a percent of each other
    bn = np.repeat(np.arange(N, dtype=np.int32), 2)
    bc = (ac[bn] // 4 + rng.integers(0, 400, B)).astype(np.int64)
    bm = (am[bn] // 4 + rng.integers(0, 1 << 30, B)).astype(np.int64)
    rc = rng.integers(0, 16000, P).astype(np.int64)
    rm = rng.integers(0, 1 << 35, P).astype(np.int64)
    sel = np.zeros((P, 1), np.uint64)
    sel[:, 0] = rng.choice(np.array([0, 1, 2, 4], np.uint64), P)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        ofc, ofm = orc.free_reduce(ac, am, bn, bc, bm)
        r = snap.select(rc, rm, sel, policy=policy, flags=PATHS[path], want_mask=False)
        o = Oracle(orc).run_packed(ofc, ofm, ac, am, lab, rc, rm, sel, policy, want_mask=False)
        assert r.path == path
        assert np.array_equal(r.score, o[1]), f"near ties {path}: score"
        assert np.array_equal(r.node_idx, o[0]), f"near ties {path}: node_idx (tie-break by node index)"
        assert np.array_equal(r.feasible_cnt, o[2])
        assert len(np.unique(r.score[r.node_idx >= 0])) <= 60  # the scores really are bunched


@pytest.mark.parametrize("path,policy", _with_policies([(p,) for p in PATHS]))
def test_least_allocated_round_fills(ks, orc, path, policy):
    """Nodes filled to exact quarters of round capacities and round requests: the memory quotient (free - request) * 100 /
    allocatable is often EXACTLY an integer, where k_least_alloc's single-precision estimate cannot know the floor and must
    fall back to the 64-bit arithmetic of the evaluation row; every node is feasible for most pods and most scores tie.
    Under policies 3 and 4 exact shares put many scores exactly on bound_walk's limits."""
    from policy_oracle import Oracle
    rng = np.random.default_rng(5)
    N, P = 9000, 2500
    ac = rng.choice(np.array([4000, 8000, 16000], np.int64), N)
    am = rng.choice(np.array([16, 32, 64], np.int64) << 30, N)
    lab = np.zeros((N, 1), np.uint64)
    bn = np.arange(N, dtype=np.int32)
    bc = (ac // 4 * rng.integers(0, 4, N)).astype(np.int64)
    bm = (am // 4 * rng.integers(0, 4, N)).astype(np.int64)
    rc = rng.choice(np.array([0, 250, 1000], np.int64), P)
    rm = rng.choice(np.array([0, 1 << 30, 1 << 32], np.int64), P)
    sel = np.zeros((P, 1), np.uint64)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        ofc, ofm = orc.free_reduce(ac, am, bn, bc, bm)
        r = snap.select(rc, rm, sel, policy=policy, flags=PATHS[path], want_mask=False)
        o = Oracle(orc).run_packed(ofc, ofm, ac, am, lab, rc, rm, sel, policy, want_mask=False)
        assert r.path == path
        assert np.array_equal(r.score, o[1]), f"round fills {path}: score"
        assert np.array_equal(r.node_idx, o[0]), f"round fills {path}: node_idx"
        assert np.array_equal(r.feasible_cnt, o[2])


def test_reason_codes_match_oracle(ks, orc):
    cl = ks.synth.make(200, 777, seed=31, bound_per_node=4)
    snap, (rc, rm, sel) = _snapshot(ks, cl)
    with snap:
        codes = snap.check_cells(rc, rm, sel)
    ocodes = _oracle(orc, cl, 0, want_codes=True)[4]
    assert np.array_equal(codes, ocodes)
    assert set(np.unique(codes)) == {0, 1, 2}


def test_objects_faithful_oracle_vs_gpu(ks, orc):
    """End-to-end object parity: strings -> faithful oracle (per-cell parse + bound re-sum) vs GPU on packed."""
    cl = ks.synth.make(48, 300, seed=77, bound_per_node=3)
    nodes_s, bound_s, pods_s = ks.objects.cluster_specs(cl)
    arena = ks.objects.ObjectArena()
    nodes, bound, pods = arena.nodes(nodes_s), arena.pods(bound_s), arena.pods(pods_s)
    oc = orc.Cluster(nodes, cl.N, bound, cl.B)
    f = oc.run(pods, cl.P, policy=0)
    snap, (rc, rm, sel) = _snapshot(ks, cl)
    with snap:
        for name, flag in PATHS.items():
            r = snap.select(rc, rm, sel, flags=flag, want_mask=True)
            _assert_same(r, f, f"objects {name}")


def test_edge_cases(ks, orc):
    one = np.ones((1, 1), np.uint64)
    with ks.Snapshot(0) as snap:
        # empty node store: every pod gets None (src/main.rs:56,70)
        snap.set_nodes(np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 1), np.uint64))
        r = snap.select([1, 2], [1, 2], np.zeros((2, 1), np.uint64))
        assert list(r.node_idx) == [-1, -1] and list(r.feasible_cnt) == [0, 0] and list(r.score) == [0, 0]
        # zero-request pod fits iff free >= 0 in both (node with negative free is infeasible)
        snap.set_nodes([1000, 1000], [100, 100], np.zeros((2, 1), np.uint64))
        snap.set_bound([1], [1001], [0])
        for flag in PATHS.values():
            r = snap.select([0, 1000, 1001], [0, 100, 0], np.zeros((3, 1), np.uint64), flags=flag, want_mask=True)
            assert list(r.feasible_cnt) == [1, 1, 0] and list(r.node_idx) == [0, 0, -1]
            assert list(r.score) == [1000 * (1 << 22) + 100, 0, 0]
        # selector bit no node carries -> NodeSelectorMismatch everywhere; fit still reported first
        assert snap.check_cell(0, 0, one[0], 0) == ks.KS_CELL_NODE_SELECTOR_MISMATCH
        assert snap.check_cell(5000, 0, one[0], 0) == ks.KS_CELL_NOT_ENOUGH_RESOURCES
        # ties -> lowest node index
        snap.set_nodes([500] * 40, [64] * 40, np.zeros((40, 1), np.uint64))
        for flag in PATHS.values():
            r = snap.select([100], [1], np.zeros((1, 1), np.uint64), flags=flag)
            assert r.node_idx[0] == 0 and r.feasible_cnt[0] == 40


def test_incremental_bind_equals_rebuild(ks, orc):
    cl = ks.synth.make(300, 500, seed=5, bound_per_node=2)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    with ks.Snapshot(0) as a, ks.Snapshot(0) as b:
        a.set_nodes(ac, am, lab)
        a.set_bound(bn, bc, bm)
        r0 = a.select(rc, rm, sel)
        # bind the first 20 schedulable pods one by one
        extra = [(int(r0.node_idx[p]), int(rc[p]), int(rm[p])) for p in range(300) if r0.node_idx[p] >= 0][:20]
        for n, c, m in extra:
            a.apply_bind(n, c, m)
        b.set_nodes(ac, am, lab)
        b.set_bound(np.concatenate([bn, [e[0] for e in extra]]), np.concatenate([bc, [e[1] for e in extra]]),
                    np.concatenate([bm, [e[2] for e in extra]]))
        fa, fb = a.free(), b.free()
        assert np.array_equal(fa[0], fb[0]) and np.array_equal(fa[1], fb[1])
        for flag in PATHS.values():
            ra = a.select(rc, rm, sel, flags=flag, want_mask=True)
            rb = b.select(rc, rm, sel, flags=flag, want_mask=True)
            assert np.array_equal(ra.node_idx, rb.node_idx) and np.array_equal(ra.mask, rb.mask)


@pytest.mark.parametrize("pitch", ["minimal", "aligned", "odd"])
def test_device_buffers_and_user_stream(ks, orc, pitch):
    """KS_MEM_DEVICE arguments (torch tensors only provide the memory and the stream), with the smallest legal mask row
    pitch, the recommended 256-byte-block pitch (ks_mask_row_bytes_aligned) and a pitch in between."""
    import torch
    cl = ks.synth.make(5000, 4500, seed=9)  # 18 tiles: 576-byte rows, 768 aligned
    snap, (rc, rm, sel) = _snapshot(ks, cl)
    o = _oracle(orc, cl, 0)
    dev = torch.device("cuda:0")
    t = [torch.from_numpy(np.ascontiguousarray(x.view(np.int64))).to(dev) for x in (rc, rm, sel)]
    row_min = ks.mask_row_bytes(cl.N)
    row = {"minimal": row_min, "aligned": ks.mask_row_bytes_aligned(cl.N), "odd": row_min + 64}[pitch]
    assert row % 32 == 0 and row >= row_min and ks.mask_row_bytes_aligned(cl.N) % 256 == 0
    idx = torch.empty(cl.P, dtype=torch.int32, device=dev)
    score = torch.empty(cl.P, dtype=torch.int64, device=dev)
    cnt = torch.empty(cl.P, dtype=torch.int32, device=dev)
    mask = torch.zeros((cl.P, row), dtype=torch.uint8, device=dev)
    st = torch.cuda.Stream()
    with snap:
        for name, flag in PATHS.items():
            idx.fill_(-7)
            mask.fill_(0xA5 if name == "bitpar" else 0)  # the bit-parallel path overwrites every whole tile of the pitch
            torch.cuda.synchronize()
            snap.select_raw(cl.P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, idx, score, cnt, ks.KS_MEM_DEVICE, mask=mask,
                            mask_row_bytes=row, mask_space=ks.KS_MEM_DEVICE, flags=flag, stream=st.cuda_stream)
            st.synchronize()
            assert np.array_equal(idx.cpu().numpy(), o[0])
            assert np.array_equal(score.cpu().numpy(), o[1])
            assert np.array_equal(cnt.cpu().numpy().view(np.uint32), o[2])
            m = mask.cpu().numpy()
            assert np.array_equal(m[:, :row_min], o[3])
            assert (m[:, row_min:] == 0).all()


def test_bad_arguments_are_status_codes(ks):
    with ks.Snapshot(0) as snap:
        with pytest.raises(ks.KsError):
            snap.set_nodes([1], [1], np.zeros((1, 3), np.uint64))  # W must be 1/2/4/8
        with pytest.raises(ks.KsError):
            snap.set_nodes([1 << 40], [1], np.zeros((1, 1), np.uint64))  # out of range
        snap.set_nodes([1], [1], np.zeros((1, 1), np.uint64))
        with pytest.raises(ks.KsError):
            snap.set_bound([3], [1], [1])  # node index out of range
        with pytest.raises(ks.KsError):
            snap.select([1], [1], np.zeros((1, 1), np.uint64), policy=7)


def _properties(ks, r, N):
    bits_cnt = np.unpackbits(r.mask, axis=1).sum(axis=1)
    assert np.array_equal(bits_cnt.astype(np.uint32), r.feasible_cnt)          # checksum of the mask
    assert np.array_equal(r.node_idx < 0, r.feasible_cnt == 0)                 # None <=> empty feasible set
    has = r.node_idx >= 0
    idx = r.node_idx[has].astype(np.int64)
    rows = np.nonzero(has)[0]
    assert ((r.mask[rows, idx // 8] >> (idx % 8).astype(np.uint8)) & 1).all()  # chosen node is feasible
    assert (r.mask[:, (N + 7) // 8:] == 0).all()                               # padding bits stay clear


@pytest.mark.parametrize("path", list(PATHS))
def test_config_c2_full_size_bit_exact(ks, orc, path):
    """BASELINE.json configs[1]: 100k pods x 10k nodes, resource_fits + nodeSelector (1e9 cells), full compare."""
    cl = ks.synth.config("c2")
    snap, (rc, rm, sel) = _snapshot(ks, cl)
    with snap:
        r = snap.select(rc, rm, sel, flags=PATHS[path], want_mask=True)
    _properties(ks, r, cl.N)
    _assert_same(r, _oracle(orc, cl, 0), f"C2 {path}")


def test_mask_dynamic_work_distribution_mid_size(ks, orc):
    """400k pods x 6000 nodes (3 column blocks, ~50 CTAs each): the mask kernel's dynamic work distribution (k_mask_rows:
    one atomic cursor per column block, warps claim pod groups, CTAs move to the block with the most work left) on a
    problem small enough for a full compare.  The mask is pre-filled so that a pod group nobody processed shows."""
    import torch
    cl = ks.synth.make(400000, 6000, seed=0x5EA1, bound_per_node=2)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    P, N = cl.P, cl.N
    dev = torch.device("cuda:0")
    row_min, row = ks.mask_row_bytes(N), ks.mask_row_bytes_aligned(N)
    t = [torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(dev) for x in (rc, rm, sel)]
    idx = torch.empty(P, dtype=torch.int32, device=dev)
    score = torch.empty(P, dtype=torch.int64, device=dev)
    cnt = torch.empty(P, dtype=torch.int32, device=dev)
    mask = torch.empty((P, row), dtype=torch.uint8, device=dev)
    st = torch.cuda.Stream()
    snap, _ = _snapshot(ks, cl)
    o_idx, o_score, o_cnt, o_mask, _ = _oracle(orc, cl, 0)
    with snap:
        for rep in range(3):  # replays of the cached graph re-arm the cursors every time
            mask.fill_(0xA5)
            cnt.fill_(-1)
            torch.cuda.synchronize()
            snap.select_raw(P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, idx, score, cnt, ks.KS_MEM_DEVICE, mask=mask,
                            mask_row_bytes=row, mask_space=ks.KS_MEM_DEVICE, flags=PATHS.get("bitpar", 0), stream=st.cuda_stream)
            st.synchronize()
            assert snap.last_path() == "bitpar"
            m = mask.cpu().numpy()
            assert np.array_equal(m[:, :row_min], o_mask), f"mask, pass {rep}"
            assert (m[:, row_min:] == 0).all(), f"mask padding, pass {rep}"
            assert np.array_equal(cnt.cpu().numpy().view(np.uint32), o_cnt), f"feasible_cnt, pass {rep}"
            assert np.array_equal(idx.cpu().numpy(), o_idx) and np.array_equal(score.cpu().numpy(), o_score)


def test_config_c3_full_size_bit_exact(ks, orc):
    """BASELINE.json configs[2]: 1M x 50k (5e10 cells).  EVERY output of the bit-parallel path is compared with the
    packed oracle: the 6.27 GB feasible mask stays in HBM and is checked slab by slab (all host threads run the
    oracle on each slab), bindings / scores / counts over the whole batch; the per-cell kernel must agree too."""
    import torch
    cl = ks.synth.config("c3")
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    P, N = cl.P, cl.N
    dev = torch.device("cuda:0")
    row_min, row = ks.mask_row_bytes(N), ks.mask_row_bytes_aligned(N)  # 6272 and 6400: the pitch bench.py uses
    t = [torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(dev) for x in (rc, rm, sel)]
    idx = torch.empty(P, dtype=torch.int32, device=dev)
    score = torch.empty(P, dtype=torch.int64, device=dev)
    cnt = torch.empty(P, dtype=torch.int32, device=dev)
    mask = torch.empty((P, row), dtype=torch.uint8, device=dev)
    mask.fill_(0xA5)  # every byte of every row must be overwritten
    st = torch.cuda.Stream()
    snap, _ = _snapshot(ks, cl)
    with snap:
        snap.select_raw(P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, idx, score, cnt, ks.KS_MEM_DEVICE, mask=mask,
                        mask_row_bytes=row, mask_space=ks.KS_MEM_DEVICE, flags=PATHS.get("bitpar", 0), stream=st.cuda_stream)
        st.synchronize()
        assert snap.last_path() == "bitpar"
        g_idx, g_score, g_cnt = idx.cpu().numpy(), score.cpu().numpy(), cnt.cpu().numpy().view(np.uint32)
        if "direct" in PATHS:
            b = snap.select(rc, rm, sel, flags=PATHS["direct"])
            assert np.array_equal(g_idx, b.node_idx) and np.array_equal(g_score, b.score) and np.array_equal(g_cnt, b.feasible_cnt)
    assert np.array_equal(g_idx < 0, g_cnt == 0)
    # slabs of 50k pods (2.5e9 cells each; ~1 s of oracle time on a 128-thread host).  The whole mask is covered unless
    # the host is so small that it would take longer than KS_TEST_C3_SECONDS (default 150): then every k-th slab is
    # checked (first and last included) and the test says so.
    import time
    import warnings
    slab = 50000
    n_slabs = (P + slab - 1) // slab
    budget = float(os.environ.get("KS_TEST_C3_SECONDS", "150"))
    stride, t_first, done = 1, None, 0
    k = 0
    while k < n_slabs:
        lo, hi = k * slab, min(P, (k + 1) * slab)
        t0 = time.perf_counter()
        o = orc.run_packed(fc, fm, ac, am, lab, rc[lo:hi], rm[lo:hi], sel[lo:hi], want_mask=True, nthreads=0)
        assert np.array_equal(g_idx[lo:hi], o[0]) and np.array_equal(g_score[lo:hi], o[1]), f"bindings, slab {k}"
        assert np.array_equal(g_cnt[lo:hi], o[2]), f"feasible_cnt, slab {k}"
        m = mask[lo:hi].cpu().numpy()
        assert np.array_equal(m[:, :row_min], o[3]), f"mask, slab {k}"
        assert (m[:, row_min:] == 0).all(), f"mask padding, slab {k}"
        done += 1
        if t_first is None:
            t_first = time.perf_counter() - t0
            stride = max(1, int(np.ceil(t_first * n_slabs / budget)))
        k = k + stride if k + stride < n_slabs or k == n_slabs - 1 else n_slabs - 1
    if stride > 1:
        warnings.warn(f"C3 mask: {done} of {n_slabs} slabs compared ({t_first:.1f} s per slab on this host)")


def test_graph_replay_tracks_snapshot_changes(ks, orc):
    """Repeated calls with identical buffers replay a cached CUDA graph (device and pinned-host buffers); any
    snapshot mutation must invalidate it, and changed pod values in the same buffers must be honoured."""
    import torch
    cl = ks.synth.make(3000, 6000, seed=21)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    dev = torch.device("cuda:0")
    row = ks.mask_row_bytes(cl.N)

    def buffers(space):
        if space == ks.KS_MEM_DEVICE:
            mk = lambda a: torch.from_numpy(np.ascontiguousarray(a.view(np.int64))).to(dev)
            out = lambda n, dt: torch.empty(n, dtype=dt, device=dev)
        else:
            mk = lambda a: torch.from_numpy(np.ascontiguousarray(a.view(np.int64))).pin_memory()
            out = lambda n, dt: torch.empty(n, dtype=dt).pin_memory()
        return [mk(rc), mk(rm), mk(sel)], out(cl.P, torch.int32), out(cl.P, torch.int64), out(cl.P, torch.int32)

    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        mask = torch.zeros((cl.P, row), dtype=torch.uint8, device=dev)
        big = 2 * cl.P  # doubled per pass, so that every pass grows the index's per-call pod scratch
        for space in (ks.KS_MEM_DEVICE, ks.KS_MEM_HOST):
            t, idx, score, cnt = buffers(space)
            st = torch.cuda.Stream()

            def run():
                snap.select_raw(cl.P, t[0], t[1], t[2], space, idx, score, cnt, space, mask=mask, mask_row_bytes=row,
                                mask_space=ks.KS_MEM_DEVICE, flags=ks.KS_SELECT_FORCE_BITPAR, stream=st.cuda_stream)
                st.synchronize()
                return idx.cpu().numpy().copy(), score.cpu().numpy().copy(), cnt.cpu().numpy().view(np.uint32).copy()

            fc, fm = snap.free()
            o = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, want_mask=False)
            for _ in range(3):  # capture, replay, replay
                g = run()
                assert all(np.array_equal(a, b) for a, b in zip(g, o[:3]))
            # mutate the snapshot: the next call must see it
            snap.apply_bind(int(o[0][o[0] >= 0][0]), 10_000_000, 1 << 40)
            fc, fm = snap.free()
            o2 = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, want_mask=False)
            g = run()
            assert all(np.array_equal(a, b) for a, b in zip(g, o2[:3]))
            assert not np.array_equal(o2[0], o[0])
            # same buffers, new pod values: the graph replays with the new contents
            rc2 = rc.copy()
            rc2[::2] += 50
            t[0].copy_(torch.from_numpy(rc2))
            torch.cuda.synchronize()
            o3 = orc.run_packed(fc, fm, ac, am, lab, rc2, rm, sel, want_mask=False)
            g = run()
            assert all(np.array_equal(a, b) for a, b in zip(g, o3[:3]))
            t[0].copy_(torch.from_numpy(rc))
            torch.cuda.synchronize()
            # an uncached device-space select of more pods moves only the index's pod scratch (pod ranks, tail list,
            # mask records): the cached graph points into the old buffers and must not be replayed
            reps = big // cl.P
            tb = [torch.from_numpy(np.ascontiguousarray(np.concatenate([a] * reps).view(np.int64))).to(dev)
                  for a in (rc, rm, sel)]
            ib = torch.empty(big, dtype=torch.int32, device=dev)
            sb = torch.empty(big, dtype=torch.int64, device=dev)
            cb = torch.empty(big, dtype=torch.int32, device=dev)
            snap.select_raw(big, tb[0], tb[1], tb[2], ks.KS_MEM_DEVICE, ib, sb, cb, ks.KS_MEM_DEVICE,
                            flags=ks.KS_SELECT_FORCE_BITPAR | ks.KS_SELECT_NO_GRAPH, stream=st.cuda_stream)
            st.synchronize()
            assert snap.last_path() == "bitpar"
            gb = ib.cpu().numpy(), sb.cpu().numpy(), cb.cpu().numpy().view(np.uint32)
            assert all(np.array_equal(a, np.tile(b, reps)) for a, b in zip(gb, o2[:3]))
            big *= 2
            g = run()
            assert all(np.array_equal(a, b) for a, b in zip(g, o2[:3]))


def test_bindings_ready_event_orders_a_side_stream(ks, orc):
    """ks_bindings.bindings_ready_event: a consumer on another stream that waits for the event must see the final
    node_idx/score of THIS call (also when the call is replayed from the cached CUDA graph with new pod values)."""
    import torch
    cl = ks.synth.make(40000, 3000, seed=33)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    dev = torch.device("cuda:0")
    row = ks.mask_row_bytes(cl.N)
    t = [torch.from_numpy(np.ascontiguousarray(x.view(np.int64))).to(dev) for x in (rc, rm, sel)]
    idx = torch.full((cl.P,), -9, dtype=torch.int32, device=dev)
    score = torch.zeros(cl.P, dtype=torch.int64, device=dev)
    cnt = torch.zeros(cl.P, dtype=torch.int32, device=dev)
    mask = torch.zeros((cl.P, row), dtype=torch.uint8, device=dev)
    st, side = torch.cuda.Stream(), torch.cuda.Stream()
    ev = torch.cuda.Event()
    ev.record(st)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        fc, fm = snap.free()
        for it in range(4):
            rc_it = rc + 50 * it
            t[0].copy_(torch.from_numpy(rc_it))
            torch.cuda.synchronize()
            snap.select_raw(cl.P, t[0], t[1], t[2], ks.KS_MEM_DEVICE, idx, score, cnt, ks.KS_MEM_DEVICE, mask=mask,
                            mask_row_bytes=row, mask_space=ks.KS_MEM_DEVICE, flags=ks.KS_SELECT_FORCE_BITPAR,
                            stream=st.cuda_stream, ready_event=ev.cuda_event)
            side.wait_event(ev)
            with torch.cuda.stream(side):
                early_idx, early_score = idx.clone(), score.clone()
            side.synchronize()
            st.synchronize()
            o = orc.run_packed(fc, fm, ac, am, lab, rc_it, rm, sel, want_mask=False)
            assert np.array_equal(early_idx.cpu().numpy(), o[0]), it
            assert np.array_equal(early_score.cpu().numpy(), o[1]), it
            assert np.array_equal(cnt.cpu().numpy().view(np.uint32), o[2]), it


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("seed,P,N,W", [(1, 3000, 700, 1), (2, 20000, 1100, 2), (3, 9000, 5000, 1), (4, 70000, 300, 4)])
def test_adversarial_values(ks, orc, path, seed, P, N, W):
    """Unstructured inputs: heavy ties in free values, negative and zero requests, values at the API limits, dense
    random selector words (many required bits, bits no node carries), nodes with negative free - vs the oracle."""
    rng = np.random.default_rng(seed)
    lim_c, lim_m = 1 << 36, 1 << 55
    pool_c = np.array([-5, 0, 1, 250, 1000, 1000, 4000, 64000, lim_c // 2], np.int64)  # free must stay within the limits
    pool_m = np.array([-1, 0, 1, 1 << 20, 1 << 30, 1 << 30, 1 << 34, lim_m // 2], np.int64)
    ac = rng.choice(pool_c, N)
    am = rng.choice(pool_m, N)
    lab = rng.integers(0, 1 << 63, size=(N, W), dtype=np.uint64) & rng.integers(0, 1 << 63, size=(N, W), dtype=np.uint64)
    B = 3 * N
    bn = rng.integers(0, N, B).astype(np.int32)
    bc = rng.choice(np.array([0, 0, 100, 1000, -100], np.int64), B)
    bm = rng.choice(np.array([0, 1, 1 << 20, 1 << 28, -1], np.int64), B)
    rc = rng.choice(np.array([-1000, 0, 0, 1, 250, 1000, 1001, 4000, 63999, lim_c], np.int64), P)
    rm = rng.choice(np.array([-1, 0, 1, (1 << 20) - 1, 1 << 20, 1 << 30, (1 << 30) + 1, lim_m], np.int64), P)
    sel = np.zeros((P, W), np.uint64)
    k = rng.integers(0, 10, P)  # 0..9 required bits per pod, taken from some node's labels or random
    for p in np.nonzero(k)[0]:
        src = lab[rng.integers(0, N)] if rng.random() < 0.7 else rng.integers(0, 1 << 63, size=W, dtype=np.uint64)
        bits = [(w, b) for w in range(W) for b in range(64) if (int(src[w]) >> b) & 1]
        for i in rng.permutation(len(bits))[:k[p]]:
            w, b = bits[i]
            sel[p, w] |= np.uint64(1) << np.uint64(b)
    with ks.Snapshot(0) as snap:
        snap.set_nodes(ac, am, lab)
        snap.set_bound(bn, bc, bm)
        fc, fm = snap.free()
        ofc, ofm = orc.free_reduce(ac, am, bn, bc, bm)
        assert np.array_equal(fc, ofc) and np.array_equal(fm, ofm)
        r = snap.select(rc, rm, sel, flags=PATHS[path], want_mask=True)
        o = orc.run_packed(ofc, ofm, ac, am, lab, rc, rm, sel)
        _assert_same(r, o, f"adversarial {path} seed {seed}")
        # the non-separable scores on the same path; negative requests void the early-exit bound of k_least_alloc and
        # bound_walk, allocatables <= 0 give no slack, free above allocatable is stored at 2^62 under policy 4
        from policy_oracle import Oracle
        for q in BOUND_ORDERED:
            r1 = snap.select(rc, rm, sel, policy=q, flags=PATHS[path], want_mask=False)
            o1 = Oracle(orc).run_packed(ofc, ofm, ac, am, lab, rc, rm, sel, q, want_mask=False)
            assert r1.path == path and np.array_equal(r1.node_idx, o1[0]) and np.array_equal(r1.score, o1[1]), q
            assert np.array_equal(r1.feasible_cnt, o1[2]), q


def _stream_states(ks, seed, P, first=0):
    return np.array([ks.capi.sampling_stream(seed, first + p) for p in range(P)], np.uint64)


@pytest.mark.parametrize("P,N,keys,attempts", [(500, 40, 8, 5), (4000, 3000, 8, 5), (3000, 777, 32, 3), (1000, 5, 8, 16)])
def test_reference_sampling_policy_bit_exact(ks, orc, P, N, keys, attempts):
    """(f)#4: the reference's own <=ATTEMPTS random draws (src/main.rs:49-71), seeded: every draw, every reason
    code and the outcome equal the oracle's restatement driven by the same generator states."""
    cl = ks.synth.make(P, N, seed=4242 + N, n_keys=keys, bound_per_node=6)
    ac, am, lab, bn, bc, bm, rc, rm, sel = cl.packed()
    fc, fm = orc.free_reduce(ac, am, bn, bc, bm)
    seed = 0xB2000005 ^ N
    o = orc.sampling_packed(fc, fm, lab, rc, rm, sel, attempts, _stream_states(ks, seed, P))
    _, _, ocnt, omask, ocodes = orc.run_packed(fc, fm, ac, am, lab, rc, rm, sel, want_codes=True)
    snap, _ = _snapshot(ks, cl)
    with snap:
        idx, used, dn, dc = snap.select_sampling(rc, rm, sel, attempts=attempts, seed=seed)
        # a chunked caller reproduces the single call through first_pod_index
        half = P // 2
        idx2, used2, _, _ = snap.select_sampling(rc[half:], rm[half:], sel[half:], attempts=attempts, seed=seed,
                                                 first_pod_index=half)
    for got, want, name in zip((idx, used, dn, dc), o, ("node_idx", "attempts", "draw_node", "draw_code")):
        assert np.array_equal(got, want), name
    assert np.array_equal(idx2, idx[half:]) and np.array_equal(used2, used[half:])
    # the policy's contract against the exhaustive answer: a pick is feasible; no feasible node -> None;
    # None is allowed although feasible nodes exist (the reference gives up after its draws)
    bits = mask_bits(omask, N)
    picked = idx >= 0
    assert bits[np.nonzero(picked)[0], idx[picked]].all()
    assert (idx[ocnt == 0] == -1).all()
    made = dn >= 0
    pp = np.broadcast_to(np.arange(P)[:, None], dn.shape)
    assert np.array_equal(dc[made], ocodes[pp[made], dn[made]])
    assert picked.any() and ((~picked) & (ocnt > 0)).any() or N <= 5


def test_reference_sampling_policy_faithful_objects(ks, orc):
    """Same policy on the object path: host layer (strings -> packer -> device) vs the faithful oracle pod by pod."""
    from test_host_layer import _cluster_objects
    cl = ks.synth.make(60, 90, seed=99, bound_per_node=3)
    arena, nodes, bound, pods = _cluster_objects(ks, cl)
    oc = orc.Cluster(nodes, cl.N, bound, cl.B)
    seed = 777
    with ks.host.Context(0) as ctx:
        ctx.set_nodes(nodes, cl.N)
        ctx.set_cluster_pods(bound, cl.B)
        idx, used, dn, dc = ctx.select_node_for_pod(pods, cl.P, seed=seed)
    for p in range(cl.P):
        n, cells = oc.sampling(pods, p, 5, seed=ks.capi.sampling_stream(seed, p))
        assert (idx[p], used[p]) == (n, cells), p


def test_reference_sampling_policy_edge_cases(ks):
    one = np.zeros((1, 1), np.uint64)
    with ks.Snapshot(0) as snap:
        # empty node store: every attempt is wasted (src/main.rs:56,60)
        idx, used, dn, dc = snap.select_sampling(np.array([1], np.int64), np.array([1], np.int64), one, seed=3)
        assert idx[0] == -1 and used[0] == 0 and (dn == -1).all() and (dc == 0xff).all()
        snap.set_nodes(np.array([1000], np.int64), np.array([1 << 30], np.int64), one)
        idx, used, dn, dc = snap.select_sampling(np.array([1000, 1001], np.int64), np.array([1, 1], np.int64),
                                                 np.zeros((2, 1), np.uint64), seed=3)
        assert idx.tolist() == [0, -1] and used.tolist() == [1, 5]
        assert dc[0].tolist() == [0, 255, 255, 255, 255] and dc[1].tolist() == [1] * 5
        idx, used, _, _ = snap.select_sampling(np.array([1], np.int64), np.array([1], np.int64), one, attempts=0)
        assert idx[0] == -1 and used[0] == 0
        e = np.zeros(0, np.int64)
        idx, _, _, _ = snap.select_sampling(e, e, np.zeros((0, 1), np.uint64))
        assert idx.shape == (0,)
