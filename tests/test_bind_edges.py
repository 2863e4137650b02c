"""Bind-walk edges, CPU part: reduced_reference (tests/bind_edges.py) against the five calls' oracles on every value
family of test_commit_paths_gpu.py and every policy each call takes, so that the reference and the oracles agree at the
edge values before a device compares with either; and the generators of test_bind_edges_gpu.py hitting the boundaries
they claim: ties on both sides of every slice edge of the walk, existing-pod sets that take the setup kernels' grid-stride
loop round a second time, slices longer than 256 nodes, node-rule words beyond one grid-stride pass, and a full-size
queue that fills most nodes before it ends."""
import numpy as np
import pytest

from bind_edges import (CALLS, EXISTING_E, EXISTING_N, FAMILY_N, FULL_N, FULL_P, LARGE_N, POLICIES, RULE_CLASSES,
                        RULE_N, TIE_N, bind_family, bind_slices, edge_keys, existing_pods, full_queue, no_rules, oracle,
                        reduced_reference, reduced_resources, resource_maps, setup_passes)
from test_commit_paths_gpu import FAMILIES

SMS = (114, 132)  # H100 PCIe and SXM


def _same(got, want, tag):
    for name, g, w in zip(("node_idx", "score", "parts", "refused"), got[:4], want[:4]):
        assert np.array_equal(g, w), f"{name} {tag}: first rows {np.nonzero(np.asarray(g) != np.asarray(w))[0][:8]}"


@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("call", CALLS)
def test_reduced_reference_is_the_oracle(call, fam):
    """Groups without constraints and group -1, no terms, no soft keys, rules that pass every node, and for fit three
    resources (pod slots, GPUs, FPGAs; negative free included): node, score, parts, refusals, the charged free[] and
    free_r of reduced_reference equal the oracle's, at every policy the call takes and at N around the slice edges of
    132 SMs"""
    G, R = 3, 3
    for policy in POLICIES[call]:
        for N, W, P in ((1, 1, 12), (37, 2, 40), (300, 8, 60)):
            rng = np.random.default_rng([CALLS.index(call), FAMILIES.index(fam), policy, N])
            ac, am, lab, fc, fm, rc, rm, sel, group, keys = bind_family(fam, rng, N, P, W, 132, G)
            node_free, pod_req = reduced_resources(rng, N, P, R) if call == "fit" else (None, None)
            res = resource_maps(node_free, pod_req) if call == "fit" else None
            ofc, ofm, rfc, rfm = fc.copy(), fm.copy(), fc.copy(), fm.copy()
            want = oracle(call, ofc, ofm, ac, am, lab, rc, rm, sel, group, G, keys, policy,
                          skew=np.zeros((G, len(keys)), np.uint32) if call == "spread" else None,
                          cluster=no_rules(N, G), res=res)
            got = reduced_reference(call, rfc, rfm, ac, am, lab, rc, rm, sel, policy, node_free, pod_req)
            tag = f"{call} {fam} policy={policy} N={N}"
            _same(got, want, tag)
            assert np.array_equal(rfc, ofc) and np.array_equal(rfm, ofm), tag
            assert all(not c.any() for c in want[4]), tag  # no constraint: every count stays 0
            if call == "fit":
                assert np.array_equal(got[6], want[6]), tag
            if call == "fit" and N > 1:
                assert got[3][:, 0].any(), tag


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("N", FAMILY_N + (LARGE_N,))
def test_slice_ties_straddle_every_bind_slice_edge(sms, N):
    """"slice ties": the best free on both sides of every edge between two CTA slices of the walk, and on the first and
    last node; allocatables equal, so the nodes tie under every policy.  The zones of edge_keys cross every edge."""
    rng = np.random.default_rng(N + sms)
    ac, am, lab, fc, fm, rc, rm, sel, group, keys = bind_family("slice ties", rng, N, 8, 1, sms, 3)
    grid, chunk = bind_slices(N, sms)
    best = (fc == fc.max()) & (fm == fm.max())
    assert best[0] and best[-1] and (ac == ac[0]).all() and (am == am[0]).all()
    zone = keys[0][0]
    for s in range(1, grid):
        e = s * chunk
        if e < N:
            assert best[e - 1] and best[e], (s, e)
            inside = zone[max(0, e - chunk // 2):e + 1]
            assert len(set(inside[inside >= 0].tolist())) <= 1  # both sides in one zone (or without the key)
    for g in np.unique(group[group >= 0]):  # one selector per group
        assert (sel[group == g] == sel[group == g][:1]).all()


@pytest.mark.parametrize("sms", SMS)
def test_large_shapes_have_slices_longer_than_a_cta(sms):
    """The large-N and tie shapes give each thread several nodes of its slice (slice > 256 = threads per CTA); the
    family rotation's largest N too"""
    for N in (TIE_N, LARGE_N, FAMILY_N[-1]):
        grid, chunk = bind_slices(N, sms)
        assert grid == sms and chunk > 256, (N, grid, chunk)
    assert bind_slices(TIE_N - 1, 132)[1] == 256  # one node less: one node per thread on 132 SMs


@pytest.mark.parametrize("sms", SMS)
def test_existing_pods_take_a_second_setup_turn(sms):
    """E = 20,000 existing pods exceed the 8 * 4 * SMs warps of k_affinity_setup / k_profile_setup, so their grid-stride
    loop turns at least twice; about 5% of them sit on nodes that lack a key"""
    assert EXISTING_E > 8 * 4 * sms and setup_passes(EXISTING_E, sms) >= 2
    assert setup_passes(8 * 4 * sms, sms) == 1 and setup_passes(8 * 4 * sms + 1, sms) == 2
    rng = np.random.default_rng(sms)
    keys = edge_keys(rng, EXISTING_N, sms)
    _, nodes = existing_pods(rng, keys, 16, EXISTING_E)
    lack = ((keys[0][0][nodes] < 0) | (keys[1][0][nodes] < 0)).mean()
    assert 0.03 < lack < 0.07


@pytest.mark.parametrize("sms", SMS)
def test_rule_words_exceed_one_grid_stride_pass(sms):
    """64 node-rule classes x 16,897 nodes = 1.08 M rule words, more than k_node_rules_setup's 4 * SMs CTAs of 256
    threads cover in one pass"""
    assert RULE_CLASSES * RULE_N > 4 * sms * 256
    assert RULE_CLASSES * RULE_N > 1 << 20


def test_full_queue_fills_most_nodes():
    """The full-size queue (65,536 pods, 2,000 nodes): most pod slots and GPU nodes fill and the end of the queue is
    mostly refused under fit; without the resources, cpu and memory run out before the queue ends"""
    rng = np.random.default_rng(7)
    fc, fm, ac, am, lab, rc, rm, sel, group, keys, node_free, pod_req = full_queue(rng, FULL_N, FULL_P)
    node, _, _, refused, _, _, free_r = reduced_reference("fit", fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, 4,
                                                          node_free, pod_req)
    gpu_nodes = node_free[1] > 0
    assert (free_r[0] == 0).mean() > 0.4 and (free_r[1][gpu_nodes] == 0).mean() > 0.8
    assert (node[-2000:] < 0).mean() > 0.9 and refused[:, 0].any()
    node, *_ = reduced_reference("spread", fc.copy(), fm.copy(), ac, am, lab, rc, rm, sel, 1)
    assert (node[-2000:] < 0).mean() > 0.9 and (node >= 0).sum() > FULL_P // 2
