"""Shared test helpers: spec normalisation for golden fixtures, mask decoding, packed-oracle wrappers."""
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_golden(name):
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)


def mask_bits(mask_rows, n_nodes):
    """uint8 [P,row] -> bool [P,N] (bit n%8 of byte n/8)."""
    bits = np.unpackbits(np.ascontiguousarray(mask_rows), axis=1, bitorder="little")
    return bits[:, :n_nodes].astype(bool)


def rows_to_str(bits):
    return ["".join("1" if b else "0" for b in row) for row in bits]


def pack_by_dictionary(node_label_maps, pod_selector_maps):
    """Test-side label packing (independent of the C++ packer): one bit per (key,value) pair carried by some
    node; every pair no node carries shares the last bit of the last word.  Returns labels[N,W], sel[P,W]."""
    pairs = {}
    for lab in node_label_maps:
        for kv in (lab or {}).items():
            pairs.setdefault(kv, len(pairs))
    W = 1
    while len(pairs) + 1 > 64 * W:
        W *= 2
    absent = 64 * W - 1
    labels = np.zeros((len(node_label_maps), W), np.uint64)
    for n, lab in enumerate(node_label_maps):
        for kv in (lab or {}).items():
            b = pairs[kv]
            labels[n, b // 64] |= np.uint64(1) << np.uint64(b % 64)
    sel = np.zeros((len(pod_selector_maps), W), np.uint64)
    for p, s in enumerate(pod_selector_maps):
        for kv in (s or {}).items():
            b = pairs.get(kv, absent)
            sel[p, b // 64] |= np.uint64(1) << np.uint64(b % 64)
    return labels, sel


def string_list_cases(full, size=lambda s: len(s.encode()) + 1):
    """The three buffer sizes worth checking for a string-list output (entries back to back, each NUL-terminated, -1 for
    an entry that does not fit) whose entries, with room for all, are `full` (None = no entry), and what comes back:
    room for all; no room; room for exactly one shorter entry that follows a longer one, which is skipped."""
    first = next(i for i, s in enumerate(full) if s is not None)
    k = next(i for i, s in enumerate(full) if s is not None and i > first and size(s) < size(full[first]))
    skip = [None] * len(full)
    skip[k] = full[k]
    return [(sum(size(s) for s in full if s is not None), list(full)), (0, [None] * len(full)), (size(full[k]), skip)]
