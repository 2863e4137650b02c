"""H100-native pod-to-node scheduling core — Python face of the C ABI in include/ksched.h.

The product is libksched.so (hand-written sm_90a CUDA kernels + a C ABI + a C++ host layer that mirrors
the reference's check_node_validity / select_node_for_pod / reconcile surface).  This package only binds
it with ctypes for tests and bench.py.  There is NO CPU fallback: importing works without a GPU (so the
symbol table can be checked), but every compute entry point returns KS_ERR_NO_DEVICE without an H100, and a
missing libksched.so raises at import time.
"""
from ._capi import (  # noqa: F401
    KS_OK, KS_MEM_HOST, KS_MEM_DEVICE, KS_SCORE_LEFTOVER, KS_SCORE_LEAST_ALLOCATED, KS_SCORE_MOST_ALLOCATED,
    KS_SCORE_LEAST_BALANCED,
    KS_SELECT_AUTO, KS_SELECT_FORCE_DIRECT, KS_SELECT_FORCE_BITPAR, KS_SELECT_TIMING, KS_SELECT_NO_GRAPH,
    KS_CELL_OK, KS_CELL_NOT_ENOUGH_RESOURCES, KS_CELL_NODE_SELECTOR_MISMATCH,
    KsError, lib, LIB_PATH, declared_symbols, mask_row_bytes, mask_row_bytes_aligned, device_count, launch_count,
)
from . import _capi as capi  # noqa: F401
from .snapshot import Snapshot, SelectResult, Stream  # noqa: F401
from . import synth, objects, host, multigpu  # noqa: F401
