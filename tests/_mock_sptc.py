"""NumPy stand-ins for sparse_b200._kernels.sptc_join / sptc_keys -- TEST INFRASTRUCTURE ONLY.

tests/test_sptc.py puts them in place of the real wrappers while the NumPy mock of the kernel layer is installed, so
sptc's host-side logic (axes, compressed rows, caches, index widths, limits) runs without a GPU.  They follow
include/sparse_b200.h (b2s_sptc_join, b2s_sptc_keys) with the argument contracts of the real wrappers.
"""
from __future__ import annotations

import numpy as np
import torch


def _i64(t, what):
    if t.dtype != torch.int64:
        raise TypeError(f"mock: {what} must be int64, got {t.dtype}")
    return t.detach().numpy()


def sptc_join(query, keys, idx_dtype=np.int64):
    q, s = _i64(query, "query"), _i64(keys, "keys")
    if np.dtype(idx_dtype) not in (np.dtype(np.int32), np.dtype(np.int64)):
        raise TypeError(f"mock: idx_dtype must be int32 / int64, got {np.dtype(idx_dtype)}")
    assert np.dtype(idx_dtype) == np.int64 or len(s) < 2**31 - 1
    assert len(s) < 2 or (np.diff(s) > 0).all(), "the set must be ascending without duplicates"
    pos = np.searchsorted(s, q, side="left")
    hit = pos < len(s)
    hit[hit] = s[pos[hit]] == q[hit]
    return torch.from_numpy(np.where(hit, pos, len(s)).astype(idx_dtype))


def sptc_keys(rows, cols, xrows, ycols, g_ext):
    r, c = _i64(rows, "rows"), _i64(cols, "cols")
    assert g_ext >= 1
    return torch.from_numpy(_i64(xrows, "xrows")[r] * np.int64(g_ext) + _i64(ycols, "ycols")[c])


STAND_INS = {"sptc_join": sptc_join, "sptc_keys": sptc_keys}
