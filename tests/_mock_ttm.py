"""NumPy stand-in for sparse_b200._kernels.ttm_mode -- TEST INFRASTRUCTURE ONLY.

tests/test_ttm_mode.py puts it in place of the real wrapper for the mock backend (the rest of the kernel layer is
replaced by _mock_kernels.install()), so the host-side logic of ttm_mode runs without a GPU.  It follows the order and
the slot layout of b2s_ttm_mode (include/sparse_b200.h) for all fibers at once; tests/_ttm_order.py restates the
result independently, from the coordinates.
"""
from __future__ import annotations

import numpy as np
import torch

from sparse_b200 import _device as D


def ttm_mode_long_flags(fptr, long_min):
    fp = fptr.detach().numpy().astype(np.int64)
    return torch.from_numpy((np.diff(fp) > long_min).astype(np.uint8))


def ttm_mode(kcoord, vals, fptr, fgroup, gptr, fkey, pkey, long_ids, long_min, U, R, q_ext):
    """Every fiber's running sums over its entries in stream order from +0, written to the slots and keys of the real
    wrapper with the flag y != 0 (the real kernel's two fiber roles give the same bits).  Same argument contract as
    the real wrapper."""
    D.dtype_code(D.np_dtype(vals))  # TypeError outside the CUDA dtype matrix, as the real call
    for c in (kcoord, fptr, fgroup, gptr):
        if c.dtype not in (torch.int32, torch.int64) or c.dtype != kcoord.dtype:
            raise TypeError(f"mock: index arrays must be int32 / int64 of one width, got {c.dtype}")
    assert fkey.dtype == torch.int64 and pkey.dtype == torch.int64 and U.dtype == vals.dtype
    assert int(U.shape[1]) == R
    assert long_ids.dtype == torch.int64
    fp_ = fptr.detach().numpy().astype(np.int64)
    assert np.array_equal(long_ids.detach().numpy(), np.flatnonzero(np.diff(fp_) > long_min))
    k = kcoord.detach().numpy().astype(np.int64)
    fp = fptr.detach().numpy().astype(np.int64)
    v = vals.detach().numpy()
    u = U.detach().numpy()
    nf = len(fp) - 1
    length = np.diff(fp)
    acc = np.zeros((nf, R), dtype=v.dtype)
    with np.errstate(all="ignore"):
        for j in range(int(length.max()) if nf else 0):
            live = np.flatnonzero(length > j)
            e = fp[live] + j
            acc[live] = acc[live] + v[e][:, None] * u[k[e]]
    f = np.arange(nf)
    g = fgroup.detach().numpy().astype(np.int64)
    gp = gptr.detach().numpy().astype(np.int64)
    g0, sg = gp[g], gp[g + 1] - gp[g]
    P, F = pkey.detach().numpy(), fkey.detach().numpy()
    r = np.arange(R)
    slot = (R * g0 + f - g0)[:, None] + r[None, :] * sg[:, None]
    out = np.empty(nf * R, v.dtype)
    keys = np.empty(nf * R, np.int64)
    out[slot] = acc
    keys[slot] = (P[:, None] * R + r[None, :]) * q_ext + (F - P * q_ext)[:, None]
    flags = (out != 0).astype(np.uint8)
    return torch.from_numpy(out), torch.from_numpy(keys), torch.from_numpy(flags)
