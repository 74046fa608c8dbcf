"""NumPy stand-in for sparse_b200._kernels.tttp -- TEST INFRASTRUCTURE ONLY.

tests/test_tttp.py puts it in place of the real wrapper for the mock backend (the rest of the kernel layer is replaced
by _mock_kernels.install()), so the host-side logic of tttp runs without a GPU.  It follows the order of b2s_tttp
(include/sparse_b200.h) for all entries at once; tests/_tttp_order.py restates the same order entry by entry,
independently.
"""
from __future__ import annotations

import numpy as np
import torch

from sparse_b200 import _device as D


def tttp(coords, vals, factors, R):
    """Column products in ascending mode order, their sum in ascending r from +0, then one multiply by the value.
    Same argument contract as the real wrapper."""
    D.dtype_code(D.np_dtype(vals))  # TypeError outside the CUDA dtype matrix, as the real call
    for c in coords:
        if c.dtype not in (torch.int32, torch.int64) or c.dtype != coords[0].dtype:
            raise TypeError(f"mock: coordinates must be int32 / int64 of one width, got {c.dtype}")
    assert len(factors) == len(coords)
    c = [x.detach().numpy().astype(np.int64) for x in coords]
    v = vals.detach().numpy()
    with np.errstate(all="ignore"):
        q = np.ones((len(v), R), dtype=v.dtype)
        for m, f in enumerate(factors):
            assert f.dtype == vals.dtype and int(f.shape[1]) == R
            g = f.detach().numpy()[c[m]]
            q = g if m == 0 else q * g
        # np.cumsum adds in order; `+ 0` turns the -0 that an all -0 row leaves into the +0 of the leading +0
        m_ = np.cumsum(q, axis=1, dtype=v.dtype)[:, -1] + v.dtype.type(0) if R else np.zeros(len(v), v.dtype)
        return torch.from_numpy(np.ascontiguousarray(v * m_))
