"""NumPy stand-in for sparse_b200._kernels.ttmc_mode -- TEST INFRASTRUCTURE ONLY.

tests/test_ttmc_mode.py puts it in place of the real wrapper for the mock backend (the rest of the kernel layer is
replaced by _mock_kernels.install()), so the host-side logic of ttmc_mode runs without a GPU.  It follows the order of
b2s_ttmc_mode (include/sparse_b200.h) for the whole tensor at once; tests/_ttmc_order.py restates the same order row by
row, independently.
"""
from __future__ import annotations

import numpy as np
import torch

from _mock_mttkrp import _chunked_row_sums
from sparse_b200 import _device as D


def ttmc_mode(coords, vals, factors, mode, rows, ranks):
    """Kronecker products in ascending mode order (C-order columns), partials per (chunk, row) run in stream order, row
    results over the chunks in chunk order, every sum starting from +0.  Same argument contract as the real wrapper."""
    D.dtype_code(D.np_dtype(vals))  # TypeError outside the CUDA dtype matrix, as the real call
    for c in coords:
        if c.dtype not in (torch.int32, torch.int64):
            raise TypeError(f"mock: mode stream coordinates must be int32 / int64, got {c.dtype}")
    W = 1
    for m in range(len(coords)):
        if m != mode:
            W *= int(ranks[m])
    c = [x.detach().numpy().astype(np.int64) for x in coords]
    v = vals.detach().numpy()
    out = np.zeros((rows, W), dtype=v.dtype)
    if len(v) and rows and W:
        p = v[:, None]
        with np.errstate(all="ignore"):
            for m in range(len(c)):
                if m != mode:
                    f = factors[m].detach().numpy()[c[m]]
                    p = (p[:, :, None] * f[:, None, :]).reshape(len(v), -1)
        out = _chunked_row_sums(p, c[mode], rows)
    return torch.from_numpy(out)
