"""NumPy stand-in for sparse_b200._kernels.cp_completion_mode -- TEST INFRASTRUCTURE ONLY.

tests/test_cp_completion_mode.py puts it in place of the real wrapper for the mock backend (the rest of the kernel
layer is replaced by _mock_kernels.install()), so the host-side logic of cp_completion_mode runs without a GPU.  It
forms every entry's Gram and right-hand-side terms at once and sums them with the mttkrp_mode stand-in's chunked row
sums; the factorisation and solves are the restatement's (tests/_completion_order.py).
"""
from __future__ import annotations

import numpy as np
import torch

import _completion_order as CO
from _mock_mttkrp import _chunked_row_sums
from sparse_b200 import _device as D
from sparse_b200 import _kernels as Kn


def cp_completion_mode(coords, vals, factors, mode, rows, R, reg):
    """Same argument contract as the real wrapper."""
    D.dtype_code(D.np_dtype(vals))  # TypeError outside the CUDA dtype matrix, as the real call
    for c in coords:
        if c.dtype not in (torch.int32, torch.int64) or c.dtype != coords[0].dtype:
            raise TypeError(f"mock: mode stream coordinates must be int32 / int64 of one width, got {c.dtype}")
    assert 0 < R <= Kn.cp_completion_max_rank()
    c = [x.detach().numpy().astype(np.int64) for x in coords]
    v = vals.detach().numpy()
    dt = v.dtype
    h = p = None
    with np.errstate(all="ignore"):
        for m in range(len(c)):
            if m == mode:
                continue
            f = factors[m].detach().numpy()[c[m]]
            assert f.dtype == dt and f.shape[1] == R
            h = f if h is None else h * f
            p = v[:, None] * f if p is None else p * f
        r, s = CO.slots(R)
        terms = np.concatenate([h[:, r] * h[:, s], p * dt.type(1)], axis=1)
    sums = _chunked_row_sums(terms, c[mode], rows)
    return torch.from_numpy(np.ascontiguousarray(CO.solve(sums[:, : len(r)], sums[:, len(r):], reg, dt)))
