"""NumPy stand-in for sparse_b200._kernels.cp_apr_phi_mode -- TEST INFRASTRUCTURE ONLY.

tests/test_cp_apr_phi_mode.py puts it in place of the real wrapper while the NumPy mock of the kernel layer is
installed, so the op's host-side logic runs without a GPU.  It follows the order of b2s_cp_apr_phi_mode
(include/sparse_b200.h) for the whole tensor at once, with the helpers of the other sparse-tensor stand-ins in
_mock_tensor.py: tttp's model values first, then the ratios, then mttkrp_mode's products and chunked row sums.
tests/_cp_apr_order.py restates the same order row by row, independently.
"""
from __future__ import annotations

import numpy as np
import torch

from _mock_tensor import _check, _chunked_row_sums, _products, _stream
from sparse_b200 import _kernels as Kn


def cp_apr_phi_mode(coords, vals, factors, mode, rows, R, eps):
    """The model m over every factor (tttp's order), d = eps where m < eps (NaN stays NaN), w = v / d, then
    mttkrp_mode's products of w and chunked row sums.  Same argument contract as the real wrapper."""
    _check(vals, coords)
    assert 0 < R <= Kn.cp_apr_phi_max_rank() and len(factors) == len(coords)
    for f in factors:
        assert f.dtype == vals.dtype and int(f.shape[1]) == R
    c, v, g = _stream(coords, vals, factors, None)
    e = v.dtype.type(eps)
    with np.errstate(all="ignore"):
        # np.cumsum adds in order; `+ 0` turns the -0 an all -0 row leaves into the +0 of the leading +0
        m_ = np.cumsum(_products(None, g), axis=1, dtype=v.dtype)[:, -1] + v.dtype.type(0)
        w = v / np.where(m_ < e, e, m_)
    p = _products(w, [g[m] for m in range(len(g)) if m != mode])
    return torch.from_numpy(_chunked_row_sums(p, c[mode], rows))
