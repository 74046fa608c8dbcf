"""NumPy stand-in for sparse_b200._kernels.masked_spgemm and its helpers -- TEST INFRASTRUCTURE ONLY.

_mock_kernels.install() puts these in place of the real wrappers along with the rest of the kernel layer, so the
host-side logic of masked_matmul runs without a GPU.  masked_spgemm
restates the order of b2s_masked_spgemm (include/sparse_b200.h) entry by entry; `order_contract` is the same
restatement on plain NumPy CSR arrays, shared with the GPU tests and the benchmark's sampled-row check.
"""
from __future__ import annotations

import numpy as np
import torch

from sparse_b200 import _device as D


def _np(x):
    return x.detach().cpu().numpy()


def order_contract(m_ptr, m_cols, m_vals, a_ptr, a_cols, a_vals, bt_ptr, bt_cols, bt_vals, rows=None):
    """Values of mask * (A @ B) at the stored mask entries of `rows` (all rows when None), in stored order:
    c' = ((+0 + a_ik1 * b_k1j) + a_ik2 * b_k2j) + ... over the common k in ascending order, in the dtype of a_vals;
    then v = T(m) * T(c') with T = m_vals.dtype.  Returns (entry positions, values)."""
    Tc, T = a_vals.dtype, m_vals.dtype
    rows = range(len(m_ptr) - 1) if rows is None else rows
    pos, out = [], []
    with np.errstate(all="ignore"):
        for i in rows:
            ak = a_cols[a_ptr[i]:a_ptr[i + 1]]
            av = a_vals[a_ptr[i]:a_ptr[i + 1]]
            for p in range(m_ptr[i], m_ptr[i + 1]):
                j = m_cols[p]
                bk = bt_cols[bt_ptr[j]:bt_ptr[j + 1]]
                bv = bt_vals[bt_ptr[j]:bt_ptr[j + 1]]
                _, ia, ib = np.intersect1d(ak, bk, assume_unique=True, return_indices=True)  # ascending k
                c = Tc.type(0)
                for x, y in zip(av[ia], bv[ib]):
                    c = Tc.type(c + Tc.type(x * y))
                pos.append(p)
                out.append(T.type(m_vals[p] * T.type(c)))
    return np.asarray(pos, dtype=np.int64), np.asarray(out, dtype=T)


def masked_spgemm(m_indptr, m_cols, m_vals, a_indptr, a_cols, a_vals, bt_indptr, bt_cols, bt_vals, M, N, K):
    """Same argument contract as the real wrapper."""
    D.dtype_code(D.np_dtype(a_vals))  # TypeError outside the CUDA dtype matrix, as the real call
    idx = {x.dtype for x in (m_indptr, m_cols, a_indptr, a_cols, bt_indptr, bt_cols)}
    assert len(idx) == 1 and idx <= {torch.int32, torch.int64}, idx
    assert a_vals.dtype == bt_vals.dtype
    _, out = order_contract(*(_np(x) for x in (m_indptr, m_cols, m_vals, a_indptr, a_cols, a_vals, bt_indptr, bt_cols,
                                               bt_vals)))
    return torch.from_numpy(out.astype(D.np_dtype(m_vals), copy=False))


def masked_spgemm_set_stage(cap: int = 0):
    """The staging capacity changes nothing in the results; the mock only validates the argument."""
    assert 0 <= cap <= 512


def _rows_strict(ptr, idx):
    ptr, idx = _np(ptr).astype(np.int64), _np(idx).astype(np.int64)
    d = np.diff(idx)
    inside = np.ones(len(d), dtype=bool)
    inside[ptr[1:-1][(ptr[1:-1] > 0) & (ptr[1:-1] < len(idx))] - 1] = False  # pairs that straddle a row boundary
    return bool(np.all(d[inside] > 0))


def masked_spgemm_sorted(a_indptr, a_cols, M, bt_indptr, bt_cols, N) -> bool:
    ok = True
    if a_indptr is not None and M:
        ok &= _rows_strict(a_indptr, a_cols)
    if bt_indptr is not None and N:
        ok &= _rows_strict(bt_indptr, bt_cols)
    return ok


def keys_member(query, keys):
    return torch.from_numpy(np.isin(_np(query), _np(keys)).astype(np.uint8))
