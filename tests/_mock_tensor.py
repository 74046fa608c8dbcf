"""NumPy stand-ins for the sparse-tensor wrappers of sparse_b200._kernels (mttkrp_mode, ttmc_mode, tttp, ttm_mode with
ttm_mode_long_flags, cp_completion_mode) -- TEST INFRASTRUCTURE ONLY.

_mock_kernels.install() puts them in place of the real wrappers along with the rest of the kernel layer, so the
host-side logic of these ops runs without a GPU.  Each follows the order of its b2s_* entry point
(include/sparse_b200.h) for the whole tensor at once, vectorised over entries, rows and fibers; tests/_tensor_order.py
restates the same orders row by row, independently.  The one thing taken from there is the completion's factorisation
and solves (`solve`).
"""
from __future__ import annotations

import numpy as np
import torch

from _tensor_order import slots, solve
from sparse_b200 import _device as D
from sparse_b200 import _kernels as Kn


def _check(vals, index):
    """What the real wrappers refuse and NumPy would not: values outside the CUDA dtype matrix (TypeError, as the real
    call) and index arrays that are not int32 / int64 of one width."""
    D.dtype_code(D.np_dtype(vals))
    for c in index:
        if c.dtype not in (torch.int32, torch.int64) or c.dtype != index[0].dtype:
            raise TypeError(f"mock: index arrays must be int32 / int64 of one width, got {c.dtype}")


def _products(v, gathered, kron=False):
    """((v_e * f_a) * f_b) * ... over the gathered factor rows, ascending: Khatri-Rao columns, or with `kron` Kronecker
    columns in C order.  With `v` None the product starts from f_a."""
    p = None if v is None else v[:, None]
    with np.errstate(all="ignore"):
        for f in gathered:
            if p is None:
                p = f
            elif kron:
                p = (p[:, :, None] * f[:, None, :]).reshape(len(f), -1)
            else:
                p = p * f
    return p


def _ordered_sums(x, starts, lens):
    """Row s of the result is ((+0 + x[starts[s]]) + x[starts[s] + 1]) + ... over lens[s] rows of x, in order."""
    acc = np.zeros((len(starts),) + x.shape[1:], dtype=x.dtype)
    with np.errstate(all="ignore"):
        for k in range(int(lens.max()) if len(lens) else 0):
            live = lens > k
            acc[live] = acc[live] + x[starts[live] + k]
    return acc


def _chunked_row_sums(p, row, rows):
    """(rows, ...) result of the products p (one per stream entry, rows of index `row`): partials per (chunk, row) run
    in stream order, row results over the chunks in chunk order, every sum starting from +0, rows without entries +0."""
    out = np.zeros((rows,) + p.shape[1:], dtype=p.dtype)
    ch = Kn.mttkrp_mode_chunk()  # the library's constant (needs no device)
    pos = np.arange(len(row))
    head = np.ones(len(row), dtype=bool)
    head[1:] = (row[1:] != row[:-1]) | (pos[1:] % ch == 0)
    starts = np.flatnonzero(head)
    partial = _ordered_sums(p, starts, np.diff(np.append(starts, len(row))))
    prow = row[starts]
    rhead = np.ones(len(starts), dtype=bool)
    rhead[1:] = prow[1:] != prow[:-1]
    rstarts = np.flatnonzero(rhead)
    out[prow[rstarts]] = _ordered_sums(partial, rstarts, np.diff(np.append(rstarts, len(starts))))
    return out


def _stream(coords, vals, factors, mode):
    """(coordinates as int64 arrays, values, the other modes' gathered factor rows ascending) of a mode stream."""
    c = [x.detach().numpy().astype(np.int64) for x in coords]
    return c, vals.detach().numpy(), [factors[m].detach().numpy()[c[m]] for m in range(len(c)) if m != mode]


def mttkrp_mode(coords, vals, factors, mode, rows, R):
    """Products in ascending mode order, partials per (chunk, row) run in stream order, row results over the chunks
    in chunk order, every sum starting from +0.  Same argument contract as the real wrapper."""
    _check(vals, coords)
    c, v, g = _stream(coords, vals, factors, mode)
    if not (len(v) and rows and R):
        return torch.from_numpy(np.zeros((rows, R), dtype=v.dtype))
    return torch.from_numpy(_chunked_row_sums(_products(v, g), c[mode], rows))


def ttmc_mode(coords, vals, factors, mode, rows, ranks):
    """Kronecker products in ascending mode order (C-order columns), then mttkrp_mode's chunked row sums.  Same
    argument contract as the real wrapper."""
    _check(vals, coords)
    W = int(np.prod([int(ranks[m]) for m in range(len(coords)) if m != mode]))
    c, v, g = _stream(coords, vals, factors, mode)
    if not (len(v) and rows and W):
        return torch.from_numpy(np.zeros((rows, W), dtype=v.dtype))
    return torch.from_numpy(_chunked_row_sums(_products(v, g, kron=True), c[mode], rows))


def tttp(coords, vals, factors, R):
    """Column products in ascending mode order, their sum in ascending r from +0, then one multiply by the value.
    Same argument contract as the real wrapper."""
    _check(vals, coords)
    assert len(factors) == len(coords)
    for f in factors:
        assert f.dtype == vals.dtype and int(f.shape[1]) == R
    _, v, g = _stream(coords, vals, factors, None)
    with np.errstate(all="ignore"):
        q = _products(None, g)
        # np.cumsum adds in order; `+ 0` turns the -0 that an all -0 row leaves into the +0 of the leading +0
        m_ = np.cumsum(q, axis=1, dtype=v.dtype)[:, -1] + v.dtype.type(0) if R else np.zeros(len(v), v.dtype)
        return torch.from_numpy(np.ascontiguousarray(v * m_))


def ttm_mode_long_flags(fptr, long_min):
    fp = fptr.detach().numpy().astype(np.int64)
    return torch.from_numpy((np.diff(fp) > long_min).astype(np.uint8))


def ttm_mode(kcoord, vals, fptr, fgroup, gptr, fkey, pkey, long_ids, long_min, U, R, q_ext):
    """Every fiber's running sums over its entries in stream order from +0, written to the slots and keys of the real
    wrapper with the flag y != 0 (the real kernel's two fiber roles give the same bits).  Same argument contract as
    the real wrapper."""
    _check(vals, (kcoord, fptr, fgroup, gptr))
    assert fkey.dtype == torch.int64 and pkey.dtype == torch.int64 and U.dtype == vals.dtype
    assert int(U.shape[1]) == R
    assert long_ids.dtype == torch.int64
    fp = fptr.detach().numpy().astype(np.int64)
    assert np.array_equal(long_ids.detach().numpy(), np.flatnonzero(np.diff(fp) > long_min))
    k = kcoord.detach().numpy().astype(np.int64)
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


def cp_completion_mode(coords, vals, factors, mode, rows, R, reg):
    """Every entry's Gram and right-hand-side terms at once, summed with mttkrp_mode's chunked row sums; the
    factorisation and solves are the restatement's.  Same argument contract as the real wrapper."""
    _check(vals, coords)
    assert 0 < R <= Kn.cp_completion_max_rank()
    c, v, g = _stream(coords, vals, factors, mode)
    for f in g:
        assert f.dtype == v.dtype and f.shape[1] == R
    h, p = _products(None, g), _products(v, g)
    r, s = slots(R)
    with np.errstate(all="ignore"):
        terms = np.concatenate([h[:, r] * h[:, s], p], axis=1)
    sums = _chunked_row_sums(terms, c[mode], rows)
    return torch.from_numpy(np.ascontiguousarray(solve(sums[:, : len(r)], sums[:, len(r):], reg, v.dtype)))
