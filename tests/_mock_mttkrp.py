"""NumPy stand-in for sparse_b200._kernels.mttkrp_mode -- TEST INFRASTRUCTURE ONLY.

tests/test_mttkrp_mode.py puts it in place of the real wrapper for the mock backend (the rest of the kernel layer is
replaced by _mock_kernels.install()), so the host-side logic of mttkrp_mode runs without a GPU.  It follows the order
of b2s_mttkrp_mode (include/sparse_b200.h) for the whole tensor at once; tests/_mttkrp_order.py restates the same
order row by row, independently.
"""
from __future__ import annotations

import numpy as np
import torch

from sparse_b200 import _device as D
from sparse_b200 import _kernels as Kn


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


def mttkrp_mode(coords, vals, factors, mode, rows, R):
    """Products in ascending mode order, partials per (chunk, row) run in stream order, row results over the chunks
    in chunk order, every sum starting from +0.  Same argument contract as the real wrapper."""
    D.dtype_code(D.np_dtype(vals))  # TypeError outside the CUDA dtype matrix, as the real call
    for c in coords:
        if c.dtype not in (torch.int32, torch.int64):
            raise TypeError(f"mock: mode stream coordinates must be int32 / int64, got {c.dtype}")
    c = [x.detach().numpy().astype(np.int64) for x in coords]
    v = vals.detach().numpy()
    out = np.zeros((rows, R), dtype=v.dtype)
    if len(v) and rows and R:
        p = np.repeat(v[:, None], R, axis=1)
        with np.errstate(all="ignore"):
            for m in range(len(c)):
                if m != mode:
                    p = p * factors[m].detach().numpy()[c[m]]
        out = _chunked_row_sums(p, c[mode], rows)
    return torch.from_numpy(out)
