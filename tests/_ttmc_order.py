"""CPU restatement of the order of operations of ttmc_mode (include/sparse_b200.h, b2s_ttmc_mode), row by row.

Shared by tests/test_ttmc_mode.py and the benchmark's parity check (tools/bench_configs.py).  The products differ from
mttkrp_mode's (Kronecker instead of Khatri-Rao columns); the per-chunk partials and the row sums over chunks are the
same, so they come from tests/_mttkrp_order.py.  Independent of the NumPy stand-in in _mock_ttmc.py."""
import numpy as np

from _mttkrp_order import row_result, same_bits  # noqa: F401  (re-exported for the callers)


def products(vals, gathered, dtype):
    """p_e[col] = ((v_e * U_a[i_a, r_a]) * U_b[i_b, r_b]) * ..., col = ((r_a * R_b + r_b) * R_c + r_c) ...:
    `gathered` holds the factor rows of the other modes, ascending."""
    dtype = np.dtype(dtype)
    p = np.asarray(vals, dtype=dtype)[:, None]
    with np.errstate(all="ignore"):
        for g in gathered:
            g = np.asarray(g, dtype=dtype)
            p = (p[:, :, None] * g[:, None, :]).reshape(len(p), -1)
    return p


def ttmc_mode(coords, vals, factors, mode, rows, chunk, dtype):
    """The whole result for a tensor given by C-order `coords` (N x nnz) and `vals`."""
    dtype = np.dtype(dtype)
    coords = np.asarray(coords, dtype=np.int64)
    order = np.argsort(coords[mode], kind="stable")
    c, v = coords[:, order], np.asarray(vals)[order]
    others = [m for m in range(len(factors)) if m != mode]
    W = int(np.prod([np.shape(factors[m])[1] for m in others]))
    p = products(v, [np.asarray(factors[m])[c[m]] for m in others], dtype).reshape(len(v), W)
    out = np.zeros((rows, W), dtype=dtype)
    bounds = np.searchsorted(c[mode], np.arange(rows + 1))
    for i in range(rows):
        s, e = bounds[i], bounds[i + 1]
        if e > s:
            out[i] = row_result(p[s:e], s, chunk, dtype)
    return out
