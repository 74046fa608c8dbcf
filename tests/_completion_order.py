"""CPU restatement of the order of operations of cp_completion_mode (include/sparse_b200.h, b2s_cp_completion_mode).

Shared by tests/test_cp_completion_mode.py, the NumPy stand-in (_mock_completion.py, which takes only `solve` from
here) and the benchmark's parity check (tools/bench_configs.py).  Each operation is a float32 / float64 NumPy array
operation: correctly rounded, and never contracted into an FMA.  The sums of steps 2-3 go row by row through the
mttkrp_mode restatement (_mttkrp_order.row_result); the factorisation and the solves of steps 4-7 are vectorised over
rows."""
import numpy as np

import _mttkrp_order as MO


def slots(R):
    """(r, s) of the upper-triangle accumulators, r <= s, row by row."""
    return np.triu_indices(R)


def khatri_rao(vals, gathered, dtype):
    """(h_e, p_e): h_e = (U_a[i_a] * U_b[i_b]) * ..., p_e = ((v_e * U_a[i_a]) * U_b[i_b]) * ..., the other modes'
    gathered factor rows ascending."""
    dtype = np.dtype(dtype)
    h = None
    with np.errstate(all="ignore"):
        for g in gathered:
            g = np.asarray(g, dtype=dtype)
            h = g if h is None else h * g
    return h, MO.products(vals, gathered, dtype)


def row_system(h, p, start, chunk, dtype):
    """(upper triangle of G_i, b_i) of one row from its entries' h and p in stream order, the first at stream position
    `start`: per chunk ((+0 + x_1) + x_2) + ..., then over the chunks in chunk order."""
    dtype = np.dtype(dtype)
    R = h.shape[1]
    r, s = slots(R)
    with np.errstate(all="ignore"):
        g = h[:, r] * h[:, s]
    both = MO.row_result(np.concatenate([g, p], axis=1), start, chunk, dtype)
    return both[: len(r)], both[len(r):]


def solve(Gu, b, reg, dtype):
    """Steps 4-7 for a stack of rows: Gu (n, R(R+1)/2) the upper triangles, b (n, R).  Rows with a pivot that is not
    positive are NaN."""
    dtype = np.dtype(dtype)
    Gu, b = np.asarray(Gu, dtype), np.asarray(b, dtype)
    n, R = b.shape
    reg = dtype.type(reg)
    r, s = slots(R)
    L = np.zeros((n, R, R), dtype)
    L[:, r, s] = Gu
    L[:, s, r] = Gu
    ok = np.ones(n, dtype=bool)
    with np.errstate(all="ignore"):
        d = np.arange(R)
        L[:, d, d] = L[:, d, d] + reg
        for j in range(R):
            dj = L[:, j, j]  # ((A_jj - L_j0 L_j0) - L_j1 L_j1) - ..., left by the updates of earlier columns
            ok &= dj > 0
            ljj = np.sqrt(dj)
            L[:, j + 1:, j] = L[:, j + 1:, j] / ljj[:, None]
            L[:, j, j] = ljj
            col = L[:, j + 1:, j]
            L[:, j + 1:, j + 1:] = L[:, j + 1:, j + 1:] - col[:, :, None] * col[:, None, :]
        y = b.copy()
        for j in range(R):
            yj = y[:, j] / L[:, j, j]
            y[:, j] = yj
            y[:, j + 1:] = y[:, j + 1:] - L[:, j + 1:, j] * yj[:, None]
        x = y.copy()
        for j in range(R - 1, -1, -1):
            t = y[:, j].copy()
            for k in range(j + 1, R):
                t = t - L[:, k, j] * x[:, k]
            x[:, j] = t / L[:, j, j]
    x[~ok] = np.nan
    return x


def stream(coords, vals, mode):
    """The mode stream: C-order `coords` (N x nnz) and `vals` sorted stably by coordinate `mode`."""
    coords = np.asarray(coords, dtype=np.int64)
    order = np.argsort(coords[mode], kind="stable")
    return coords[:, order], np.asarray(vals)[order]


def systems(coords, vals, factors, mode, rows, chunk, dtype):
    """(Gu (rows, R(R+1)/2), b (rows, R)) for a tensor given by C-order `coords` and `vals`; rows without entries +0."""
    dtype = np.dtype(dtype)
    c, v = stream(coords, vals, mode)
    R = next(np.shape(f)[1] for m, f in enumerate(factors) if m != mode)
    h, p = khatri_rao(v, [np.asarray(factors[m])[c[m]] for m in range(len(factors)) if m != mode], dtype)
    h, p = h.reshape(len(v), R), p.reshape(len(v), R)
    Gu = np.zeros((rows, R * (R + 1) // 2), dtype)
    b = np.zeros((rows, R), dtype)
    bounds = np.searchsorted(c[mode], np.arange(rows + 1))
    for i in range(rows):
        lo, hi = bounds[i], bounds[i + 1]
        if hi > lo:
            Gu[i], b[i] = row_system(h[lo:hi], p[lo:hi], lo, chunk, dtype)
    return Gu, b


def cp_completion_mode(coords, vals, factors, mode, rows, chunk, dtype, reg):
    """The whole result; rows without entries go through the same solve (+0 for reg > 0, NaN for reg = 0)."""
    Gu, b = systems(coords, vals, factors, mode, rows, chunk, dtype)
    return solve(Gu, b, reg, dtype)


same_bits = MO.same_bits
