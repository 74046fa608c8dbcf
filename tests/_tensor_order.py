"""CPU restatement of the order of operations of the sparse-tensor ops (include/sparse_b200.h: b2s_mttkrp_mode,
b2s_ttmc_mode, b2s_tttp, b2s_ttm_mode, b2s_cp_completion_mode), row by row, entry by entry or fiber by fiber.

Shared by the op tests and the benchmark's parity checks (tools/bench_configs.py).  Independent of the NumPy stand-ins
in _mock_tensor.py, which restate the same orders for the whole tensor at once; it imports nothing from them, so a
GPU result that matches it means something.  Each operation is a float32 / float64 NumPy array operation: correctly
rounded, and never contracted into an FMA."""
import numpy as np


def _ordered_sum(x, dtype):
    """((+0 + x[0]) + x[1]) + ... along axis 0 (np.cumsum accumulates in order; `+ 0` turns the -0 an all -0 run
    would leave into the +0 the contract's leading +0 gives)."""
    if len(x) == 0:
        return np.zeros(x.shape[1:], dtype=dtype)
    with np.errstate(all="ignore"):
        return np.cumsum(x, axis=0, dtype=dtype)[-1] + dtype.type(0)


def products(vals, gathered, dtype, kron=False):
    """p_e = ((v_e * U_a[i_a]) * U_b[i_b]) * ...: `gathered` holds the factor rows of the other modes, ascending.
    Khatri-Rao columns (mttkrp_mode: column r of every factor), or with `kron` Kronecker columns (ttmc_mode:
    p_e[col] = ((v_e * U_a[i_a, r_a]) * U_b[i_b, r_b]) * ..., col = ((r_a * R_b + r_b) * R_c + r_c) ...).  With
    `vals` None the product starts from U_a[i_a] (cp_completion_mode's h_e)."""
    dtype = np.dtype(dtype)
    p = None if vals is None else np.asarray(vals, dtype=dtype)[:, None]
    with np.errstate(all="ignore"):
        for g in gathered:
            g = np.asarray(g, dtype=dtype)
            if p is None:
                p = g
            elif kron:
                p = (p[:, :, None] * g[:, None, :]).reshape(len(p), -1)
            else:
                p = p * g
    return p


def row_result(p, start, chunk, dtype):
    """out[i] from the products `p` of row i's entries in stream order, the first at stream position `start`: per chunk
    ((+0 + p_1) + p_2) + ..., then over the chunks in chunk order from +0."""
    dtype = np.dtype(dtype)
    pos = start + np.arange(len(p))
    cuts = np.flatnonzero(np.diff(pos // chunk)) + 1
    partials = [_ordered_sum(piece, dtype) for piece in np.split(p, cuts)] if len(p) else []
    return _ordered_sum(np.array(partials, dtype=dtype).reshape(len(partials), p.shape[1]), dtype)


def _row_sums(coords, vals, factors, mode, rows, chunk, dtype, width, terms):
    """(rows, width) row sums for a tensor given by C-order `coords` (N x nnz) and `vals`: the entries sorted stably by
    coordinate `mode` (the mode stream), each entry's terms = terms(v, gathered factor rows of the other modes,
    ascending), then row_result row by row; rows without entries +0."""
    dtype = np.dtype(dtype)
    coords = np.asarray(coords, dtype=np.int64)
    order = np.argsort(coords[mode], kind="stable")
    c, v = coords[:, order], np.asarray(vals)[order]
    t = terms(v, [np.asarray(factors[m])[c[m]] for m in range(len(factors)) if m != mode]).reshape(len(v), width)
    out = np.zeros((rows, width), dtype=dtype)
    bounds = np.searchsorted(c[mode], np.arange(rows + 1))
    for i in range(rows):
        s, e = bounds[i], bounds[i + 1]
        if e > s:
            out[i] = row_result(t[s:e], s, chunk, dtype)
    return out


def _rank(factors, mode):
    return next(np.shape(f)[1] for m, f in enumerate(factors) if m != mode)


def mttkrp_mode(coords, vals, factors, mode, rows, chunk, dtype):
    """The whole mttkrp_mode result for a tensor given by C-order `coords` (N x nnz) and `vals`."""
    return _row_sums(coords, vals, factors, mode, rows, chunk, dtype, _rank(factors, mode),
                     lambda v, g: products(v, g, dtype))


def ttmc_mode(coords, vals, factors, mode, rows, chunk, dtype):
    """The whole ttmc_mode result for a tensor given by C-order `coords` (N x nnz) and `vals`."""
    W = int(np.prod([np.shape(factors[m])[1] for m in range(len(factors)) if m != mode]))
    return _row_sums(coords, vals, factors, mode, rows, chunk, dtype, W, lambda v, g: products(v, g, dtype, kron=True))


def sampled_rows_exact(got, coords, vals, U, mode, rows, chunk, kron):
    """Whether rows `rows` of the device result `got` of mttkrp_mode (or ttmc_mode with `kron`) equal this restatement
    bit for bit.  `coords` (N x nnz) and `vals` are the tensor's device entries in C order, so a row's entries are in
    stream order, the first at the stream position that counts the entries of the rows before it."""
    import torch

    exact = True
    for i in rows:
        i = int(i)
        sel = torch.nonzero(coords[mode] == i).reshape(-1)
        start = int((coords[mode] < i).sum())
        c = coords[:, sel]
        v = vals[sel].cpu().numpy()
        p = products(v, [U[m][c[m]].cpu().numpy() for m in range(len(U)) if m != mode], v.dtype, kron)
        exact &= same_bits(got[i].cpu().numpy(), row_result(p, start, chunk, v.dtype))
    return bool(exact)


def values(coords, vals, factors, dtype):
    """tttp's z_e for the entries given by `coords` (N x nnz, any order) and `vals`:
    q_r = ((U_0[i_0, r] * U_1[i_1, r]) * ...) in ascending mode order, m = ((+0 + q_0) + q_1) + ..., z = v * m.
    The columns are added one at a time in an explicit loop from +0."""
    dtype = np.dtype(dtype)
    coords = np.asarray(coords, dtype=np.int64)
    nnz = coords.shape[1]
    R = np.shape(factors[0])[1]
    m = np.zeros(nnz, dtype=dtype)
    with np.errstate(all="ignore"):
        for r in range(R):
            q = np.asarray(factors[0], dtype=dtype)[coords[0], r]
            for k in range(1, len(factors)):
                q = q * np.asarray(factors[k], dtype=dtype)[coords[k], r]
            m = m + q
        return np.asarray(vals, dtype=dtype) * m


def result(coords, vals, shape, U, mode, dtype):
    """(coordinates (ndim x nnz) in C order, values) of ttm_mode(X, U, mode) for the entries (coords, vals) of X.

    Fibers come from np.unique over the other coordinates, each (fiber, r) value is added entry by entry from +0 in
    ascending i_mode, and the result's coordinates are built by inserting r at `mode` and sorted with np.lexsort -- no
    slot or key formula."""
    dtype = np.dtype(dtype)
    coords = np.asarray(coords, dtype=np.int64)
    vals = np.asarray(vals, dtype=dtype)
    U = np.asarray(U)
    ttv = U.ndim == 1
    U = np.asarray(U.reshape(-1, 1) if ttv else U, dtype=dtype)
    N, R = len(shape), U.shape[1]
    others = [m for m in range(N) if m != mode]
    # ascending i_mode inside each fiber
    order = np.lexsort([coords[mode]] + [coords[m] for m in reversed(others)])
    c, v = coords[:, order], vals[order]
    fib, inv = np.unique(c[others].T, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    nf = len(fib)
    y = np.zeros((nf, R), dtype=dtype)
    with np.errstate(all="ignore"):
        for e in range(len(v)):  # stream order: each fiber's entries in ascending i_mode
            y[inv[e]] = y[inv[e]] + v[e] * U[c[mode, e]]
    rows = []
    for pos, m in enumerate(others):
        rows.append(np.repeat(fib[:, pos], R))
    if not ttv:
        rows.insert(mode, np.tile(np.arange(R), nf))
    out = np.stack(rows) if rows else np.zeros((0, nf * R), np.int64)
    yv = y.reshape(-1)
    keep = yv != 0
    out, yv = out[:, keep], yv[keep]
    srt = np.lexsort(out[::-1]) if len(out) else np.arange(len(yv))
    return out[:, srt], yv[srt]


# cp_completion_mode: the sums of steps 2-3 go row by row through row_result (so b_i is mttkrp_mode's row bit for
# bit); the factorisation and the solves of steps 4-7 are vectorised over rows.
def slots(R):
    """(r, s) of the upper-triangle accumulators, r <= s, row by row."""
    return np.triu_indices(R)


def _system_terms(h, p):
    """Each entry's Gram terms h_e[r] * h_e[s] over the slots, then its right-hand-side terms p_e."""
    r, s = slots(h.shape[1])
    with np.errstate(all="ignore"):
        return np.concatenate([h[:, r] * h[:, s], p], axis=1)


def row_system(h, p, start, chunk, dtype):
    """(upper triangle of G_i, b_i) of one row from its entries' h and p in stream order, the first at stream position
    `start`: per chunk ((+0 + x_1) + x_2) + ..., then over the chunks in chunk order."""
    both = row_result(_system_terms(h, p), start, chunk, dtype)
    n = len(both) - h.shape[1]
    return both[:n], both[n:]


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


def systems(coords, vals, factors, mode, rows, chunk, dtype):
    """(Gu (rows, R(R+1)/2), b (rows, R)) for a tensor given by C-order `coords` and `vals`; rows without entries +0.
    h_e = (U_a[i_a] * U_b[i_b]) * ..., p_e = ((v_e * U_a[i_a]) * U_b[i_b]) * ..., the other modes ascending."""
    R = _rank(factors, mode)
    n = R * (R + 1) // 2
    both = _row_sums(coords, vals, factors, mode, rows, chunk, dtype, n + R,
                     lambda v, g: _system_terms(products(None, g, dtype), products(v, g, dtype)))
    return both[:, :n], both[:, n:]


def cp_completion_mode(coords, vals, factors, mode, rows, chunk, dtype, reg):
    """The whole result; rows without entries go through the same solve (+0 for reg > 0, NaN for reg = 0)."""
    Gu, b = systems(coords, vals, factors, mode, rows, chunk, dtype)
    return solve(Gu, b, reg, dtype)


def same_bits(got, want):
    """Bit-equal, except that any NaN matches any NaN (the device returns the canonical NaN, NumPy keeps payloads)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape or got.dtype != want.dtype:
        return False
    gn, wn = np.isnan(got), np.isnan(want)
    if not np.array_equal(gn, wn):
        return False
    w = {4: np.uint32, 8: np.uint64}[got.dtype.itemsize]
    return bool(np.array_equal(got[~gn].view(w), want[~wn].view(w)))
