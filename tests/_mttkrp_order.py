"""CPU restatement of the order of operations of mttkrp_mode (include/sparse_b200.h, b2s_mttkrp_mode), row by row.

Shared by tests/test_mttkrp_mode.py and the benchmark's parity check (tools/bench_configs.py).  Independent of the
NumPy stand-in in _mock_mttkrp.py, which restates the same order for the whole tensor at once."""
import numpy as np


def _ordered_sum(x, dtype):
    """((+0 + x[0]) + x[1]) + ... along axis 0 (np.cumsum accumulates in order; `+ 0` turns the -0 an all -0 run
    would leave into the +0 the contract's leading +0 gives)."""
    if len(x) == 0:
        return np.zeros(x.shape[1:], dtype=dtype)
    with np.errstate(all="ignore"):
        return np.cumsum(x, axis=0, dtype=dtype)[-1] + dtype.type(0)


def products(vals, gathered, dtype):
    """p_e = (((v_e * U_a[i_a]) * U_b[i_b]) * ...): `gathered` holds the factor rows of the other modes, ascending."""
    dtype = np.dtype(dtype)
    p = np.asarray(vals, dtype=dtype)[:, None]
    with np.errstate(all="ignore"):
        for g in gathered:
            p = p * np.asarray(g, dtype=dtype)
    return p


def row_result(p, start, chunk, dtype):
    """out[i] from the products `p` of row i's entries in stream order, the first at stream position `start`."""
    dtype = np.dtype(dtype)
    pos = start + np.arange(len(p))
    cuts = np.flatnonzero(np.diff(pos // chunk)) + 1
    partials = [_ordered_sum(piece, dtype) for piece in np.split(p, cuts)] if len(p) else []
    return _ordered_sum(np.array(partials, dtype=dtype).reshape(len(partials), p.shape[1]), dtype)


def mttkrp_mode(coords, vals, factors, mode, rows, chunk, dtype):
    """The whole result for a tensor given by C-order `coords` (N x nnz) and `vals`."""
    dtype = np.dtype(dtype)
    coords = np.asarray(coords, dtype=np.int64)
    order = np.argsort(coords[mode], kind="stable")
    c, v = coords[:, order], np.asarray(vals)[order]
    R = next(np.shape(f)[1] for m, f in enumerate(factors) if m != mode)
    p = products(v, [np.asarray(factors[m])[c[m]] for m in range(len(factors)) if m != mode], dtype)
    p = p.reshape(len(v), R)
    out = np.zeros((rows, R), dtype=dtype)
    bounds = np.searchsorted(c[mode], np.arange(rows + 1))
    for i in range(rows):
        s, e = bounds[i], bounds[i + 1]
        if e > s:
            out[i] = row_result(p[s:e], s, chunk, dtype)
    return out


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
