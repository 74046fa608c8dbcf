"""CPU restatement of ttm_mode's result (include/sparse_b200.h, b2s_ttm_mode), from the coordinates of X's entries.

Shared by tests/test_ttm_mode.py and the benchmark's parity check (tools/bench_configs.py).  Independent of the NumPy
stand-in in _mock_ttm.py: fibers come from np.unique over the other coordinates, each (fiber, r) value is added entry
by entry from +0 in ascending i_mode, and the result's coordinates are built by inserting r at `mode` and sorted with
np.lexsort -- no slot or key formula."""
import numpy as np

from _mttkrp_order import same_bits  # noqa: F401  (re-exported for the callers)


def result(coords, vals, shape, U, mode, dtype):
    """(coordinates (ndim x nnz) in C order, values) of ttm_mode(X, U, mode) for the entries (coords, vals) of X."""
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
