"""CPU restatement of the order of operations of tttp (include/sparse_b200.h, b2s_tttp), entry by entry.

Shared by tests/test_tttp.py and the benchmark's parity check (tools/bench_configs.py).  Independent of the NumPy
stand-in in _mock_tttp.py: this one adds the columns one at a time in an explicit loop from +0."""
import numpy as np

from _mttkrp_order import same_bits  # noqa: F401  (re-exported for the callers)


def values(coords, vals, factors, dtype):
    """z_e for the entries given by `coords` (N x nnz, any order) and `vals`:
    q_r = ((U_0[i_0, r] * U_1[i_1, r]) * ...) in ascending mode order, m = ((+0 + q_0) + q_1) + ..., z = v * m."""
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
