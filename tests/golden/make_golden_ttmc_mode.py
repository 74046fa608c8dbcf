#!/usr/bin/env python
"""Generate tests/golden/ttmc_mode_api.npz from the REFERENCE itself: mode-n TTMc as the reference computes it, the
unfused broadcast expression

    sum(X[..., None, None, ...] * U_a[..] * U_b[..] * ..., axis = every axis of X but n)

with U_m on axis m and on the trailing axis of its rank, giving a (I_n, R_a, R_b, ...) result.  Orders 3 and 4, every
mode, float32 and float64, with a different rank on every mode, so that a column-order mistake cannot pass.  Uses the
helpers of make_golden.py (same reference import, same fixture layout) and writes only this one file:

    SPARSE_REFERENCE=<checkout> python tests/golden/make_golden_ttmc_mode.py
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import Book, enc, rand_sparse, sparse  # noqa: E402


def gen_ttmc_mode():
    bk = Book("ttmc_mode_api")
    rng = np.random.default_rng(29)
    for dt in ("float32", "float64"):
        for shape, ranks in (((7, 6, 5), (3, 4, 2)), ((5, 4, 6, 3), (2, 3, 4, 5))):
            N = len(shape)
            X = rand_sparse(rng, shape, 0.25, dt)
            U = [(rng.random((s, r)) - 0.5).astype(dt) for s, r in zip(shape, ranks)]
            for mode in range(N):
                others = [m for m in range(N) if m != mode]
                t = X[(Ellipsis,) + (None,) * len(others)]
                for k, m in enumerate(others):
                    idx = [None] * (N + len(others))
                    idx[m] = idx[N + k] = slice(None)
                    t = t * U[m][tuple(idx)]
                r = sparse.sum(t, axis=tuple(others))
                bk.add({"op": "ttmc_mode", "dtype": dt, "order": N, "mode": mode}, **enc("X_", X),
                       **{f"U{m}": U[m] for m in range(N)}, **enc("out_", r))
    bk.save()


if __name__ == "__main__":
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen_ttmc_mode()
