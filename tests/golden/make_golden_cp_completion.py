#!/usr/bin/env python
"""Generate tests/golden/cp_completion_api.npz from the REFERENCE itself: the per-row Gram matrices and right-hand
sides of CP completion's ALS update, as the reference computes them with its unfused broadcast expressions (mode n of
an order-3 tensor, the other modes a < b):

    G = sum(P[..., None, None] * U_a[..., :, None] * U_a[..., None, :] * U_b[..., :, None] * U_b[..., None, :],
            axis=(a, b))                                    # P: X's pattern with ones
    b = sum(X[..., None] * U_a[..., :] * U_b[..., :], axis=(a, b))

with U_m on axis m and the rank(s) on the trailing axes.  Every product and sum is evaluated in float64 (the inputs
are float32 or float64 values), and the test solves (G_i + reg I) x = b_i in float64 against cp_completion_mode.
Orders 3 and 4, every mode.  Uses the helpers of make_golden.py (same reference import, same fixture layout) and
writes only this one file:

    SPARSE_REFERENCE=<checkout> python tests/golden/make_golden_cp_completion.py
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import Book, enc, rand_sparse, sparse  # noqa: E402


def factor_on(u, m, N, rank_axis, n_rank):
    """u (I_m, R) as a broadcast operand of N + n_rank dimensions: I_m on axis m, R on axis N + rank_axis."""
    idx = [None] * (N + n_rank)
    idx[m] = slice(None)
    idx[N + rank_axis] = slice(None)
    return u[tuple(idx)]


def gen():
    bk = Book("cp_completion_api")
    rng = np.random.default_rng(47)
    for dt in ("float32", "float64"):
        for shape, R in (((7, 6, 5), 4), ((5, 4, 6, 3), 3), ((9, 8, 7), 1)):
            N = len(shape)
            X = rand_sparse(rng, shape, 0.3, dt)
            U = [(rng.random((s, R)) - 0.5).astype(dt) for s in shape]
            X64 = X.astype(np.float64)
            P = sparse.COO(X.coords, np.ones(X.nnz), shape=X.shape)
            U64 = [u.astype(np.float64) for u in U]
            for mode in range(N):
                others = tuple(m for m in range(N) if m != mode)
                g = P[(Ellipsis, None, None)]
                for m in others:
                    g = g * factor_on(U64[m], m, N, 0, 2) * factor_on(U64[m], m, N, 1, 2)
                G = sparse.sum(g, axis=others)
                t = X64[(Ellipsis, None)]
                for m in others:
                    t = t * factor_on(U64[m], m, N, 0, 1)
                b = sparse.sum(t, axis=others)
                bk.add({"op": "cp_completion_mode", "dtype": dt, "order": N, "R": R, "mode": mode}, **enc("X_", X),
                       **{f"U{m}": U[m] for m in range(N)}, **enc("G_", G), **enc("b_", b))
    bk.save()


if __name__ == "__main__":
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen()
