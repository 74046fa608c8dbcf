#!/usr/bin/env python
"""Generate tests/golden/tttp_api.npz from the REFERENCE itself: a sparse tensor times a CP model at its stored entries,
as the reference computes it, the unfused broadcast expression

    sum(X[..., None] * U_0[:, None, ..., None, :] * U_1[None, :, ..., None, :] * ..., axis=-1)

with U_m on axis m and the rank on the trailing axis, giving a result with X's pattern.  Orders 3 and 4, float32 and
float64, signed factors (so some model values are negative and some products cancel).  Uses the helpers of
make_golden.py (same reference import, same fixture layout) and writes only this one file:

    SPARSE_REFERENCE=<checkout> python tests/golden/make_golden_tttp.py
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import Book, enc, rand_sparse, sparse  # noqa: E402


def gen_tttp():
    bk = Book("tttp_api")
    rng = np.random.default_rng(31)
    for dt in ("float32", "float64"):
        for shape, R in (((7, 6, 5), 4), ((5, 4, 6, 3), 6), ((9, 8, 7), 1)):
            N = len(shape)
            X = rand_sparse(rng, shape, 0.3, dt)
            U = [(rng.random((s, R)) - 0.5).astype(dt) for s in shape]
            t = X[(Ellipsis, None)]
            for m in range(N):
                idx = [None] * (N + 1)
                idx[m] = idx[N] = slice(None)
                t = t * U[m][tuple(idx)]
            r = sparse.sum(t, axis=-1)
            bk.add({"op": "tttp", "dtype": dt, "order": N, "R": R}, **enc("X_", X),
                   **{f"U{m}": U[m] for m in range(N)}, **enc("out_", r))
    bk.save()


if __name__ == "__main__":
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen_tttp()
