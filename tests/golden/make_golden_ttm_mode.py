#!/usr/bin/env python
"""Generate tests/golden/ttm_mode_api.npz from the REFERENCE itself: mode-n tensor times matrix (and vector) of a sparse
tensor as the reference computes it,

    sparse.moveaxis(sparse.tensordot(X, U, axes=([n], [0]), return_type=sparse.COO), -1, n)    (2-D U, TTM)
    sparse.tensordot(X, U, axes=([n], [0]), return_type=sparse.COO)                             (1-D U, TTV)

Orders 3 and 4, every mode, float32 and float64, signed values and factors, and fibers whose products cancel exactly
(so some sums are +-0 and are not stored).  Uses the helpers of make_golden.py (same reference import, same fixture
layout) and writes only this one file:

    SPARSE_REFERENCE=<checkout> python tests/golden/make_golden_ttm_mode.py
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import Book, enc, rand_sparse, sparse  # noqa: E402


def gen_ttm_mode():
    bk = Book("ttm_mode_api")
    rng = np.random.default_rng(47)
    for dt in ("float32", "float64"):
        for shape, R in (((7, 6, 5), 4), ((5, 4, 6, 3), 3)):
            N = len(shape)
            X = rand_sparse(rng, shape, 0.35, dt)
            X = sparse.COO(X.coords, (X.data * rng.choice([-1, 1], X.nnz)).astype(dt), shape=shape)
            for n in range(N):
                U = (rng.random((shape[n], R)) - 0.5).astype(dt)
                U[1] = U[0]  # rows 0 and 1 equal: fibers holding +v at i_n = 0 and -v at i_n = 1 cancel exactly
                u = (rng.random(shape[n]) - 0.5).astype(dt)
                u[1] = u[0]
                c0, v0 = X.coords, X.data
                lead = c0[n] == 0
                twin = c0[:, lead].copy()
                twin[n] = 1
                keep = ~np.isin(np.ravel_multi_index(c0, shape), np.ravel_multi_index(twin, shape))
                c = np.concatenate([c0[:, keep], twin], axis=1)
                v = np.concatenate([v0[keep], -v0[lead]]).astype(dt)
                Xn = sparse.COO(c, v, shape=shape)
                ttm = sparse.moveaxis(sparse.tensordot(Xn, U, axes=([n], [0]), return_type=sparse.COO), -1, n)
                ttv = sparse.tensordot(Xn, u, axes=([n], [0]), return_type=sparse.COO)
                bk.add({"op": "ttm_mode", "dtype": dt, "order": N, "mode": n, "R": R}, **enc("X_", Xn), U=U,
                       **enc("out_", ttm))
                bk.add({"op": "ttv", "dtype": dt, "order": N, "mode": n, "R": 0}, **enc("X_", Xn), U=u,
                       **enc("out_", ttv))
    bk.save()


if __name__ == "__main__":
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen_ttm_mode()
