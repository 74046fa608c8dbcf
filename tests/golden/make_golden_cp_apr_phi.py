#!/usr/bin/env python
"""Generate tests/golden/cp_apr_phi_api.npz from the REFERENCE itself: CP-APR's ratio MTTKRP Phi as the reference
computes it with its own unfused expressions (U_m on axis m and its rank on a trailing axis, see
make_golden_tensor_ops.factor_on; P is X's pattern with ones):

    M = sum(P[..., None] * U_0[..] * U_1[..] * ..., axis=-1)        the model at X's entries
    W = elemwise(lambda x, m: x / maximum(m, eps), X, M)
    Phi = sum(W[..., None] * U_a[..] * U_b[..] * ..., axis = every axis but n)

Nonnegative data and factors, orders 3 and 4, every mode, float32 and float64, and eps the lower quartile of M, so
that some entries are clamped.  Uses the helpers of make_golden.py (same reference import, same fixture layout) and
writes only this file:

    SPARSE_REFERENCE=<checkout> python tests/golden/make_golden_cp_apr_phi.py
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import Book, enc, rand_sparse, sparse  # noqa: E402
from make_golden_tensor_ops import factor_on  # noqa: E402


def gen_cp_apr_phi():
    bk = Book("cp_apr_phi_api")
    rng = np.random.default_rng(53)
    for dt in ("float32", "float64"):
        for shape, R in (((7, 6, 5), 4), ((5, 4, 6, 3), 3)):
            N = len(shape)
            X = rand_sparse(rng, shape, 0.3, dt)
            U = [rng.random((s, R)).astype(dt) for s in shape]
            P = sparse.COO(X.coords, np.ones(X.nnz, dt), shape=X.shape)
            t = P[(Ellipsis, None)]
            for m in range(N):
                t = t * factor_on(U[m], m, N)
            M = sparse.sum(t, axis=-1)
            eps = float(np.asarray(np.quantile(M.data, 0.25), dt))  # a quarter of the entries are clamped
            W = sparse.elemwise(lambda x, m: x / np.maximum(m, eps), X, M)
            for mode in range(N):
                others = tuple(m for m in range(N) if m != mode)
                t = W[(Ellipsis, None)]
                for m in others:
                    t = t * factor_on(U[m], m, N)
                r = sparse.sum(t, axis=others)
                bk.add({"op": "cp_apr_phi_mode", "dtype": dt, "order": N, "mode": mode, "eps": eps}, **enc("X_", X),
                       **{f"U{m}": U[m] for m in range(N)}, **enc("out_", r))
    bk.save()


if __name__ == "__main__":
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen_cp_apr_phi()
