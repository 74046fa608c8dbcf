#!/usr/bin/env python
"""Generate the sparse-tensor op fixtures in tests/golden/ from the REFERENCE itself, each as the reference computes the
op with its own unfused expressions (U_m on axis m and its rank on a trailing axis, see `factor_on`):

    mttkrp_mode_api.npz    sum(X[..., None] * U_a[..] * U_b[..] * ..., axis = every axis but n)
    ttmc_mode_api.npz      sum(X[..., None, None, ...] * U_a[..] * U_b[..] * ..., axis = every axis of X but n): a
                           (I_n, R_a, R_b, ...) result, with a different rank on every mode so that a column-order
                           mistake cannot pass
    tttp_api.npz           sum(X[..., None] * U_0[..] * U_1[..] * ..., axis=-1): X's pattern; signed factors, so some
                           model values are negative and some products cancel
    ttm_mode_api.npz       moveaxis(tensordot(X, U, axes=([n], [0]), return_type=COO), -1, n) for a 2-D U (TTM) and
                           tensordot(X, u, axes=([n], [0]), return_type=COO) for a 1-D u (TTV); signed values and
                           factors, and fibers whose products cancel exactly (so some sums are +-0 and not stored)
    cp_completion_api.npz  the per-row Gram matrices and right-hand sides of CP completion's ALS update (mode n, the
                           other modes a < b, P X's pattern with ones), every product and sum in float64:
                               G = sum(P[..., None, None] * U_a[..., :, None] * U_a[..., None, :] * U_b[..] * ...)
                               b = sum(X[..., None] * U_a[..., :] * U_b[..., :] * ...)
                           the test solves (G_i + reg I) x = b_i in float64 against cp_completion_mode

Orders 3 and 4 (and an order-3 R = 1 case for tttp and cp_completion), every mode, float32 and float64.  Uses the
helpers of make_golden.py (same reference import, same fixture layout) and writes only these five files:

    SPARSE_REFERENCE=<checkout> python tests/golden/make_golden_tensor_ops.py
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import Book, enc, rand_sparse, sparse  # noqa: E402


def factor_on(u, m, N, rank_axis=0, n_rank=1):
    """u (I_m, R) as a broadcast operand of N + n_rank dimensions: I_m on axis m, R on axis N + rank_axis."""
    idx = [None] * (N + n_rank)
    idx[m] = slice(None)
    idx[N + rank_axis] = slice(None)
    return u[tuple(idx)]


def gen_mttkrp_mode():
    bk = Book("mttkrp_mode_api")
    rng = np.random.default_rng(23)
    for dt in ("float32", "float64"):
        for shape, R in (((7, 6, 5), 4), ((5, 4, 6, 3), 3)):
            N = len(shape)
            X = rand_sparse(rng, shape, 0.25, dt)
            U = [(rng.random((s, R)) - 0.5).astype(dt) for s in shape]
            for mode in range(N):
                others = tuple(m for m in range(N) if m != mode)
                t = X[(Ellipsis, None)]
                for m in others:
                    t = t * factor_on(U[m], m, N)
                r = sparse.sum(t, axis=others)
                bk.add({"op": "mttkrp_mode", "dtype": dt, "order": N, "mode": mode}, **enc("X_", X),
                       **{f"U{m}": U[m] for m in range(N)}, **enc("out_", r))
    bk.save()


def gen_ttmc_mode():
    bk = Book("ttmc_mode_api")
    rng = np.random.default_rng(29)
    for dt in ("float32", "float64"):
        for shape, ranks in (((7, 6, 5), (3, 4, 2)), ((5, 4, 6, 3), (2, 3, 4, 5))):
            N = len(shape)
            X = rand_sparse(rng, shape, 0.25, dt)
            U = [(rng.random((s, r)) - 0.5).astype(dt) for s, r in zip(shape, ranks)]
            for mode in range(N):
                others = tuple(m for m in range(N) if m != mode)
                t = X[(Ellipsis,) + (None,) * len(others)]
                for k, m in enumerate(others):
                    t = t * factor_on(U[m], m, N, k, len(others))
                r = sparse.sum(t, axis=others)
                bk.add({"op": "ttmc_mode", "dtype": dt, "order": N, "mode": mode}, **enc("X_", X),
                       **{f"U{m}": U[m] for m in range(N)}, **enc("out_", r))
    bk.save()


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
                t = t * factor_on(U[m], m, N)
            r = sparse.sum(t, axis=-1)
            bk.add({"op": "tttp", "dtype": dt, "order": N, "R": R}, **enc("X_", X),
                   **{f"U{m}": U[m] for m in range(N)}, **enc("out_", r))
    bk.save()


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


def gen_cp_completion():
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
                    t = t * factor_on(U64[m], m, N)
                b = sparse.sum(t, axis=others)
                bk.add({"op": "cp_completion_mode", "dtype": dt, "order": N, "R": R, "mode": mode}, **enc("X_", X),
                       **{f"U{m}": U[m] for m in range(N)}, **enc("G_", G), **enc("b_", b))
    bk.save()


if __name__ == "__main__":
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for gen in (gen_mttkrp_mode, gen_ttmc_mode, gen_tttp, gen_ttm_mode, gen_cp_completion):
            gen()
