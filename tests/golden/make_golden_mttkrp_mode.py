#!/usr/bin/env python
"""Generate tests/golden/mttkrp_mode_api.npz from the REFERENCE itself: mode-n MTTKRP as the reference computes it,
the unfused broadcast expression

    sum(X[..., None] * U_a[..] * U_b[..] * ..., axis = every axis but n)

for orders 3 and 4, every mode, float32 and float64.  Uses the helpers of make_golden.py (same reference import, same
fixture layout) and writes only this one file:

    SPARSE_REFERENCE=<checkout> python tests/golden/make_golden_mttkrp_mode.py
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import Book, enc, rand_sparse, sparse  # noqa: E402


def gen_mttkrp_mode():
    bk = Book("mttkrp_mode_api")
    rng = np.random.default_rng(23)
    for dt in ("float32", "float64"):
        for shape, R in (((7, 6, 5), 4), ((5, 4, 6, 3), 3)):
            N = len(shape)
            X = rand_sparse(rng, shape, 0.25, dt)
            U = [(rng.random((s, R)) - 0.5).astype(dt) for s in shape]
            for mode in range(N):
                t = X[(Ellipsis, None)]
                for m in range(N):
                    if m != mode:
                        idx = [None] * (N + 1)
                        idx[m] = idx[N] = slice(None)
                        t = t * U[m][tuple(idx)]
                r = sparse.sum(t, axis=tuple(m for m in range(N) if m != mode))
                bk.add({"op": "mttkrp_mode", "dtype": dt, "order": N, "mode": mode}, **enc("X_", X),
                       **{f"U{m}": U[m] for m in range(N)}, **enc("out_", r))
    bk.save()


if __name__ == "__main__":
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen_mttkrp_mode()
