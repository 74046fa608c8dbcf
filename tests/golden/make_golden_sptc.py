#!/usr/bin/env python
"""Generate tests/golden/sptc_api.npz from the REFERENCE itself: its own `sparse.tensordot(COO, COO, axes,
return_type=COO)` on small seeded tensors of order 1..5, one, two and all-but-one contracted axes, axes paired out of
order and negative, float32 / float64 / int64, signed values (so that some sums cancel).  Uses the helpers of
make_golden.py (same reference import, same fixture layout) and writes only this file:

    SPARSE_REFERENCE=<checkout> python tests/golden/make_golden_sptc.py
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import Book, enc, rand_sparse, sparse  # noqa: E402

# (shape of X, shape of Y, axes)
CASES = [
    ((7, 6, 5), (5, 4), 1),
    ((7, 6, 5), (6, 5, 3), 2),
    ((7, 6, 5), (5, 7, 4), ([2, 0], [0, 1])),
    ((7, 6, 5), (4, 6), ([1], [1])),
    ((7, 6, 5), (6, 3, 7), ([-2, 0], [0, -1])),
    ((5, 4, 6, 3), (3, 5, 6, 2), ([3, 0, 2], [0, 1, 2])),
    ((5, 4, 6, 3), (6, 4), ([2, 1], [0, 1])),
    ((4, 3, 2, 3, 4), (3, 4, 5), ([3, 4], [0, 1])),
    ((9, 8), (8, 7), 1),
    ((9, 8), (9, 8), 2),
    ((9,), (9, 4), 1),
    ((6, 9), (9,), ([1], [0])),
    ((5, 4), (3, 2), 0),
]


def signed(rng, x, dt):
    s = rng.choice([-1, 1], x.nnz)
    return sparse.COO(x.coords, (x.data * s).astype(dt), shape=x.shape)


def gen_sptc():
    bk = Book("sptc_api")
    rng = np.random.default_rng(53)
    for dt in ("float32", "float64", "int64"):
        for k, (xs, ys, axes) in enumerate(CASES):
            X = signed(rng, rand_sparse(rng, xs, 0.4, dt), dt)
            Y = signed(rng, rand_sparse(rng, ys, 0.4, dt), dt)
            r = sparse.tensordot(X, Y, axes=axes, return_type=sparse.COO)
            bk.add({"op": "sptc", "dtype": dt, "case": k, "axes": axes}, **enc("X_", X), **enc("Y_", Y),
                   **enc("out_", r))
    bk.save()


if __name__ == "__main__":
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen_sptc()
