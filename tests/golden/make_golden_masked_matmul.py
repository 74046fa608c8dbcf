#!/usr/bin/env python
"""Generate tests/golden/masked_matmul_api.npz from the REFERENCE itself: the unfused masked product

    mask * (a @ b)

(examples/triangles_example.py computes sum(a @ a * a) / 6 this way) for float32, float64 and int64 operands: random
matrices with negative values, -0.0, inf and NaN in a, b and the mask, empty rows and columns, K = 0, an empty mask,
and a small symmetric graph.  The inputs are stored as canonical COO; the tests build every COO / GCXS layout from
them.  Uses the helpers of make_golden.py (same reference import, same fixture layout) and writes only this one file:

    SPARSE_REFERENCE=<checkout> python tests/golden/make_golden_masked_matmul.py
"""
import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import Book, enc, rand_sparse, sparse  # noqa: E402


def _special(rng, x, dt):
    """Negative values, -0.0, inf and NaN in the stored data of x (floats), negative values for integers."""
    d = x.data.copy()
    if len(d) == 0:
        return x
    sign = rng.choice(np.array([-1, 1], dtype=dt), len(d))
    d = (d * sign).astype(dt)
    if np.issubdtype(np.dtype(dt), np.floating):
        picks = rng.choice(len(d), size=min(3, len(d)), replace=False)
        for p, v in zip(picks, (-0.0, np.inf, np.nan)):
            d[p] = v
    return sparse.COO(x.coords, d, shape=x.shape)


def _graph(rng, n, p):
    u = np.triu(rng.random((n, n)) < p, 1)
    adj = (u | u.T).astype(np.float64)
    return sparse.COO.from_numpy(adj)


def gen_masked_matmul():
    bk = Book("masked_matmul_api")
    rng = np.random.default_rng(20261015)
    shapes = [((9, 11, 7), 0.35), ((16, 13, 20), 0.2), ((1, 5, 1), 0.9), ((12, 0, 10), 0.3), ((10, 6, 14), 0.0)]
    for dt in ("float32", "float64", "int64"):
        for (M, K, N), dens in shapes:
            for special in (False, True):
                mask = rand_sparse(rng, (M, N), max(dens, 0.0) if dens else 0.0, dt)
                if dens == 0.0:
                    mask = sparse.COO(np.zeros((2, 0), dtype=np.int64), np.zeros(0, dtype=dt), shape=(M, N))
                a = rand_sparse(rng, (M, K), dens or 0.3, dt)
                b = rand_sparse(rng, (K, N), dens or 0.3, dt)
                if M > 3 and K > 3 and N > 3:
                    # an empty row of a and the mask, an empty column of b
                    a = sparse.COO.from_numpy(np.where(np.arange(M)[:, None] == 2, 0, a.todense()).astype(dt))
                    b = sparse.COO.from_numpy(np.where(np.arange(N)[None, :] == 3, 0, b.todense()).astype(dt))
                if special:
                    mask, a, b = _special(rng, mask, dt), _special(rng, a, dt), _special(rng, b, dt)
                out = mask * (a @ b)
                nonneg = not special
                bk.add({"op": "masked_matmul", "dtype": dt, "shape": [M, K, N], "special": special,
                        "full_equal": nonneg}, **enc("mask_", mask), **enc("a_", a), **enc("b_", b),
                       **enc("out_", out))
    for n, p in ((40, 0.15), (64, 0.08)):
        adj = _graph(rng, n, p)
        out = adj @ adj * adj
        bk.add({"op": "triangles", "dtype": "float64", "shape": [n, n, n], "special": False, "full_equal": True,
                "triangles": float(sparse.sum(out) / 6)}, **enc("mask_", adj), **enc("a_", adj), **enc("b_", adj),
               **enc("out_", out))
    bk.save()


if __name__ == "__main__":
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gen_masked_matmul()
