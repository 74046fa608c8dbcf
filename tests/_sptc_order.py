"""CPU restatement of sptc's contract (include/sparse_b200.h, b2s_sptc_join) -- TEST INFRASTRUCTURE ONLY.

Written from the contract alone, with dictionaries: no matricisation, no row pointers, nothing sized by an extent.
"""
import numpy as np


def same_bits(x, y):
    """Bit-equal, except that any NaN matches any NaN (the device returns the canonical NaN, NumPy keeps payloads)."""
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    if x.shape != y.shape or x.dtype != y.dtype:
        return False
    if x.dtype.kind == "f":
        xn, yn = np.isnan(x), np.isnan(y)
        if not np.array_equal(xn, yn):
            return False
        x, y = x[~xn], y[~yn]
    return np.array_equal(x.view(np.uint8), y.view(np.uint8))


def _key(coords, shape, axes):
    """C-order linear key (Python ints) of every entry over `axes`, in that order."""
    k = [0] * coords.shape[1]
    for a in axes:
        s = int(shape[a])
        k = [v * s + int(c) for v, c in zip(k, coords[a])]
    return k


def result(xc, xv, xshape, yc, yv, yshape, axes_x, axes_y, dtype):
    """(linear keys over free(X) + free(Y), ascending, int64; values) of sptc on the stored entries (xc, xv) and
    (yc, yv): z(F, G) = ((+0 + x(F, C_1) * y(C_1, G)) + ...) over the common C ascending, each product and sum
    rounded in `dtype`, stored iff its bits differ from +0."""
    dtype = np.dtype(dtype)
    xc, yc = np.asarray(xc, np.int64), np.asarray(yc, np.int64)
    xv, yv = np.asarray(xv).astype(dtype), np.asarray(yv).astype(dtype)
    axes_x = [a % len(xshape) for a in axes_x]
    axes_y = [a % len(yshape) for a in axes_y]
    free_x = [a for a in range(len(xshape)) if a not in axes_x]
    free_y = [a for a in range(len(yshape)) if a not in axes_y]
    g_ext = 1
    for a in free_y:
        g_ext *= int(yshape[a])
    by_c = {}
    for C, G, v in zip(_key(yc, yshape, axes_y), _key(yc, yshape, free_y), yv):
        by_c.setdefault(C, []).append((G, v))
    terms = {}
    for F, C, v in zip(_key(xc, xshape, free_x), _key(xc, xshape, axes_x), xv):
        for G, w in by_c.get(C, ()):
            terms.setdefault(F * g_ext + G, []).append((C, v, w))
    keys, vals = [], []
    zero = dtype.type(0)
    with np.errstate(all="ignore"):
        for k in sorted(terms):
            acc = zero
            for _, v, w in sorted(terms[k], key=lambda t: t[0]):
                acc = dtype.type(acc + dtype.type(v * w))
            if acc.tobytes() != zero.tobytes():
                keys.append(k)
                vals.append(acc)
    return np.array(keys, np.int64), np.array(vals, dtype)
