"""Plain CPU restatement of the CSR x CSR row product (spgemm.cu), for tests/test_spgemm_rows_gpu.py.

Gustavson, row by row: the products of a row are visited A entry by A entry in stored order, each through its B row in
stored order.  A product is rounded in the value type T; the products that meet in one column are summed in visiting
order in the accumulator (T, or float64 for `wide`, the `sums` array of _dot_csc_ndarray_sparse).  Integer arithmetic
wraps.  `wide` narrows each sum to T, a sum equal to 0 becoming +0 (the reference skips it; a pruned product drops it).

Columns of a row come out in reverse order of first touch (the reference's intrusive linked list), or ascending in
SORTED order; when every row is completely dense the REF rows are reversed.  The oracle (oracle.dot_csr_csr) computes
the same thing and is pinned against the reference; this restatement is for what it cannot take: wrapping integer
products (C's signed overflow), the float64 accumulator over any CSR operands, and columns of 2^32 and more."""
import numpy as np

_UNSIGNED = {4: np.uint32, 8: np.uint64}


def _mul(x, y):
    if x.dtype.kind == "f":
        return x * y
    u = _UNSIGNED[x.dtype.itemsize]
    return (x.view(u) * y.view(u)).view(x.dtype)


def _add(x, y):
    if x.dtype.kind == "f":
        return x + y
    u = _UNSIGNED[x.dtype.itemsize]
    return (x.view(u) + y.view(u)).view(x.dtype)


def spgemm(a, b, M, n_col, *, sorted_order=False, wide=False):
    """(indptr, indices, data, nnz_struct) of A @ B, A = (data, indices, indptr) with M rows, B likewise; no pruning
    (see `prune`).  nnz_struct counts every (row, column) some product reaches."""
    with np.errstate(invalid="ignore", over="ignore"):  # NaN and Inf operands are part of the tests
        return _spgemm(a, b, M, n_col, sorted_order, wide)


def _spgemm(a, b, M, n_col, sorted_order, wide):
    ad, ai, ap = a
    bd, bi, bp = b
    T = np.dtype(ad.dtype)
    ai = np.asarray(ai, np.int64)
    ap = np.asarray(ap, np.int64)
    bi = np.asarray(bi, np.int64)
    bp = np.asarray(bp, np.int64)
    blen = bp[ai + 1] - bp[ai]
    n = int(blen.sum())
    ent = np.repeat(np.arange(len(ai), dtype=np.int64), blen)           # A entry of every product, visiting order
    first = np.cumsum(blen) - blen
    q = bp[ai][ent] + (np.arange(n, dtype=np.int64) - first[ent])       # its B entry
    row = np.repeat(np.arange(M, dtype=np.int64), np.diff(ap))[ent]
    col = bi[q]
    prod = _mul(ad[ent], bd[q])
    o = np.lexsort((col, row))                                          # stable: visiting order inside a column
    rs, cs = row[o], col[o]
    new = np.ones(n, bool)
    new[1:] = (rs[1:] != rs[:-1]) | (cs[1:] != cs[:-1])
    gstart = np.flatnonzero(new)
    gid = np.cumsum(new) - 1
    rank = np.arange(n, dtype=np.int64) - gstart[gid]
    W = np.dtype(np.float64) if wide else T
    pw = prod[o].astype(W)
    acc = np.zeros(len(gstart), W)
    by_rank = np.argsort(rank, kind="stable")
    bounds = np.concatenate([[0], np.cumsum(np.bincount(rank))]) if n else [0]
    for k in range(len(bounds) - 1):                                    # the k-th add of every column at once
        sel = by_rank[bounds[k]:bounds[k + 1]]
        acc[gid[sel]] = _add(acc[gid[sel]], pw[sel])
    if wide:
        val = acc.astype(T)
        val[acc == 0] = 0
    else:
        val = acc
    g_row, g_col, g_first = rs[gstart], cs[gstart], o[gstart]
    if not sorted_order:
        dense = n_col > 0 and len(gstart) == M * n_col
        order = np.lexsort((g_first if dense else -g_first, g_row))
        g_row, g_col, val = g_row[order], g_col[order], val[order]
    indptr = np.zeros(M + 1, np.int64)
    np.cumsum(np.bincount(g_row, minlength=M), out=indptr[1:])
    return indptr, g_col, val, len(gstart)


def positive_zero(x):
    """Mask of the entries whose bits are +0 (what prune=True drops)."""
    x = np.ascontiguousarray(x)
    return x.view(_UNSIGNED[x.dtype.itemsize]) == 0


def prune(indptr, indices, data):
    """Drop the entries whose value is +0 bit for bit (-0.0 stays)."""
    keep = ~positive_zero(data)
    M = len(indptr) - 1
    row = np.repeat(np.arange(M, dtype=np.int64), np.diff(indptr))
    out = np.zeros(M + 1, np.int64)
    np.cumsum(np.bincount(row[keep], minlength=M), out=out[1:])
    return out, indices[keep], data[keep]


def sort_rows(indptr, indices, data):
    """SORTED order from a REF result: columns ascending inside each row."""
    M = len(indptr) - 1
    row = np.repeat(np.arange(M, dtype=np.int64), np.diff(indptr))
    o = np.lexsort((indices, row))
    return indptr, indices[o], data[o]
