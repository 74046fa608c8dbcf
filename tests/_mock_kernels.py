"""NumPy stand-in for sparse_b200._kernels -- TEST INFRASTRUCTURE ONLY.

Lets the host-side logic of the package (axis bookkeeping, dispatch tables, broadcasting rules, fill values,
result types, errors) be exercised on a box without a GPU: `install()` flips sparse_b200._device._TEST_CPU and
replaces every function of sparse_b200._kernels with a NumPy restatement operating on CPU torch tensors.  The
product never imports this module; the `-m gpu` tests run the same test bodies against the real CUDA kernels.
Dot kernels are delegated to the oracle (bit-exact with the reference).
"""
from __future__ import annotations

import numpy as np
import torch

import oracle
from sparse_b200 import _device as D
from sparse_b200 import _kernels as Kn

_ORIG = {}

_BIN = {0: np.add, 1: np.subtract, 2: np.multiply, 3: np.true_divide, 4: np.maximum, 5: np.minimum, 6: np.fmax,
        7: np.fmin, 8: np.power, 9: np.floor_divide, 10: np.remainder, 11: np.bitwise_and, 12: np.bitwise_or,
        13: np.bitwise_xor, 14: lambda a, b: np.where(np.isnan(a), b, a),
        15: lambda a, b: np.where(a != 0, b, np.asarray(b).dtype.type(0)),
        16: lambda a, b: np.where(a != 0, np.asarray(b).dtype.type(0), b),
        17: lambda a, b: (np.asarray(a).view(f"u{np.asarray(a).dtype.itemsize}") | np.asarray(b).view(f"u{np.asarray(b).dtype.itemsize}")).view(np.asarray(a).dtype),
        18: np.left_shift, 19: np.right_shift,
        32: np.greater, 33: np.greater_equal, 34: np.less, 35: np.less_equal, 36: np.equal,
        37: np.not_equal, 38: np.logical_and, 39: np.logical_or, 40: np.logical_xor}
_UN = {0: np.negative, 1: np.absolute, 2: np.sqrt, 3: np.square, 4: np.sign, 5: np.exp, 6: np.expm1, 7: np.log,
       8: np.log1p, 9: np.sin, 10: np.cos, 11: np.tan, 12: np.tanh, 13: np.sinh, 14: np.cosh, 15: np.arcsin,
       16: np.arctan, 17: np.floor, 18: np.ceil, 19: np.trunc, 20: np.rint, 21: np.reciprocal, 22: np.positive,
       23: np.invert, 24: np.arcsinh, 25: np.arctanh, 26: np.deg2rad, 27: np.rad2deg, 28: np.exp2, 29: np.log2,
       30: np.log10, 31: np.cbrt, 64: np.isnan, 65: np.isinf, 66: np.isfinite, 67: np.logical_not, 68: np.signbit}
_RED = {0: np.add, 1: np.multiply, 2: np.maximum, 3: np.minimum, 4: np.logical_and, 5: np.logical_or,
        6: np.bitwise_and, 7: np.bitwise_or, 8: np.bitwise_xor, 9: np.fmax, 10: np.fmin}


def n(x):
    return x.detach().numpy()


def T(a):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.copy())


def bits_ne(a, fill):
    a = np.ascontiguousarray(a)
    f = np.array([fill], dtype=a.dtype)
    if a.itemsize == 16:
        return (a.view(np.uint64).reshape(-1, 2) != f.view(np.uint64)).any(axis=1)
    w = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.itemsize]
    return a.view(w) != f.view(w)[0]


# ---- K1 / prims ------------------------------------------------------------------------------------------
def csr_rows_sorted(a_indices, a_indptr, M):
    ip, ix = n(a_indptr), n(a_indices)
    return all((np.diff(ix[ip[r]:ip[r + 1]]) >= 0).all() for r in range(M))


def csr_max_row_nnz(a_indptr, M):
    ip = n(a_indptr)
    return int(np.diff(ip).max()) if M else 0


def spmm_csr_dense(a_data, a_indices, a_indptr, b, M, K, N, out=None, n_panels=1, rows_sorted=None, long_rows=False):
    r = oracle.dot_csr_ndarray((M, N), n(a_data), n(a_indices), n(a_indptr), np.ascontiguousarray(n(b)))
    r = T(r)
    if out is not None:
        out.copy_(r)
        return out
    return r


def spmm_csr_dense_host(a_data, a_indices, a_indptr, b, out=None):
    """Host-buffer form of K1 (the real one uploads, launches and downloads inside one C call): same product, host
    arrays in and out, the dtype matrix of the real wrapper."""
    D.dtype_code(a_data.dtype)
    assert b.dtype == a_data.dtype
    M, (K, N) = len(a_indptr) - 1, b.shape
    r = oracle.dot_csr_ndarray((M, N), np.asarray(a_data), np.asarray(a_indices), np.asarray(a_indptr),
                               np.ascontiguousarray(b))
    if out is not None:
        out[...] = r
        return out
    return r


def linearize(coords, strides):
    c = n(coords).astype(np.int64)
    k = np.zeros(c.shape[1], dtype=np.int64)
    for d in range(c.shape[0]):
        k += c[d] * int(strides[d])
    return T(k)


def diag_flags(coords, first):
    c = n(coords)
    keep = np.ones(c.shape[1], dtype=bool)
    for d, f in enumerate(first):
        if f != d:
            keep &= c[d] == c[f]
    return T(keep.astype(np.uint8))


def slice_keys(keys, shape, start, step, count, out_stride):
    k = n(keys)
    c = np.stack(np.unravel_index(k, shape)) if len(k) else np.zeros((len(shape), 0), np.int64)
    keep = np.ones(len(k), dtype=bool)
    ok = np.zeros(len(k), dtype=np.int64)
    for d in range(len(shape)):
        off = (c[d] - start[d]) * (1 if step[d] > 0 else -1)
        j = off // abs(step[d])
        keep &= (off >= 0) & (off % abs(step[d]) == 0) & (j < count[d])
        ok += np.where(keep, j, 0) * out_stride[d]
    return T(keep.astype(np.uint8)), T(ok)


def unravel(keys, shape, idx_dtype=np.int64):
    k = n(keys)
    if len(shape) == 0:
        return T(np.zeros((0, len(k)), dtype=idx_dtype))
    if len(k) == 0:
        return T(np.zeros((len(shape), 0), dtype=idx_dtype))
    return T(np.stack(np.unravel_index(k, shape)).astype(idx_dtype))


def keys_flags(keys):
    k = n(keys)
    if len(k) < 2:
        return False, False
    d = np.diff(k)
    return bool((d < 0).any()), bool((d == 0).any())


def sort_keys(keys, key_bits=64):
    """Like b2s_sort_keys: stable, UNSIGNED order over the low `key_bits` bits (a negative int64 sorts after every
    non-negative one)."""
    k = n(keys)
    ku = np.ascontiguousarray(k).view(np.uint64)
    if 0 < key_bits < 64:
        ku = ku & np.uint64((1 << key_bits) - 1)
    perm = np.argsort(ku, kind="stable")
    return T(k[perm]), T(perm.astype(np.int64))


def gather(x, perm):
    return T(n(x)[n(perm)])


def gather_rows(x2d, perm):
    return T(n(x2d)[:, n(perm)])


def flag_heads(keys):
    k = n(keys)
    f = np.ones(len(k), dtype=np.uint8)
    if len(k) > 1:
        f[1:] = k[1:] != k[:-1]
    return T(f)


def flag_not_fill(data, fill_value):
    return T(bits_ne(n(data), fill_value).astype(np.uint8))


def scan_flags(flags):
    f = n(flags).astype(np.int64)
    pos = np.cumsum(f) - f
    return T(pos), int(f.sum())


def compact(x, flags, pos, total):
    return T(n(x)[n(flags).astype(bool)])


def compact_rows(x2d, flags, pos, total):
    return T(n(x2d)[:, n(flags).astype(bool)])


def segment_sum(data, heads, pos, total):
    d = n(data)
    (starts,) = np.nonzero(n(heads))
    return T(np.add.reduceat(d, starts, dtype=d.dtype)) if len(d) else T(d)


def indptr_from_sorted(rows, nrows, idx_dtype=np.int64):
    return T(np.searchsorted(n(rows), np.arange(nrows + 1), side="left").astype(idx_dtype))


def csr_from_keys(keys, nrows, ncols, idx_dtype=np.int64, want_rows=False, want_indptr=True):
    k = n(keys)
    ncols = max(ncols, 1)
    rows = k // ncols
    indices = (k % ncols).astype(idx_dtype)
    indptr = np.searchsorted(k, np.arange(nrows + 1) * ncols, side="left").astype(idx_dtype) if want_indptr else None
    return (T(rows.astype(idx_dtype)) if want_rows else None, T(indices), T(indptr) if want_indptr else None)


def rows_from_indptr(indptr, nnz, idx_dtype=np.int64):
    ip = n(indptr).astype(np.int64)
    return T(np.repeat(np.arange(len(ip) - 1), np.diff(ip)).astype(idx_dtype))


def full(nn, value, dtype):
    return T(np.full(nn, value, dtype=dtype))


def iota(nn):
    return T(np.arange(nn, dtype=np.int64))


def scatter(data, keys, out):
    o = n(out)
    o[n(keys)] = n(data)
    return out


def cast(x, dtype):
    if D.np_dtype(x) == np.dtype(dtype):
        return x
    D.cast_code(D.np_dtype(x)), D.cast_code(dtype)  # same TypeError as the real wrapper for dtypes b2s_cast lacks
    with np.errstate(all="ignore"):
        return T(n(x).astype(dtype))


def transpose_dense(x):
    return T(n(x).T.copy())


def any_nan(x):
    a = n(x)
    return bool(np.isnan(a).any()) if a.dtype.kind == "f" else False


def indptr_remap(old_indptr, pos, nn, total):
    ip = n(old_indptr).astype(np.int64)
    p = np.concatenate([n(pos), [total]])
    return T(p[np.minimum(ip, nn)].astype(D.np_dtype(old_indptr)))


# ---- K4 / K3 ---------------------------------------------------------------------------------------------------
def spgemm(a_indptr, a_indices, a_data, b_indptr, b_indices, b_data, M, K, n_col, *, sorted_order=False, wide=False,
           prune=False, want_indptr=True, want_rows=False):
    ad, bd = n(a_data), n(b_data)
    dt = ad.dtype
    if wide:
        # float64 accumulator, product rounded to dt first (restated directly; small inputs only)
        data_l, idx_l, ptr = [], [], [0]
        ap, ai, bp, bi = n(a_indptr), n(a_indices), n(b_indptr), n(b_indices)
        for r in range(M):
            order, acc = [], {}
            for p in range(ap[r], ap[r + 1]):
                for q in range(bp[ai[p]], bp[ai[p] + 1]):
                    c = int(bi[q])
                    if c not in acc:
                        acc[c] = 0.0
                        order.append(c)
                    acc[c] = acc[c] + float(dt.type(ad[p] * bd[q]))
            for c in reversed(order):
                v = acc[c]
                idx_l.append(c)
                data_l.append(dt.type(0) if v == 0 else dt.type(v))
            ptr.append(len(idx_l))
        data, indices, indptr = np.array(data_l, dtype=dt), np.array(idx_l, dtype=np.int64), np.array(ptr, np.int64)
        nstruct = len(indices)
    else:
        data, indices, indptr = oracle.dot_csr_csr((M, n_col), ad, bd, n(a_indices), n(b_indices), n(a_indptr),
                                                   n(b_indptr))
        nstruct = len(indices)
    rows = np.repeat(np.arange(M), np.diff(indptr))
    if sorted_order:
        if nstruct == M * n_col and M * n_col > 0:  # undo the dense flip before sorting (irrelevant to sorted order)
            pass
        o = np.lexsort((indices, rows))
        data, indices = data[o], indices[o]
    if prune:
        keep = bits_ne(data, dt.type(0))
        data, indices, rows = data[keep], indices[keep], rows[keep]
        indptr = np.searchsorted(rows, np.arange(M + 1), side="left").astype(np.int64)
    return (T(indptr) if want_indptr else None, T(indices), T(rows.astype(np.int64)) if want_rows else None, T(data),
            nstruct)


def spmm_csr_dense_flagged(a_data, a_indices, a_indptr, b, M, K, N):
    bb = np.ascontiguousarray(n(b))
    data, indices, indptr = oracle.dot_csr_ndarray_sparse((M, N), n(a_data), n(a_indices), n(a_indptr), bb)
    out = np.zeros((M, N), dtype=data.dtype)
    flags = np.zeros((M, N), dtype=np.uint8)
    rows = np.repeat(np.arange(M), np.diff(indptr))
    out[rows, indices] = data
    flags[rows, indices] = 1
    return T(out), T(flags)


def dense_to_csr(x, flags=None, mode=0, want_rows=False, want_indptr=True):
    a = n(x)
    M, N = a.shape
    if flags is not None:
        keep = n(flags).reshape(M, N).astype(bool)
    elif mode == 0:
        keep = a != 0
    else:
        keep = bits_ne(a.reshape(-1), a.dtype.type(0)).reshape(M, N)
    rows, cols = np.nonzero(keep)
    indptr = np.searchsorted(rows, np.arange(M + 1), side="left").astype(np.int64)
    return (T(rows.astype(np.int64)) if want_rows else None, T(cols.astype(np.int64)), T(a[keep]),
            T(indptr) if want_indptr else None)


# ---- K5 -----------------------------------------------------------------------------------------------------------
def _virt(keys, data, R):
    k, d = n(keys), n(data)
    if R == 1:
        return k, d
    return (k[:, None] * R + np.arange(R)[None, :]).reshape(-1), np.repeat(d, R)


def _apply_bin(op, a, b, out_dtype):
    with np.errstate(all="ignore"):
        return np.asarray(_BIN[op](a, b)).astype(out_dtype)


def ew_merge(op, keys_a, data_a, Ra, keys_b, data_b, Rb, fill_a, fill_b, out_fill, out_dtype):
    ka, da = _virt(keys_a, data_a, Ra)
    kb, db = _virt(keys_b, data_b, Rb)
    keys = np.union1d(ka, kb)
    dt = da.dtype
    va = np.full(len(keys), fill_a, dtype=dt)
    vb = np.full(len(keys), fill_b, dtype=dt)
    va[np.searchsorted(keys, ka)] = da
    vb[np.searchsorted(keys, kb)] = db
    r = _apply_bin(op, va, vb, out_dtype)
    flags = bits_ne(r, np.dtype(out_dtype).type(out_fill)).astype(np.uint8)
    return T(keys), T(r), T(flags)


def ew_merge_fused(op, keys_a, data_a, Ra, keys_b, data_b, Rb, fill_a, fill_b, out_fill, out_dtype, shape,
                   want_coords=True):
    keys, vals, flags = ew_merge(op, keys_a, data_a, Ra, keys_b, data_b, Rb, fill_a, fill_b, out_fill, out_dtype)
    keep = n(flags).astype(bool)
    k = T(n(keys)[keep])
    return (unravel(k, shape, np.int64) if want_coords else None), T(n(vals)[keep]), k


def ew_map(op, mode, x, scalar, out_fill, out_dtype):
    a = n(x)
    with np.errstate(all="ignore"):
        if mode == 2:
            r = np.asarray(_UN[op](a)).astype(out_dtype)
        elif mode == 0:
            r = _apply_bin(op, a, a.dtype.type(scalar), out_dtype)
        else:
            r = _apply_bin(op, a.dtype.type(scalar), a, out_dtype)
    return T(r), T(bits_ne(r, np.dtype(out_dtype).type(out_fill)).astype(np.uint8))


def ew_dense(op, swap, keys_a, data_a, Ra, dense, shape, dense_strides, out_fill, out_dtype):
    k, d = _virt(keys_a, data_a, Ra)
    dn = n(dense).reshape(-1)
    if len(shape):
        coords = np.stack(np.unravel_index(k, shape)) if len(k) else np.zeros((len(shape), 0), np.int64)
        off = np.zeros(len(k), dtype=np.int64)
        for dd in range(len(shape)):
            off += coords[dd] * int(dense_strides[dd])
    else:
        off = np.zeros(len(k), dtype=np.int64)
    dv = dn[off]
    r = _apply_bin(op, dv, d, out_dtype) if swap else _apply_bin(op, d, dv, out_dtype)
    return T(k), T(r), T(bits_ne(r, np.dtype(out_dtype).type(out_fill)).astype(np.uint8))


def ew_expand(coords, result_shape, is_bcast, src_row):
    c = n(coords).astype(np.int64)
    nn = c.shape[1]
    bdims = [d for d, b in enumerate(is_bcast) if b]
    R = int(np.prod([result_shape[d] for d in bdims])) if bdims else 1
    st = [1] * len(result_shape)
    for d in range(len(result_shape) - 2, -1, -1):
        st[d] = st[d + 1] * int(result_shape[d + 1])
    keys = np.zeros((nn, R), dtype=np.int64)
    r = np.arange(R)
    digits = {}
    for d in reversed(bdims):
        digits[d] = r % int(result_shape[d])
        r = r // int(result_shape[d])
    for d in range(len(result_shape)):
        if is_bcast[d]:
            keys += digits[d][None, :] * st[d]
        else:
            keys += (c[src_row[d]] * st[d])[:, None]
    src = np.repeat(np.arange(nn), R)
    return T(keys.reshape(-1)), T(src.astype(np.int64))


# ---- K7 ------------------------------------------------------------------------------------------------------------
def group_ids(keys, ncols):
    return T(n(keys) // ncols)


def reduce_by_key(op, gid, vals):
    g, v = n(gid), n(vals)
    heads = np.ones(len(g), dtype=bool)
    heads[1:] = g[1:] != g[:-1]
    (starts,) = np.nonzero(heads)
    with np.errstate(all="ignore"):
        r = _RED[op].reduceat(v, starts).astype(v.dtype)
    counts = np.diff(np.concatenate([starts, [len(g)]]))
    return T(g[starts]), T(r), T(counts.astype(np.int64))


def reduce_fused(op, keys, vals, ncols, fill_value, result_fill, kept_shape, want_coords=True):
    gid = group_ids(keys, ncols)
    groups, r, counts = reduce_by_key(op, gid, vals)
    reduce_fill_fix(op, r, counts, ncols, fill_value)
    neq = int((~bits_ne(n(r), n(r).dtype.type(result_fill))).sum())
    return (unravel(groups, kept_shape, np.int64) if want_coords else None), groups, r, neq


def reduce_fill_fix(op, vals, counts, ncols, fill_value):
    v, c = n(vals), n(counts)
    nf = ncols - c
    fill = v.dtype.type(fill_value)
    with np.errstate(all="ignore"):
        if op in (0, 1):
            # contribution and combine in the type NumPy promotes T and int64 n_fill to (float64 for float32, int64 for
            # the integers), rounded to T once at the end, as _sparse_array.py:410-421 does
            method, sup, identity = (np.add, np.multiply, 0) if op == 0 else (np.multiply, np.power, 1)
            contrib = np.where(nf == 0, identity, sup(fill, nf))
            v[:] = method(v, contrib).astype(v.dtype)
        else:
            m = nf != 0
            v[m] = _RED[op](v[m], fill).astype(v.dtype)
    return vals


# ---- K8 / K9 ----------------------------------------------------------------------------------------------------------
def sddmm(indptr, cols, s_vals, a, bt, M, N, K):
    ip, c, sv = n(indptr).astype(np.int64), n(cols).astype(np.int64), n(s_vals)
    rows = np.repeat(np.arange(M), np.diff(ip))
    dots = np.einsum("nk,nk->n", n(a)[rows], n(bt)[c]).astype(sv.dtype)
    return T(sv * dots)


def mttkrp(indptr, kk, ll, vals, Dm, Cm, I_, J):
    ip = n(indptr).astype(np.int64)
    rows = np.repeat(np.arange(I_), np.diff(ip))
    contrib = n(vals)[:, None] * n(Dm)[n(ll).astype(np.int64)] * n(Cm)[n(kk).astype(np.int64)]
    out = np.zeros((I_, J), dtype=n(vals).dtype)
    np.add.at(out, rows, contrib)
    return T(out)


def spgemm_set_thresholds(t0=64, t1=256):
    return None


def spmm_set_variant(variant=1, unroll=8):
    return None


def spmm_host_set_threads(n=-1):
    return None


def spmm_host_set_pipeline(chunks=16, slots=4):
    return None


def host_narrow(src, dst):
    dst[...] = src.astype(np.int32)
    return dst


# ---- K10-K15: the sparse-tensor ops; K11: masked SpGEMM (stand-ins in their own modules) --------------------------
from _mock_masked import keys_member, masked_spgemm, masked_spgemm_set_stage, masked_spgemm_sorted  # noqa: E402,F401
from _mock_tensor import cp_completion_mode, mttkrp_mode, ttm_mode, ttm_mode_long_flags, ttmc_mode, tttp  # noqa: E402,F401

_NAMES = [k for k, v in list(globals().items()) if callable(v) and not k.startswith("_") and hasattr(Kn, k)
          and k not in ("n", "T", "bits_ne", "install", "uninstall")]


# wrappers whose REAL counterpart passes a b2s_dtype code for its value tensors: the mock applies the same dtype
# matrix (D.dtype_code raises TypeError for anything else), so storage-only dtypes cannot slip through on CPU only
_CODED = {"spmm_csr_dense", "segment_sum", "spgemm", "spmm_csr_dense_flagged", "dense_to_csr", "ew_merge_fused",
          "ew_map", "ew_dense", "reduce_fused", "sddmm", "mttkrp"}


def _strict(name, fn):
    import functools

    @functools.wraps(fn)
    def checked(*args, **kwargs):
        for a in args:
            if isinstance(a, torch.Tensor) and a.dtype not in (torch.int32, torch.int64, torch.uint8) \
                    and not (a.dtype == torch.bool and name in ("dense_to_csr",)):
                D.dtype_code(D.np_dtype(a))
        return fn(*args, **kwargs)

    return checked


_IDX = (torch.int32, torch.int64)


def _need_idx(t, what):
    if isinstance(t, torch.Tensor) and t.dtype not in _IDX:
        raise TypeError(f"mock: {what} must be int32 / int64 on the device (the kernels take idx_bytes 4 or 8), "
                        f"got {t.dtype}")


def _need_i64(t, what):
    if isinstance(t, torch.Tensor) and t.dtype != torch.int64:
        raise TypeError(f"mock: {what} must be int64, got {t.dtype}")


def _need_np_idx(dt, what):
    if np.dtype(dt) not in (np.dtype(np.int32), np.dtype(np.int64)):
        raise TypeError(f"mock: {what} must be int32 / int64, got {np.dtype(dt)}")


# the argument contracts of the real wrappers (sparse_b200/_kernels.py) that NumPy would silently accept
_CONTRACTS = {
    "linearize": lambda a, k: _need_idx(a[0], "coords"),
    "diag_flags": lambda a, k: _need_idx(a[0], "coords"),
    "unravel": lambda a, k: (_need_i64(a[0], "keys"), _need_np_idx(a[2] if len(a) > 2 else k.get("idx_dtype", np.int64), "idx_dtype")),
    "slice_keys": lambda a, k: _need_i64(a[0], "keys"),
    "keys_flags": lambda a, k: _need_i64(a[0], "keys"),
    "sort_keys": lambda a, k: _need_i64(a[0], "keys"),
    "flag_heads": lambda a, k: _need_i64(a[0], "keys"),
    "gather": lambda a, k: _need_i64(a[1], "perm"),
    "gather_rows": lambda a, k: _need_i64(a[1], "perm"),
    "scatter": lambda a, k: _need_i64(a[1], "keys"),
    "compact_rows": lambda a, k: _need_idx(a[0], "coordinate rows"),
    "csr_from_keys": lambda a, k: (_need_i64(a[0], "keys"), _need_np_idx(a[3] if len(a) > 3 else k.get("idx_dtype", np.int64), "idx_dtype")),
    "rows_from_indptr": lambda a, k: (_need_idx(a[0], "indptr"), _need_np_idx(a[2] if len(a) > 2 else k.get("idx_dtype", np.int64), "idx_dtype")),
    "indptr_from_sorted": lambda a, k: _need_np_idx(a[2] if len(a) > 2 else k.get("idx_dtype", np.int64), "idx_dtype"),
    "indptr_remap": lambda a, k: _need_idx(a[0], "indptr"),
    "spmm_csr_dense": lambda a, k: (_need_idx(a[1], "indices"), _need_idx(a[2], "indptr")),
    "spmm_csr_dense_flagged": lambda a, k: (_need_idx(a[1], "indices"), _need_idx(a[2], "indptr")),
    "spgemm": lambda a, k: [_need_idx(a[i], "index array") for i in (0, 1, 3, 4)],
    "ew_merge_fused": lambda a, k: (_need_i64(a[1], "keys_a"), _need_i64(a[4], "keys_b")),
    "ew_dense": lambda a, k: _need_i64(a[2], "keys"),
    "ew_expand": lambda a, k: _need_idx(a[0], "coords"),
    "reduce_fused": lambda a, k: _need_i64(a[1], "keys"),
}


def _contract(name, fn):
    import functools

    check = _CONTRACTS[name]

    @functools.wraps(fn)
    def checked(*args, **kwargs):
        check(args, kwargs)
        return fn(*args, **kwargs)

    return checked


def install():
    """Route sparse_b200 through the NumPy mock (CPU torch tensors)."""
    if _ORIG:
        return
    D._TEST_CPU = True
    for name in _NAMES:
        _ORIG[name] = getattr(Kn, name)
        fn = globals()[name]
        if name in _CONTRACTS:
            fn = _contract(name, fn)
        setattr(Kn, name, _strict(name, fn) if name in _CODED else fn)


def uninstall():
    for name, fn in _ORIG.items():
        setattr(Kn, name, fn)
    _ORIG.clear()
    D._TEST_CPU = False
