"""Fused SDDMM and MTTKRP: the reference's two example paths as single device kernels.

* sddmm(s, a, b)   == s * (a @ b)                       (examples/sddmm_example.py:51-52)
* mttkrp(B, D, C)  == sparse.sum(B[:, :, :, None] * D[None, None, :, :] * C[None, :, None, :], axis=(1, 2))
                                                        (examples/mttkrp_example.py:51-52)
The unfused expressions also run (through elemwise + reduce); these entry points avoid the dense (a @ b)
intermediate and the nnz x J broadcast products.  Floating-point association differs from the reference's
BLAS / reduceat order, so parity is tolerance-based (rtol 1e-5 f32, 1e-12 f64 in the tests).

mttkrp_mode(X, factors, mode) generalises mttkrp to any mode of a tensor of order 2..8 (the CP-ALS step); it has no
counterpart in the reference beyond the unfused broadcast expression / einsum.  ttmc_mode(X, factors, mode) is its
Kronecker counterpart, the TTMc step of Tucker / HOOI, with the same inputs and a rank per mode.  tttp(X, factors)
evaluates a CP model at X's stored entries (X * [[U_0, ..., U_{N-1}]], the order-N sddmm) and keeps X's pattern.
ttm_mode(X, U, mode) is the mode-n tensor times matrix (or vector) with a sparse result: tensordot(X, U, axes=([mode],
[0])) bit for bit, in O(nnz + result) memory instead of a dense intermediate over the other extents.
cp_completion_mode(X, factors, mode, reg) is the row-wise least-squares ALS update of CP completion, and
cp_apr_phi_mode(X, factors, mode, eps) the ratio MTTKRP of Poisson CP (CP-APR): mttkrp_mode of X / max(model, eps)
at X's entries, fused on the same cached mode stream.
sptc(X, Y, axes) is tensordot for two sparse tensors with a sparse result, bit for bit, on rows that exist only where
there are entries: its memory does not depend on the extents.

masked_matmul(mask, a, b) == mask * (a @ b) at mask's stored positions, for sparse a and b: the masked SpGEMM of
examples/triangles_example.py (sum(a @ a * a) / 6) and of the GraphBLAS masked mxm.  It never forms the product
a @ b, so its memory is O(nnz(mask)), and it is bit-identical to the unfused expression on the mask's pattern.
"""
from __future__ import annotations

import operator

import numpy as np
from numpy.exceptions import AxisError

from . import _device as D
from . import _kernels as Kn
from ._coo import COO
from ._dot import _coo_as_csr, _csr_arrays, _dense_dev, _narrow_idx, _return_dense
from ._sparse_array import SparseArray
from ._utils import check_zero_fill_value


def _dense_dt(x):
    return x.dtype if isinstance(x, np.ndarray) else D.np_dtype(x)


def sddmm(s, a, b, *, b_transposed=False):
    """Sampled dense-dense matrix product: ``s * (a @ b)`` for sparse 2-D ``s`` and dense ``a`` (M,K), ``b`` (K,N).
    With ``b_transposed=True`` `b` is given as b^T (N,K), the layout the kernel gathers from."""
    from ._gcxs import GCXS

    if not isinstance(s, SparseArray) or s.ndim != 2:
        raise TypeError("sddmm: `s` must be a 2-D sparse_b200 array")
    check_zero_fill_value(s)
    M, N = s.shape
    if b_transposed:
        bN, bK = int(b.shape[0]), int(b.shape[1])
    else:
        bK, bN = int(b.shape[0]), int(b.shape[1])
    if a.ndim != 2 or b.ndim != 2 or a.shape[0] != M or bN != N or a.shape[1] != bK:
        raise ValueError(f"sddmm: shape mismatch s{s.shape}, a{tuple(a.shape)}, b{tuple(b.shape)}")
    K = int(a.shape[1])
    T = np.result_type(s.dtype, _dense_dt(a), _dense_dt(b))
    if T not in (np.dtype("float32"), np.dtype("float64")):
        raise TypeError(f"sddmm: dtype {T} is outside the CUDA dtype matrix (float32, float64)")
    was_gcxs = isinstance(s, GCXS)
    c = s.tocoo() if was_gcxs else s
    vals, cols, indptr = _coo_as_csr(c, T)
    ad = _dense_dev(a, T)
    bt = _dense_dev(b, T) if b_transposed else Kn.transpose_dense(_dense_dev(b, T))  # (N, K): contiguous gathers
    out = Kn.sddmm(indptr, cols, vals, ad, bt, M, N, K)
    fill = T.type(0)
    if isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and M and N and K:
        # the unfused expression's fill value is `0 * (a @ b)[0, 0]` (_umath.py:520-527: the first element of
        # func(fill, ndarray)), i.e. -0.0 when that corner is negative -- and the prune test below is by bit pattern,
        # so the sign decides WHICH zeros stay stored.  K multiply-adds on the host; device operands keep +0.0
        # (no read-back on the asynchronous path)
        with np.errstate(all="ignore"):
            corner = np.dot(a[0].astype(T, copy=False), (b[0] if b_transposed else b[:, 0]).astype(T, copy=False))
            if np.isfinite(corner):
                fill = T.type(T.type(0) * (corner + T.type(0)))  # a sum that starts at +0.0 is never -0.0
    res = COO._from_device(c._coords, out, s.shape, fill, keys=c.sorted_keys())
    res._canonicalise(check_sort=False, sum_dups=False, prune=True)  # s * dense drops exact zeros (_umath.py:627-633)
    return res.asformat("gcxs", compressed_axes=s.compressed_axes) if was_gcxs else res


def mttkrp(B, Dm, Cm):
    """Matricised tensor times Khatri-Rao product: out[i, j] = sum_{k,l} B[i,k,l] * D[l,j] * C[k,j]."""
    from ._gcxs import GCXS

    if not isinstance(B, SparseArray) or B.ndim != 3:
        raise TypeError("mttkrp: `B` must be a 3-D sparse_b200 array")
    check_zero_fill_value(B)
    I_, K_, L_ = B.shape
    if Dm.ndim != 2 or Cm.ndim != 2 or Dm.shape[0] != L_ or Cm.shape[0] != K_ or Dm.shape[1] != Cm.shape[1]:
        raise ValueError(f"mttkrp: shape mismatch B{B.shape}, D{tuple(Dm.shape)}, C{tuple(Cm.shape)}")
    J = int(Dm.shape[1])
    T = np.result_type(B.dtype, _dense_dt(Dm), _dense_dt(Cm))
    if T not in (np.dtype("float32"), np.dtype("float64")):
        raise TypeError(f"mttkrp: dtype {T} is outside the CUDA dtype matrix (float32, float64)")
    was_gcxs = isinstance(B, GCXS)
    c = B.tocoo() if was_gcxs else B
    coords, data = c._dev()
    c.sorted_keys()
    lead = coords[0].contiguous()
    indptr = Kn.indptr_from_sorted(lead, I_, D.np_dtype(coords))
    kk, ll, indptr = _narrow_idx(coords[1].contiguous(), coords[2].contiguous(), indptr, limit=max(K_, L_, c.nnz))
    out = Kn.mttkrp(indptr, kk, ll, Kn.cast(data, T), _dense_dev(Dm, T), _dense_dev(Cm, T), I_, J)
    rows, cols, vals, _ = Kn.dense_to_csr(out, mode=1, want_rows=True, want_indptr=False)
    t = D.torch()
    res = COO._from_device(t.stack([rows, cols]), vals, (I_, J), T.type(0))
    return GCXS.from_coo(res) if was_gcxs else res


# Test hook: True keeps the mode streams' coordinates int64 even when every extent and nnz fit int32.
_FORCE_WIDE_INDEX = False


def _index_limit(X):
    """The largest value X's coordinate arrays must hold: int32 suffices below 2**31 - 1."""
    return 2**63 if _FORCE_WIDE_INDEX else max(*X.shape, X.nnz)


def _mode_stream(X, mode):
    """Coordinate rows (a list of N device index tensors) and values of X's entries in the order of the mode stream
    S_mode: C order for mode 0, C order sorted stably by coordinate `mode` otherwise.  Cached on X per mode."""
    from ._gcxs import GCXS
    from ._utils import key_bits

    limit = _index_limit(X)
    key = (mode, limit < 2**31 - 1)
    cache = X._mode_streams
    if cache is not None and key in cache:
        return cache[key]
    c = X.tocoo() if isinstance(X, GCXS) else X
    coords, vals = c._dev()
    rows = [coords[m].contiguous() for m in range(X.ndim)]
    if mode != 0:
        sorted_rows, perm = Kn.sort_keys(Kn.cast(rows[mode], np.int64), key_bits(X.shape[mode]))
        rows = [sorted_rows if m == mode else Kn.gather(rows[m], perm) for m in range(X.ndim)]
        vals = Kn.gather(vals, perm)
    stream = (_narrow_idx(*rows, limit=limit), vals)
    if cache is None:
        cache = X._mode_streams = {}
    cache[key] = stream
    return stream


def _tensor_and_mode(name, X, mode):
    """Checks of the tensor operand shared by the sparse-tensor ops: (order N, mode in 0..N-1, or None for None)."""
    from ._gcxs import GCXS

    if not isinstance(X, (COO, GCXS)):
        raise TypeError(f"{name}: `X` must be a sparse_b200 COO or GCXS array")
    N = X.ndim
    if not 2 <= N <= 8:
        raise ValueError(f"{name}: order {N} outside 2..8")
    check_zero_fill_value(X)
    if mode is not None:
        mode = operator.index(mode)
        if not -N <= mode < N:
            raise AxisError(mode, N)
        mode %= N
    return N, mode


def _tensor_and_factors(name, X, factors, mode, one_rank):
    """Checks shared by mttkrp_mode, ttmc_mode and tttp: (order N, mode in 0..N-1, the factors as a list with the other
    modes' ones as NumPy arrays or device tensors, the other modes ascending, the result dtype T, the ranks: a list of N
    with ranks[m] = factors[m].shape[1] for the other modes and 0 for `mode`).  `mode` None (tttp) reads every factor.
    With `one_rank` every factor read must have the same number of columns."""
    N, mode = _tensor_and_mode(name, X, mode)
    factors = list(factors)
    if len(factors) != N:
        raise ValueError(f"{name}: {len(factors)} factors for an order-{N} tensor")
    others = [m for m in range(N) if m != mode]
    if mode is None:
        for m in others:
            if factors[m] is None:
                raise ValueError(f"{name}: factor {m} is None ({name} reads every factor)")
    for m in others:
        if not D.is_device_tensor(factors[m]):
            factors[m] = np.asarray(factors[m])
    ranks = [0] * N
    R = int(factors[others[0]].shape[1]) if factors[others[0]].ndim == 2 else -1
    for m in others:
        f = factors[m]
        if f.ndim != 2 or int(f.shape[0]) != X.shape[m] or (one_rank and int(f.shape[1]) != R):
            expected = f"({X.shape[m]}, R) with one R for all factors" if one_rank else f"({X.shape[m]}, R_{m})"
            raise ValueError(f"{name}: shape mismatch X{X.shape}, factor {m} {tuple(f.shape)} (expected {expected})")
        ranks[m] = int(f.shape[1])
    T = np.result_type(X.dtype, *(_dense_dt(factors[m]) for m in others))
    if T not in (np.dtype("float32"), np.dtype("float64")):
        raise TypeError(f"{name}: dtype {T} is outside the CUDA dtype matrix (float32, float64)")
    return N, mode, factors, T, ranks


def _mode_product(X, factors, mode, T, W, empty, kernel, *args):
    """The dense (X.shape[mode], W) result of mttkrp_mode / ttmc_mode / cp_completion_mode after their checks: `empty`
    when nothing is stored, else `kernel(coords, vals, factors, mode, rows, *args)` over the cached mode stream."""
    N, rows = X.ndim, X.shape[mode]
    if X.nnz == 0 or rows == 0 or W == 0:
        out = Kn.full(rows * W, empty, T).reshape(rows, W)
    else:
        coords, vals = _mode_stream(X, mode)
        fac = [None if m == mode else _dense_dev(factors[m], T) for m in range(N)]
        out = kernel(coords, Kn.cast(vals, T), fac, mode, rows, *args)
    return _return_dense(out, [f for f in factors if f is not None])


def mttkrp_mode(X, factors, mode):
    """Mode-`mode` MTTKRP of a sparse tensor: the product of the mode-`mode` matricisation of `X` with the Khatri-Rao
    product of every other factor, the step CP-ALS runs once per mode and iteration.

        out[i, r] = sum over stored entries e with i_mode(e) = i of  v_e * prod_{m != mode} factors[m][i_m(e), r]

    `X` is a COO or GCXS of order 2..8 with a zero fill value.  `factors` holds N dense 2-D arrays (NumPy arrays or
    CUDA tensors), `factors[m]` of shape (X.shape[m], R) with one R for all; `factors[mode]` is never read and may be
    None.  `mode` counts from the end when negative.  The result is dense, (X.shape[mode], R), of dtype
    result_type(X.dtype, other factor dtypes) (float32 or float64): a NumPy array, or a CUDA tensor when a factor is
    one.

    The summation order is fixed (include/sparse_b200.h, b2s_mttkrp_mode), so results are reproducible bit for bit.
    Product association differs from `mttkrp`, so the two agree to rounding, not bit for bit.

    Memory: the entries ordered by coordinate `mode` are cached on `X` for the next call with the same mode (they are
    dropped when X's contents are replaced, and are not copied or pickled).  A cached mode holds
    (N * index bytes + value bytes) * nnz of device memory -- index bytes 4 when every extent and nnz fit int32, else 8.
    """
    N, mode, factors, T, ranks = _tensor_and_factors("mttkrp_mode", X, factors, mode, True)
    R = max(ranks)  # the one R of the other factors (ranks[mode] is 0)
    return _mode_product(X, factors, mode, T, R, 0, Kn.mttkrp_mode, R)


def ttmc_mode(X, factors, mode):
    """Mode-`mode` TTMc (tensor times matrix chain) of a sparse tensor: X multiplied by the transpose of every factor but
    `factors[mode]`, matricised along `mode`, the step HOOI (Tucker decomposition) runs once per mode and iteration.

        out[i, col] = sum over stored entries e with i_mode(e) = i of  v_e * prod_{m != mode} factors[m][i_m(e), r_m]

    `X` is a COO or GCXS of order 2..8 with a zero fill value.  `factors` holds N dense 2-D arrays (NumPy arrays or
    CUDA tensors), `factors[m]` of shape (X.shape[m], R_m), each mode with its own R_m; `factors[mode]` is never read
    and may be None.  `mode` counts from the end when negative.  The result is dense, (X.shape[mode], W) with
    W = prod_{m != mode} R_m, of dtype result_type(X.dtype, other factor dtypes) (float32 or float64): a NumPy array,
    or a CUDA tensor when a factor is one.

    Columns are in C order over the other modes, ascending: with a < b < ... the modes other than `mode`,
    col = ((r_a * R_b + r_b) * R_c + r_c) ..., so `out.reshape(X.shape[mode], R_a, R_b, ...)` is
    `np.einsum` of X with the factors and output subscripts "i" + "abc...".  HOOI takes the leading R_mode left
    singular vectors of `out`, which do not depend on the column order.  W is at most `_kernels.ttmc_mode_max_width()`
    (2,097,120: the combine kernel's launch geometry); a larger W raises ValueError before anything is allocated.

    The summation order is fixed (include/sparse_b200.h, b2s_ttmc_mode), so results are reproducible bit for bit.
    With every R_m = R, the columns (r, r, ..., r) equal `mttkrp_mode`'s column r bit for bit.

    Memory: the result, rows * W * itemsize; the mode stream of `mode`, cached on `X` and shared with `mttkrp_mode`
    ((N * index bytes + value bytes) * nnz, as described there); and, during the call, a scratch array of
    2 * ceil(nnz / 512) * W' * itemsize bytes (W' = W rounded up to a multiple of 4) for the rows that cross chunks.
    """
    N, mode, factors, T, ranks = _tensor_and_factors("ttmc_mode", X, factors, mode, False)
    W = int(np.prod([ranks[m] for m in range(N) if m != mode], dtype=object))
    if W > Kn.ttmc_mode_max_width():
        raise ValueError(f"ttmc_mode: {W} output columns (the product of the other modes' ranks) exceed the limit of "
                         f"{Kn.ttmc_mode_max_width()}")
    return _mode_product(X, factors, mode, T, W, 0, Kn.ttmc_mode, ranks)


def _gcxs_coords(X, limit):
    """Per-axis coordinates of a GCXS's entries in its stored order: the compressed row of each entry from `indptr`,
    the row and `indices` unravelled over the compressed and the other axes, put back in axis order.  No sort."""
    _, indices, indptr = X._dev()
    idt = np.int32 if limit < 2**31 - 1 else np.int64
    rs, k = X._reordered_shape, X._axisptr
    lead = Kn.unravel(Kn.rows_from_indptr(indptr, X.nnz, np.int64), rs[:k], idt)
    rest = Kn.unravel(Kn.cast(indices, np.int64), rs[k:], idt)
    coords = [None] * X.ndim
    for pos, a in enumerate(X._axis_order):
        coords[a] = lead[pos] if pos < k else rest[pos - k]
    return coords


def tttp(X, factors):
    """A sparse tensor times a CP (Kruskal) model at its stored entries, ``X * [[U_0, ..., U_{N-1}]]`` (TTTP, the
    order-N SDDMM): the model's residual, loss derivative or ratio at the observed entries that tensor completion, GCP
    and CP-APR need, without forming the dense model or the nnz x R broadcast products.

        z_e = v_e * sum_r  U_0[i_0(e), r] * U_1[i_1(e), r] * ... * U_{N-1}[i_{N-1}(e), r]

    `X` is a COO or GCXS of order 2..8 with a zero fill value.  `factors` holds N dense 2-D arrays (NumPy arrays or CUDA
    tensors, which may be mixed), `factors[m]` of shape (X.shape[m], R) with one R for all (R = 0 gives v_e * +0); every
    factor is read.  The result has X's format and shape (a GCXS keeps ``X.compressed_axes``), dtype
    result_type(X.dtype, factor dtypes) (float32 or float64) and fill value +0.  It stores X's entries except those
    whose z_e is bitwise +0; stored -0.0 and NaN results stay (the prune rule of `sddmm` and `masked_matmul`).  At order
    2 it equals ``sddmm(X, U_0, U_1, b_transposed=True)`` to rounding (K8 sums in another order).

    The order of operations is fixed (include/sparse_b200.h, b2s_tttp): for each r the product in ascending mode order,
    the sum over r ascending from +0, then one multiply by v_e; results are reproducible bit for bit.  With that order,
    CP weights lam fold into the first factor: ``tttp(X, [U_0 * lam, U_1, ...])`` has the bits of a kernel that starts
    each product with lam_r, ((lam_r * U_0) * U_1) * ..., so there is no weights argument.

    One difference from the unfused ``X * model``: its fill value is ``0 * model[0, ..., 0]``, which is -0.0 when that
    corner of the model is negative; tttp always returns +0, as `masked_matmul` does.

    Entries are taken in place, with no sort: a COO in its canonical order (the mode-0 stream that `mttkrp_mode` also
    uses and caches), a GCXS in its stored order, and the GCXS result shares X's index arrays unless entries are pruned.
    A GCXS whose rows repeat an index gets one product per stored entry.  Memory: the result values, plus N coordinate
    arrays of nnz entries for a GCXS during the call.
    """
    from ._gcxs import GCXS

    _, _, factors, T, ranks = _tensor_and_factors("tttp", X, factors, None, True)
    R = ranks[0]
    if isinstance(X, GCXS):
        data, indices, indptr = X._dev()
        if X.nnz == 0:
            out = Kn.full(0, 0, T)
        else:
            out = Kn.tttp(_gcxs_coords(X, _index_limit(X)), Kn.cast(data, T), [_dense_dev(f, T) for f in factors], R)
        res = GCXS._from_device(out, indices, indptr, X.shape, X.compressed_axes, T.type(0))
        res._idx_vis = X._idx_vis
        res._prune()  # drops results that are bitwise +0, as X * model does
        return res
    if X.nnz == 0:
        out = Kn.full(0, 0, T)
    else:
        coords, vals = _mode_stream(X, 0)
        out = Kn.tttp(coords, Kn.cast(vals, T), [_dense_dev(f, T) for f in factors], R)
    res = COO._from_device(X._dev()[0], out, X.shape, T.type(0), keys=X._keys)
    res._canonicalise(check_sort=False, sum_dups=False, prune=True)  # drops bitwise +0 results, as X * model does
    return res


def cp_completion_mode(X, factors, mode, reg):
    """One ALS update of CP tensor completion: the new factor of mode `mode`, each row the solution of its own
    regularised least-squares problem over the entries observed in that row.

        h_e[r] = prod_{m != mode} factors[m][i_m(e), r]           (the Khatri-Rao row of entry e)
        (sum_{e in row i} h_e h_e^T + reg * I) u_i = sum_{e in row i} v_e h_e,      out[i] = u_i

    `X` is a COO or GCXS of order 2..8 with a zero fill value; its stored entries are the observed set, stored zeros
    included (a COO built with the default ``prune=False`` keeps them, and they count as observations of 0).
    `factors` is as for `mttkrp_mode`: N dense 2-D arrays (NumPy arrays or CUDA tensors, which may be mixed),
    `factors[m]` of shape (X.shape[m], R) with one R for all; `factors[mode]` is not read and may be None.  `reg` is a
    finite real >= 0, cast to the result dtype.  The result is dense, (X.shape[mode], R), of dtype
    result_type(X.dtype, other factor dtypes) (float32 or float64): a NumPy array, or a CUDA tensor when a factor is
    one.  R is at most `_kernels.cp_completion_max_rank()` (64); a larger R raises ValueError before anything is
    allocated.

    A row without entries is the solution of reg * I u = 0: zero for reg > 0, NaN for reg = 0.  A row whose
    Cholesky factorisation meets a pivot that is not positive (a rank-deficient row at reg = 0, or NaN / inf inputs)
    comes back as all NaN; the other rows are unaffected.

    The order of operations is fixed (include/sparse_b200.h, b2s_cp_completion_mode), so results are reproducible bit
    for bit; the right-hand side sum_e v_e h_e is `mttkrp_mode(X, factors, mode)[i]` bit for bit.

    An ALS sweep, with `tttp` for the training loss:

        for it in range(sweeps):
            for n in range(X.ndim):
                U[n] = cp_completion_mode(X, U, n, reg)
            P = COO(X.coords, np.ones(X.nnz), shape=X.shape)             # X's pattern with ones
            resid = tttp(P, U) - X
            loss = 0.5 * (resid.data ** 2).sum() + 0.5 * reg * sum((u ** 2).sum() for u in U)

    Memory: the mode stream of `mode`, cached on `X` and shared with `mttkrp_mode` (not rebuilt); the result,
    rows * R * itemsize; and, during the call, a scratch array of 2 * ceil(nnz / 512) * W * itemsize bytes
    (W = R(R+1)/2 + R rounded up to a multiple of 4) for the rows that cross chunks.  No (rows, R^2) array is formed.
    """
    N, mode, factors, T, ranks = _tensor_and_factors("cp_completion_mode", X, factors, mode, True)
    R = max(ranks)
    if isinstance(reg, (bool, np.bool_)) or not isinstance(reg, (int, float, np.integer, np.floating)):
        raise TypeError(f"cp_completion_mode: `reg` must be a real number, got {type(reg).__name__}")
    with np.errstate(over="ignore"):
        reg_t = T.type(reg)
    if not np.isfinite(reg_t) or reg_t < 0:
        raise ValueError(f"cp_completion_mode: `reg` must be finite and >= 0 in {T}, got {reg!r}")
    if R > Kn.cp_completion_max_rank():
        raise ValueError(f"cp_completion_mode: R = {R} exceeds the limit of {Kn.cp_completion_max_rank()}")
    return _mode_product(X, factors, mode, T, R, 0 if reg_t > 0 else np.nan, Kn.cp_completion_mode, R, float(reg_t))


def cp_apr_phi_mode(X, factors, mode, eps=1e-10):
    """The ratio MTTKRP Phi of Poisson CP (CP-APR, Chi & Kolda 2012): the product of the mode-`mode` matricisation of
    X / max(model, eps), taken at X's stored entries, with the Khatri-Rao product of every other factor -- the kernel
    that CP-APR's multiplicative update runs up to l_max times per mode and outer iteration.

        m_e      = sum_r prod_m factors[m][i_m(e), r]             (the CP model at entry e, factors[mode] included)
        out[i, r] = sum over stored entries e with i_mode(e) = i of  v_e / max(m_e, eps) * prod_{m != mode} factors[m][i_m(e), r]

    `X` is a COO or GCXS of order 2..8 with a zero fill value.  `factors` holds N dense 2-D arrays (NumPy arrays or CUDA
    tensors, which may be mixed), `factors[m]` of shape (X.shape[m], R) with one R for all; every factor is read,
    `factors[mode]` (B, the factor being updated, with the weights absorbed) included.  `eps` is a finite real >= 0,
    cast to the result dtype.  The result is dense, (X.shape[mode], R), of dtype result_type(X.dtype, factor dtypes)
    (float32 or float64): a NumPy array, or a CUDA tensor when a factor is one.  Rows without entries are +0.  R is at
    most `_kernels.cp_apr_phi_max_rank()` (64); a larger R raises ValueError before anything is allocated.

    CP-APR expects X >= 0 and nonnegative factors; signs are not checked (that would read the data back from the
    device), and the formula is computed for any inputs.  One difference from MATLAB's ``max(M, eps)``: a NaN model
    value stays NaN rather than becoming eps, so that a NaN in the model shows up instead of turning into v / eps.

    The order of operations is fixed (include/sparse_b200.h, b2s_cp_apr_phi_mode), so results are reproducible bit for
    bit.  m_e is `tttp(P, factors)` at e bit for bit (P: X's pattern with ones), and the result is
    ``mttkrp_mode(COO(X.coords, w), factors, mode)`` bit for bit, with w_e = v_e / max(m_e, eps) correctly rounded.

    One CP-APR multiplicative-update (MU) sweep over the modes, the factors' columns summing to 1 and the weights lam
    absorbed into the mode being updated:

        for n in range(X.ndim):
            B = U[n] * lam
            for it in range(l_max):                            # inner iterations, typically 10
                Phi = cp_apr_phi_mode(X, U[:n] + [B] + U[n + 1:], n, eps)
                if np.abs(np.minimum(B, 1 - Phi)).max() < tol:  # the KKT test
                    break
                B = B * Phi                                    # the multiplicative update
            lam = B.sum(axis=0)                                # column normalisation
            U[n] = B / lam
        P = COO(X.coords, np.ones(X.nnz), shape=X.shape)       # X's pattern with ones
        m = tttp(P, [U[0] * lam] + U[1:]).data                 # the model at X's entries (positive, so all stored)
        nll = lam.sum() - (X.data * np.log(m)).sum()           # the negative log-likelihood

    Memory: the mode stream of `mode`, cached on `X` and shared with `mttkrp_mode`, `ttmc_mode` and
    `cp_completion_mode` (not rebuilt); the result, rows * R * itemsize; and, during the call, a scratch array of
    2 * ceil(nnz / 512) * R' * itemsize bytes (R' = R rounded up to a multiple of 4) for the rows that cross chunks,
    plus an aligned copy of any factor whose rows are not 16-byte aligned or whose R is not a multiple of
    16 / itemsize.  No nnz-sized intermediate is formed.
    """
    name = "cp_apr_phi_mode"
    N, _, factors, T, ranks = _tensor_and_factors(name, X, factors, None, True)
    _, mode = _tensor_and_mode(name, X, mode)
    R = ranks[0]
    if isinstance(eps, (bool, np.bool_)) or not isinstance(eps, (int, float, np.integer, np.floating)):
        raise TypeError(f"{name}: `eps` must be a real number, got {type(eps).__name__}")
    with np.errstate(over="ignore"):
        eps_t = T.type(eps)
    if not np.isfinite(eps_t) or eps_t < 0:
        raise ValueError(f"{name}: `eps` must be finite and >= 0 in {T}, got {eps!r}")
    if R > Kn.cp_apr_phi_max_rank():
        raise ValueError(f"{name}: R = {R} exceeds the limit of {Kn.cp_apr_phi_max_rank()}")
    rows = X.shape[mode]
    if X.nnz == 0 or rows == 0 or R == 0:
        out = Kn.full(rows * R, 0, T).reshape(rows, R)
    else:
        coords, vals = _mode_stream(X, mode)
        fac = [_dense_dev(f, T) for f in factors]
        out = Kn.cp_apr_phi_mode(coords, Kn.cast(vals, T), fac, mode, rows, R, float(eps_t))
    return _return_dense(out, factors)


# Fibers with more entries than this get whole CTAs in b2s_ttm_mode (a module value so that tests can move it).
_TTM_LONG_FIBER = 512


def _long_fibers(X, mode, fptr):
    """The ascending indices (int64) of the fibers of `mode` with more than _TTM_LONG_FIBER entries; cached next to the
    fiber stream."""
    key = ("fiber-long", mode, _index_limit(X) < 2**31 - 1, _TTM_LONG_FIBER)
    if key not in X._mode_streams:
        flags = Kn.ttm_mode_long_flags(fptr, _TTM_LONG_FIBER)
        pos, n = Kn.scan_flags(flags)
        X._mode_streams[key] = Kn.compact(Kn.iota(flags.shape[0]), flags, pos, n)
    return X._mode_streams[key]


def _fiber_stream(X, mode):
    """The fiber stream of `mode` (the inputs of b2s_ttm_mode): (kcoord, vals, fptr, fgroup, gptr, fkey, pkey).

    Entries are ordered by the key over the axes (other modes ascending, then `mode`): X's canonical order when `mode`
    is the last axis, one stable sort otherwise.  Fibers (runs sharing every coordinate but `mode`) and groups (runs of
    fibers sharing the coordinates before `mode`) come from the flag / scan / compact primitives.  Cached on X under
    ("fiber", mode, int32 indices), apart from the mode streams of mttkrp_mode and dropped with them."""
    from ._gcxs import GCXS
    from ._utils import c_strides, key_bits

    limit = _index_limit(X)
    key = ("fiber", mode, limit < 2**31 - 1)
    cache = X._mode_streams
    if cache is not None and key in cache:
        return cache[key]
    c = X.tocoo() if isinstance(X, GCXS) else X
    N, shape, nnz = X.ndim, X.shape, X.nnz
    coords, vals = c._dev()
    if mode == N - 1:
        pc = coords  # canonical order is already the fiber stream's
    else:
        axes = [m for m in range(N) if m != mode] + [mode]
        pshape = [shape[a] for a in axes]
        strides = [0] * N
        for a, s in zip(axes, c_strides(pshape)):
            strides[a] = s
        keys, perm = Kn.sort_keys(Kn.linearize(coords, strides), key_bits(X.size))
        pc = Kn.unravel(keys, pshape, np.int64)  # rows: the other modes ascending, then `mode`
        vals = Kn.gather(vals, perm)
    fkey = Kn.linearize(pc[:N - 1], c_strides([shape[m] for m in range(N) if m != mode]))
    pkey = Kn.linearize(pc[:mode], c_strides(shape[:mode])) if mode else Kn.full(nnz, 0, np.int64)
    heads = Kn.flag_heads(fkey)
    pos, nf = Kn.scan_flags(heads)
    fstart = Kn.compact(Kn.iota(nnz), heads, pos, nf)
    fkey, pkey = Kn.compact(fkey, heads, pos, nf), Kn.compact(pkey, heads, pos, nf)
    gheads = Kn.flag_heads(pkey)
    gpos, ng = Kn.scan_flags(gheads)
    t = D.torch()
    gptr = t.cat([Kn.compact(Kn.iota(nf), gheads, gpos, ng), Kn.full(1, nf, np.int64)])
    fgroup = Kn.rows_from_indptr(gptr, nf, np.int64)
    fptr = t.cat([fstart, Kn.full(1, nnz, np.int64)])
    kc, fptr, fgroup, gptr = _narrow_idx(pc[N - 1].contiguous(), fptr, fgroup, gptr, limit=limit)
    stream = (kc, vals, fptr, fgroup, gptr, fkey, pkey)
    if cache is None:
        cache = X._mode_streams = {}
    cache[key] = stream
    return stream


def ttm_mode(X, U, mode):
    """Mode-`mode` tensor times matrix (TTM) of a sparse tensor, ``X ×_mode Uᵀ``, with a sparse result; with a 1-D `U`,
    tensor times vector (TTV).  The step of Tucker / HOSVD built from a chain of TTMs, of projecting a tensor onto a basis
    along one mode, and of contracting one mode with a vector.

        Y[i_0, ..., r, ..., i_{N-1}] = sum_{i_mode} X[i_0, ..., i_mode, ..., i_{N-1}] * U[i_mode, r]

    `X` is a COO or GCXS of order 2..8 with a zero fill value; `mode` counts from the end when negative.  `U` is a NumPy
    array or a CUDA tensor: 2-D of shape (X.shape[mode], R), R >= 0, gives X's shape with axis `mode` replaced by R;
    1-D of shape (X.shape[mode],) gives X's shape with axis `mode` removed (order N - 1).  The dtype is
    result_type(X.dtype, U.dtype), float32 or float64.  The result is always a canonical COO with fill value +0.  A
    GCXS result is not offered: its indptr would span the product of the compressed extents, the size this op avoids.

    The order of operations is fixed (include/sparse_b200.h, b2s_ttm_mode): each value is ((+0 + v_1 * U[k_1, r]) +
    v_2 * U[k_2, r]) + ... over the mode-`mode` fiber's entries in ascending k, each product and sum rounded, and an
    entry is stored iff its value != 0 (+-0 are dropped, NaN is kept).  So for a COO X the result equals
    ``moveaxis(tensordot(X, U, axes=([mode], [0]), return_type=COO), -1, mode)`` (or the plain tensordot for a 1-D U)
    bit for bit, wherever that fits in memory: tensordot builds an indptr over the product of the other extents and a
    dense (that product x R) intermediate, where ttm_mode needs O(nnz + result).  For a GCXS X the result is
    ``ttm_mode(X.tocoo(), U, mode)`` bit for bit; GCXS tensordot sums in float64 and agrees only to rounding.

    Memory: the fiber stream of `mode` is cached on `X` for the next call with the same mode (dropped when X's contents
    are replaced, not copied or pickled): nnz * (index bytes + value bytes) + n_fibers * (3 * index bytes + 16), index
    bytes 4 when every extent and nnz fit int32, else 8, plus 8 bytes per fiber of more than 512 entries (such fibers
    get whole thread blocks, so skewed fiber lengths do not hold up the rest).  During the call, n_fibers * R * (value bytes + 17) bytes of
    slots before pruning, and the result, nnz(Y) * (value bytes + 8).  A result shape of 2**63 elements or more raises
    ValueError before anything is allocated.
    """
    N, mode = _tensor_and_mode("ttm_mode", X, mode)
    if not D.is_device_tensor(U):
        U = np.asarray(U)
    if U.ndim not in (1, 2) or int(U.shape[0]) != X.shape[mode]:
        raise ValueError(f"ttm_mode: shape mismatch X{X.shape}, U {tuple(U.shape)} (expected ({X.shape[mode]},) or "
                         f"({X.shape[mode]}, R) for mode {mode})")
    T = np.result_type(X.dtype, _dense_dt(U))
    if T not in (np.dtype("float32"), np.dtype("float64")):
        raise TypeError(f"ttm_mode: dtype {T} is outside the CUDA dtype matrix (float32, float64)")
    ttv = U.ndim == 1
    R = 1 if ttv else int(U.shape[1])
    shape = X.shape[:mode] + (() if ttv else (R,)) + X.shape[mode + 1:]
    if int(np.prod(shape, dtype=object)) >= 2**63:
        raise ValueError(f"ttm_mode: result shape {shape} has 2**63 elements or more (the COO index limit)")
    if X.nnz == 0 or R == 0:
        return COO._from_device(None, Kn.full(0, 0, T), shape, T.type(0), keys=Kn.full(0, 0, np.int64))
    kc, vals, fptr, fgroup, gptr, fkey, pkey = _fiber_stream(X, mode)
    long_ids = _long_fibers(X, mode, fptr)
    q_ext = int(np.prod(X.shape[mode + 1:], dtype=object))
    out, keys, flags = Kn.ttm_mode(kc, Kn.cast(vals, T), fptr, fgroup, gptr, fkey, pkey, long_ids, _TTM_LONG_FIBER,
                                   _dense_dev(U.reshape(-1, 1) if ttv else U, T), R, q_ext)
    pos, total = Kn.scan_flags(flags)
    if total != int(out.shape[0]):
        out, keys = Kn.compact(out, flags, pos, total), Kn.compact(keys, flags, pos, total)
    return COO._from_device(None, out, shape, T.type(0), keys=keys)


# Test hook: True keeps masked_matmul's index arrays int64 even when every extent and nnz fit int32.
_FORCE_WIDE_INDEX_MASKED = False

_MASKED_DTYPES = tuple(np.dtype(d) for d in ("float32", "float64", "int32", "int64"))

# Test hook: True keeps sptc's index arrays int64 even when every row count and nnz fit int32.
_FORCE_WIDE_INDEX_SPTC = False


def _sptc_axes(X, Y, axes):
    """The contracted axes of X and of Y as two lists of non-negative ints, paired in order: the `axes` forms, checks
    and errors of `tensordot`."""
    try:
        iter(axes)
    except TypeError:
        axes_x, axes_y = list(range(-axes, 0)), list(range(axes))
    else:
        axes_x, axes_y = axes
    axes_x = list(axes_x) if hasattr(axes_x, "__len__") else [axes_x]
    axes_y = list(axes_y) if hasattr(axes_y, "__len__") else [axes_y]
    if X.ndim == 0 or Y.ndim == 0:
        raise ValueError(f"Input {int(X.ndim != 0)} operand does not have enough dimensions")
    equal = len(axes_x) == len(axes_y)
    for k in range(len(axes_x) if equal else 0):
        if X.shape[axes_x[k]] != Y.shape[axes_y[k]]:
            equal = False
            break
        axes_x[k] %= X.ndim
        axes_y[k] %= Y.ndim
    if not equal or len(set(axes_x)) != len(axes_x) or len(set(axes_y)) != len(axes_y):
        raise ValueError("shape-mismatch for sum")
    return axes_x, axes_y


def _sptc_stream(X, free, con, side, narrow):
    """One operand of sptc as doubly-compressed CSR, cached on X under ("sptc", side, contracted axes, int32 indices)
    and dropped with the other streams.  The entries are ordered by the key over (free axes, contracted axes) for side
    "x" and (contracted axes, free axes) for side "y": X's canonical order when that is its axis order, one stable sort
    otherwise.  Rows exist only where there are entries.

    "x": (row keys F [nF] int64, row pointers [nF + 1], contracted key C of every entry [nnz] int64, values)
    "y": (row keys C [nC] int64, row pointers [nC + 2] with an empty last row, distinct free keys G [nG] int64,
          the rank of every entry's G among them [nnz], values)"""
    from ._gcxs import GCXS
    from ._utils import key_bits, prod

    key = ("sptc", side, tuple(con), narrow)
    cache = X._mode_streams
    if cache is not None and key in cache:
        return cache[key]
    c = X.tocoo() if isinstance(X, GCXS) else X
    order = list(free) + list(con) if side == "x" else list(con) + list(free)
    inner = prod(X.shape[a] for a in (con if side == "x" else free))
    keys, data = c._permuted_keys(order)
    nnz = X.nnz
    rows, cols, _ = Kn.csr_from_keys(keys, 0, inner, np.int64, want_rows=True, want_indptr=False)
    heads = Kn.flag_heads(rows)
    pos, nr = Kn.scan_flags(heads)
    rowkeys = Kn.compact(rows, heads, pos, nr)
    t = D.torch()
    ptr = t.cat([Kn.compact(Kn.iota(nnz), heads, pos, nr), Kn.full(1 if side == "x" else 2, nnz, np.int64)])
    idt = np.int32 if narrow else np.int64
    ptr = Kn.cast(ptr, idt)
    if side == "x":
        stream = (rowkeys, ptr, cols, data)
    else:
        by_col, _ = Kn.sort_keys(cols, key_bits(inner))
        cheads = Kn.flag_heads(by_col)
        cpos, ng = Kn.scan_flags(cheads)
        colkeys = Kn.compact(by_col, cheads, cpos, ng)
        stream = (rowkeys, ptr, colkeys, Kn.sptc_join(cols, colkeys, idt), data)
    if cache is None:
        cache = X._mode_streams = {}
    cache[key] = stream
    return stream


def sptc(X, Y, axes=2):
    """Sparse x sparse tensor contraction with a sparse result: ``tensordot(X, Y, axes)`` for two sparse tensors whose
    extents are far larger than their numbers of entries -- contracting two sparse tensors of a tensor network or a
    quantum-chemistry code, chaining sparse Tucker cores, a TTM with a sparse matrix.

        Z[f_1, ..., g_1, ...] = sum over the contracted index tuples c of  X[f..., c...] * Y[c..., g...]

    `X` and `Y` are COO or GCXS arrays of order 1..8 with a zero fill value (a GCXS computes as its ``tocoo()``).
    `axes` has tensordot's forms: an int n (the last n axes of X with the first n of Y) or ``(axes_x, axes_y)``, ints
    or sequences, negative axes counting from the end, paired in the order given.  The dtype is that of ``X * Y``:
    float32, float64, int32 or int64, and int8 / int16 / uint8 / uint16 / uint32 through a wider integer as in
    tensordot; anything else raises TypeError.  The result is always a canonical COO of shape free(X) + free(Y) with
    fill value +0.  A dense or GCXS result is not offered: it would span the extents this op leaves out.

    The order of operations is fixed (include/sparse_b200.h, b2s_sptc_join): each value is ((+0 + x_1 * y_1) +
    x_2 * y_2) + ... over the common contracted indices in ascending C order, each product and sum rounded, integers
    wrapping, and a value is stored iff its bits differ from +0 (-0.0 and NaN stay).  Wherever tensordot fits in
    memory, ``sptc(X, Y, axes)`` equals ``tensordot(X.tocoo(), Y.tocoo(), axes, return_type=COO)`` bit for bit.
    tensordot builds a row pointer over the product of X's free extents and another over the product of the contracted
    extents; sptc keeps only the rows that hold entries, so its memory is O(nnz(X) + nnz(Y) + products) whatever the
    extents.  The products of X's and Y's free extents together, and of the contracted extents, must be below 2**63
    (ValueError before anything is allocated).

    Memory: each operand's compressed rows are cached on it for the next call with the same side and contracted axes
    (dropped when its contents are replaced, not copied or pickled).  X holds nnz * (8 + value bytes) + nF * (8 + index
    bytes), Y nnz * (index bytes + value bytes) + nC * (8 + index bytes) + nG * 8, with nF / nC / nG the numbers of
    distinct free keys of X, contracted keys of Y and free keys of Y, and index bytes 4 when both nnz fit int32, else
    8; the values are X's own array when no sort was needed.  During the call: nnz(X) * index bytes for the join, K4's
    scratch (proportional to nF and to the products) and the result, nnz(Z) * (value bytes + 8) plus 16 bytes per entry
    of K4's row and column output.
    """
    from ._dot import _dot_dtype
    from ._elemwise import _WIDE_FOR
    from ._gcxs import GCXS
    from ._utils import prod

    for name, x in (("X", X), ("Y", Y)):
        if not isinstance(x, (COO, GCXS)):
            raise TypeError(f"sptc: `{name}` must be a sparse_b200 COO or GCXS array")
    check_zero_fill_value(X, Y)
    axes_x, axes_y = _sptc_axes(X, Y, axes)
    for name, x in (("X", X), ("Y", Y)):
        if x.ndim > 8:
            raise ValueError(f"sptc: order {x.ndim} of `{name}` outside 1..8")
    T = _dot_dtype(X.dtype, Y.dtype)
    Tc = _WIDE_FOR.get(T, T)
    if Tc not in _MASKED_DTYPES:
        raise TypeError(f"sptc: dtypes ({X.dtype}, {Y.dtype}) are outside the CUDA dtype matrix (float32, float64, "
                        "int32, int64, and the narrower integers through them)")
    free_x = [a for a in range(X.ndim) if a not in axes_x]
    free_y = [a for a in range(Y.ndim) if a not in axes_y]
    shape = tuple(X.shape[a] for a in free_x) + tuple(Y.shape[a] for a in free_y)
    g_ext = prod(Y.shape[a] for a in free_y)
    if prod(shape) >= 2**63:
        raise ValueError(f"sptc: result shape {shape} has 2**63 elements or more (the COO index limit)")
    if prod(X.shape[a] for a in axes_x) >= 2**63:
        raise ValueError(f"sptc: the contracted extents {tuple(X.shape[a] for a in axes_x)} have a product of 2**63 or "
                         "more")
    if X.nnz == 0 or Y.nnz == 0:
        return COO._from_device(None, Kn.full(0, 0, T), shape, T.type(0), keys=Kn.full(0, 0, np.int64))
    narrow = not _FORCE_WIDE_INDEX_SPTC and max(X.nnz, Y.nnz) + 1 < 2**31 - 1
    xrows, xptr, xcon, xvals = _sptc_stream(X, free_x, axes_x, "x", narrow)
    yrows, yptr, ycols, yrank, yvals = _sptc_stream(Y, free_y, axes_y, "y", narrow)
    nC = int(yrows.shape[0])
    # an X entry whose contracted key no Y entry has gets column nC, Y's empty last row: X needs no compaction
    joined = Kn.sptc_join(xcon, yrows, np.int32 if narrow else np.int64)
    _, cols, rows, data, _ = Kn.spgemm(xptr, joined, Kn.cast(xvals, Tc), yptr, yrank, Kn.cast(yvals, Tc),
                                       int(xrows.shape[0]), nC + 1, int(ycols.shape[0]), sorted_order=True, prune=True,
                                       want_indptr=False, want_rows=True)
    res = COO._from_device(None, data, shape, Tc.type(0), keys=Kn.sptc_keys(rows, cols, xrows, ycols, g_ext))
    return res if Tc == T else res.astype(T, _raw=True)


def _rows_of_b(b, Tc):
    """(B^T as CSR arrays (vals, indices, indptr), whether they are b's own stored arrays)."""
    from ._gcxs import GCXS

    if isinstance(b, GCXS):
        if b.compressed_axes == (1,):
            return _csr_arrays(b._2d_transpose(), Tc), True  # O(1): CSC of b is the CSR of b^T
        return _csr_arrays(b.change_compressed_axes((1,))._2d_transpose(), Tc), False  # one conversion per call
    return _coo_as_csr(b, Tc, by_col=True), False


def _rows_of_a(a, Tc):
    """(A as CSR arrays (vals, indices, indptr), whether they are a's own stored arrays)."""
    from ._gcxs import GCXS

    if isinstance(a, GCXS):
        if a.compressed_axes == (0,):
            return _csr_arrays(a, Tc), True
        return _csr_arrays(a.change_compressed_axes((0,)), Tc), False
    return _coo_as_csr(a, Tc), False


def _masked_unfused(mask, a, b, T):
    """mask * (a @ b) through the package's own product and multiply, restricted to mask's stored positions."""
    from ._gcxs import GCXS

    r = mask * (a @ b)
    r = r.tocoo() if isinstance(r, GCXS) else r
    mc = mask.tocoo() if isinstance(mask, GCXS) else mask
    _, data = r._dev()
    keys = r.sorted_keys()
    flags = Kn.keys_member(keys, mc.sorted_keys())
    pos, total = Kn.scan_flags(flags)
    res = COO._from_device(None, Kn.cast(Kn.compact(data, flags, pos, total), T),
                           mask.shape, T.type(0), keys=Kn.compact(keys, flags, pos, total))
    return res.asformat("gcxs", compressed_axes=mask.compressed_axes) if isinstance(mask, GCXS) else res


def masked_matmul(mask, a, b):
    """Masked sparse x sparse product: the value of ``mask * (a @ b)`` at every stored position of `mask`, without
    forming ``a @ b`` (examples/triangles_example.py: ``masked_matmul(A, A, A).sum() / 6`` counts the triangles of a
    symmetric adjacency matrix A).

    `mask` (M, N), `a` (M, K) and `b` (K, N) are 2-D COO or GCXS arrays with a zero fill value.  The result has
    `mask`'s format (a GCXS result keeps ``mask.compressed_axes``) and dtype result_type(mask.dtype, result_type(a.dtype,
    b.dtype)); both dtypes must be float32, float64, int32 or int64.  Values are bit-identical to the unfused
    expression at the mask's positions: c = sum over k of a[i, k] * b[k, j] in ascending k from +0 (each product and sum
    rounded, integers wrap), then mask[i, j] * c, and entries whose result is bitwise +0 are not stored
    (include/sparse_b200.h, b2s_masked_spgemm).  The memory is O(nnz(mask) + nnz(a) + nnz(b)).

    One difference from ``mask * (a @ b)``: the unfused expression also stores entries OUTSIDE mask's pattern, ``0 * c =
    -0.0`` where (a @ b)[i, j] is negative and NaN where it is inf or NaN, because pruning compares bit patterns (-0.0
    is not +0).  masked_matmul has GraphBLAS masked semantics and never produces those entries; where ``a @ b`` is
    non-negative and finite outside the mask (graphs, for instance) the two results are equal in full.

    Layout costs: the kernel reads a by rows and b by columns.  A CSR / COO `a` and a CSC / COO `b` are used as they are
    (a COO `b` is sorted by column once per call); a CSC `a` or a CSR `b` is converted once per call, at the cost of a
    format conversion of that operand.  For a symmetric adjacency matrix, pass ``A.T`` (an O(1) view) as `b`.
    GCXS operands whose rows hold unsorted or repeated indices (possible when the arrays are built by hand) are summed
    in a different order by the unfused path; such calls are detected with one device check and computed as the
    unfused expression restricted to the mask's pattern.
    """
    from ._gcxs import GCXS

    for name, x in (("mask", mask), ("a", a), ("b", b)):
        if not isinstance(x, (COO, GCXS)) or x.ndim != 2:
            raise TypeError(f"masked_matmul: `{name}` must be a 2-D sparse_b200 COO or GCXS array")
    check_zero_fill_value(mask, a, b)
    M, N = mask.shape
    if a.shape[0] != M or b.shape[1] != N or a.shape[1] != b.shape[0]:
        raise ValueError(f"masked_matmul: shape mismatch mask{mask.shape}, a{a.shape}, b{b.shape}")
    K = a.shape[1]
    Tc = np.result_type(a.dtype, b.dtype)
    T = np.result_type(mask.dtype, Tc)
    if Tc not in _MASKED_DTYPES or T not in _MASKED_DTYPES:
        raise TypeError(f"masked_matmul: dtypes ({mask.dtype}, {a.dtype}, {b.dtype}) are outside the CUDA dtype "
                        "matrix (float32, float64, int32, int64)")
    was_gcxs = isinstance(mask, GCXS)
    if mask.nnz == 0:
        res = COO._from_device(None, Kn.full(0, 0, T), mask.shape, T.type(0), keys=Kn.full(0, 0, np.int64))
        return res.asformat("gcxs", compressed_axes=mask.compressed_axes) if was_gcxs else res
    (av, ai, ap), a_own = _rows_of_a(a, Tc)
    (bv, bi, bp), b_own = _rows_of_b(b, Tc)
    if was_gcxs:
        mv, mi_own, mp_own = mask._dev()
        mvals, mi, mp = Kn.cast(mv, T), mi_own, mp_own
    else:
        mvals, mi, mp = _coo_as_csr(mask, T)
    limit = 2**63 if _FORCE_WIDE_INDEX_MASKED else max(M, N, K, mask.nnz, a.nnz, b.nnz)
    mi, mp, ai, ap, bi, bp = _narrow_idx(mi, mp, ai, ap, bi, bp, limit=limit)
    if (a_own or b_own) and not Kn.masked_spgemm_sorted(ap if a_own else None, ai if a_own else None, M,
                                                        bp if b_own else None, bi if b_own else None, N):
        return _masked_unfused(mask, a, b, T)
    if was_gcxs:
        # a CSC mask is the CSR of mask^T: (mask o (a @ b))^T = mask^T o (b^T @ a^T), still summed in ascending k
        if mask.compressed_axes == (0,):
            out = Kn.masked_spgemm(mp, mi, mvals, ap, ai, av, bp, bi, bv, M, N, K)
        else:
            out = Kn.masked_spgemm(mp, mi, mvals, bp, bi, bv, ap, ai, av, N, M, K)
        res = GCXS._from_device(out, mi_own, mp_own, mask.shape, mask.compressed_axes, T.type(0))
        res._prune()  # mask * (a @ b) drops results that are bitwise +0 (the prune compaction)
        return res
    out = Kn.masked_spgemm(mp, mi, mvals, ap, ai, av, bp, bi, bv, M, N, K)
    res = COO._from_device(mask._coords, out, mask.shape, T.type(0), keys=mask.sorted_keys())
    res._canonicalise(check_sort=False, sum_dups=False, prune=True)  # drops bitwise +0 results, as the multiply does
    return res
