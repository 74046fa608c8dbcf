"""Broadcasting element-wise operations (`elemwise`, `__array_ufunc__` target).

Host-side mirror of sparse/numba_backend/_umath.py: operand normalisation and output type selection
(`_Elemwise.__init__`, :393-455), broadcast shape rules (:95-176), fill-value computation (:505-555).  The
reference's mask enumeration + sort-merge joins (:457-503, :576-751) are replaced by one merge-path
coiteration on the device (csrc/elemwise.cu); results are identical canonical COO arrays.

Only an enumerated set of NumPy ufuncs runs on the CUDA path (see _BINARY / _UNARY); anything else raises
TypeError -- there is no CPU fallback.
"""
from __future__ import annotations

from builtins import any as builtins_any
from itertools import zip_longest

import numpy as np

from . import _device as D
from . import _kernels as Kn
from ._coo import COO, _is_scipy_sparse
from ._sparse_array import SparseArray
from ._utils import _zero_of_dtype, c_strides, isscalar, key_bits, prod

def nan_replace(a, b):
    """where(isnan(a), b, a): NumPy meaning of device op 14 (`_replace_nan`, _coo/common.py:674-693); type resolution
    and fill values run through this definition, the stored values through the map kernel."""
    return np.where(np.isnan(a), b, a)


def _sel_x(c, x):
    """c != 0 ? x : +0 (device op 15; first half of the three-operand where)."""
    x = np.asarray(x)
    return np.where(np.asarray(c) != 0, x, x.dtype.type(0))


def _sel_y(c, y):
    """c != 0 ? +0 : y (device op 16)."""
    y = np.asarray(y)
    return np.where(np.asarray(c) != 0, y.dtype.type(0), y)


def _bitor_raw(a, b):
    """OR of the raw bit patterns (device op 17): merges the two selections without touching -0.0 / NaN payloads."""
    a, b = np.asarray(a), np.asarray(b)
    dt = np.result_type(a, b)
    u = np.dtype(f"u{dt.itemsize}")
    return (a.astype(dt).view(u) | b.astype(dt).view(u)).view(dt)


# ufunc -> device op code (csrc/elemwise.cu)
_BINARY = {
    np.add: 0, np.subtract: 1, np.multiply: 2, np.true_divide: 3, np.maximum: 4, np.minimum: 5, np.fmax: 6,
    np.fmin: 7, np.power: 8, np.floor_divide: 9, np.remainder: 10, np.bitwise_and: 11, np.bitwise_or: 12,
    np.bitwise_xor: 13, nan_replace: 14, _sel_x: 15, _sel_y: 16, _bitor_raw: 17, np.left_shift: 18,
    np.right_shift: 19, np.greater: 32, np.greater_equal: 33, np.less: 34, np.less_equal: 35, np.equal: 36,
    np.not_equal: 37, np.logical_and: 38, np.logical_or: 39, np.logical_xor: 40,
}
_UNARY = {
    np.negative: 0, np.absolute: 1, np.fabs: 1, np.sqrt: 2, np.square: 3, np.sign: 4, np.exp: 5, np.expm1: 6,
    np.log: 7, np.log1p: 8, np.sin: 9, np.cos: 10, np.tan: 11, np.tanh: 12, np.sinh: 13, np.cosh: 14, np.arcsin: 15,
    np.arctan: 16, np.floor: 17, np.ceil: 18, np.trunc: 19, np.rint: 20, np.reciprocal: 21, np.positive: 22,
    np.invert: 23, np.arcsinh: 24, np.arctanh: 25, np.deg2rad: 26, np.rad2deg: 27, np.exp2: 28, np.log2: 29,
    np.log10: 30, np.cbrt: 31, np.isnan: 64, np.isinf: 65, np.isfinite: 66, np.logical_not: 67, np.signbit: 68,
}
# on two boolean operands these ufuncs ARE the logical ones (NumPy keeps bool: True + True is True)
_BOOL_BITWISE = {np.bitwise_and: np.logical_and, np.bitwise_or: np.logical_or, np.bitwise_xor: np.logical_xor,
                 np.add: np.logical_or, np.maximum: np.logical_or, np.fmax: np.logical_or,
                 np.multiply: np.logical_and, np.minimum: np.logical_and, np.fmin: np.logical_and}
_COMPUTE_DTYPES = (np.dtype("float32"), np.dtype("float64"), np.dtype("int32"), np.dtype("int64"))


def _get_broadcast_shape(shape1, shape2, is_result=False):
    """_umath.py:123-154."""
    if not all((l1 == l2) or (l1 == 1) or ((l2 == 1) and not is_result)
               for l1, l2 in zip(shape1[::-1], shape2[::-1], strict=False)):
        raise ValueError(f"operands could not be broadcast together with shapes {shape1}, {shape2}")
    return tuple(l1 if l1 != 1 else l2 for l1, l2 in zip_longest(shape1[::-1], shape2[::-1], fillvalue=1))[::-1]


def _get_nary_broadcast_shape(*shapes):
    """_umath.py:95-121."""
    result_shape = ()
    for shape in shapes:
        try:
            result_shape = _get_broadcast_shape(shape, result_shape)
        except ValueError as e:
            shapes_str = ", ".join(str(shape) for shape in shapes)
            raise ValueError(f"operands could not be broadcast together with shapes {shapes_str}") from e
    return result_shape


def _op_code(func, table, what):
    try:
        return table[func]
    except (KeyError, TypeError):
        name = getattr(func, "__name__", repr(func))
        raise TypeError(
            f"sparse_b200: {what} function {name!r} is not in the CUDA op set "
            f"({', '.join(sorted(f.__name__ for f in table))}); there is no CPU fallback."
        ) from None


# narrow / unsigned integer dtypes are storage-only on the device; their arithmetic is exact in a wider signed type and
# the C narrowing cast wraps exactly like NumPy's arithmetic in the narrow type (two's complement, modulo 2**bits)
_WIDE_FOR = {np.dtype("int8"): np.dtype("int32"), np.dtype("int16"): np.dtype("int32"),
             np.dtype("uint8"): np.dtype("int32"), np.dtype("uint16"): np.dtype("int32"),
             np.dtype("uint32"): np.dtype("int64")}
_NOT_VIA_WIDE = (np.power, np.left_shift, np.right_shift, np.true_divide)


def _check_compute_dtype(dt, func):
    if np.dtype(dt) not in _COMPUTE_DTYPES:
        raise TypeError(f"sparse_b200: {getattr(func, '__name__', func)} on dtype {dt} is outside the CUDA dtype matrix "
                        "(float32, float64, int32, int64; bool for logical ops)")


def _resolve(func, a_like, b_like=None):
    """(out_dtype, compute_dtype) using NumPy's own type resolution on zero-size stand-ins."""
    with np.errstate(all="ignore"):
        res = func(a_like) if b_like is None else func(a_like, b_like)
    out_dt = res.dtype
    code_table = _UNARY if b_like is None else _BINARY
    pred = code_table[func] >= (64 if b_like is None else 32)
    if pred:
        ins = [a_like] if b_like is None else [a_like, b_like]
        T = np.result_type(*ins)
        if T == np.bool_:
            T = np.dtype("int32")
    else:
        T = out_dt
    return out_dt, np.dtype(T)


def _stand_in(x):
    if isinstance(x, SparseArray):
        return np.empty(0, dtype=x.dtype)
    if isinstance(x, np.ndarray) and x.ndim > 0:
        return np.empty(0, dtype=x.dtype)
    if D.is_device_tensor(x):
        return np.empty(0, dtype=D.np_dtype(x))
    return x  # python / numpy scalar: keeps NEP-50 weak typing


def _finish(keys, vals, flags, shape, fill, idx_dtype=np.int64):
    """Stage B shared by every elemwise form: compact the kept candidates and derive coordinates."""
    pos, total = Kn.scan_flags(flags)
    if total != int(flags.shape[0]):
        keys = Kn.compact(keys, flags, pos, total)
        vals = Kn.compact(vals, flags, pos, total)
    return COO._from_device(None, vals, shape, fill, keys=keys)


def _stream(x, shape):
    """Sorted key stream of COO `x` broadcast to `shape`: (keys, data, R).

    Trailing broadcast axes are expanded virtually (R > 1); any other broadcast pattern is materialised with the
    expansion kernel (+ a stable sort when the expansion is not already in key order)."""
    data = x._data_dev()
    nd, xn = len(shape), x.ndim
    off = nd - xn
    # result axis d is a broadcast axis of x iff the result is wider there than x (x lacks it or has extent 1)
    bcast = [shape[d] > 1 and (d < off or x.shape[d - off] != shape[d]) for d in range(nd)]
    if not any(bcast):
        if tuple(x.shape) == tuple(shape):
            return x.sorted_keys(), data, 1
        # same C-order layout up to leading extent-1 axes: the linear keys are identical
        return x.sorted_keys(), data, 1
    first_b = bcast.index(True)
    trailing = all(bcast[d] or shape[d] == 1 for d in range(first_b, nd))
    if trailing:
        R = prod(shape[first_b:])
        st = c_strides(shape)
        strides = [(st[d + off] // R if (d + off) < first_b else 0) for d in range(xn)]
        return Kn.linearize(x._dev()[0], strides), data, R
    src_row = [(d - off if (d >= off and not bcast[d]) else -1) for d in range(nd)]
    # axes that x lacks but have extent 1 contribute coordinate 0: treat as broadcast of extent 1
    is_b = [1 if (bcast[d] or src_row[d] < 0) else 0 for d in range(nd)]
    keys, src = Kn.ew_expand(x._dev()[0], shape, is_b, src_row)
    unsorted, _ = Kn.keys_flags(keys)
    if unsorted:
        keys, perm = Kn.sort_keys(keys, key_bits(prod(shape)))
        src = Kn.gather(src, perm)
    return keys, Kn.gather(data, src), 1


def _dense_strides_over(shape, dshape):
    """Element strides of a C-contiguous dense operand of `dshape` broadcast to `shape` (0 on broadcast axes)."""
    nd, dn = len(shape), len(dshape)
    st = c_strides(dshape)
    out = [0] * nd
    for d in range(dn):
        rd = d + (nd - dn)
        out[rd] = 0 if dshape[d] == 1 and shape[rd] != 1 else st[d]
    return out


def dense_binary(func, x, y):
    """Element-wise `func` of two dense DEVICE tensors (broadcast against each other) on the element-wise kernel: the
    COO (x) dense gather with identity keys, i.e. the `_dense_result` pattern below.  Keeps dense (x) dense steps of
    einsum / complex products off torch's arithmetic."""
    t = D.torch()
    shape = tuple(int(s) for s in t.broadcast_shapes(tuple(x.shape), tuple(y.shape)))
    dt = np.result_type(D.np_dtype(x), D.np_dtype(y))
    _check_compute_dtype(dt, func)
    xb = Kn.cast(x, dt).broadcast_to(shape).contiguous().reshape(-1)
    yb = Kn.cast(y, dt).broadcast_to(shape).contiguous().reshape(-1)
    n = int(xb.shape[0])
    if n == 0:
        return xb.reshape(shape)
    code = _BINARY[func]
    out_dt = np.dtype(np.bool_) if code >= 32 else dt  # predicates write bool, value ops the operand dtype
    _, vals, _ = Kn.ew_dense(code, False, Kn.iota(n), xb, 1, yb, shape if shape else (1,),
                             c_strides(shape) if shape else [1], False if code >= 32 else 0, out_dt)
    return vals.reshape(shape)


def _out_format(sparse_args):
    """Result format of an element-wise call (_umath.py:414-425): DOK when every sparse operand is DOK, GCXS when
    every one is GCXS (with their compressed axes when they all agree), COO otherwise."""
    from ._dok import DOK
    from ._gcxs import GCXS

    if all(isinstance(arg, DOK) for arg in sparse_args):
        return DOK, {}
    if all(isinstance(arg, GCXS) for arg in sparse_args):
        if len({arg.compressed_axes for arg in sparse_args}) == 1:
            return GCXS, {"compressed_axes": sparse_args[0].compressed_axes}
        return GCXS, {}
    return COO, {}


def _refuse_negative_exponent(exponent, T):
    """Integer np.power raises on a negative exponent anywhere in its operands; the kernel has no error path, so the
    exponent (scalar on the host; stored entries, fill value or dense operand with one device pass) is checked first."""
    msg = "Integers to negative integer powers are not allowed."
    if isinstance(exponent, COO):
        if exponent.fill_value < 0:
            raise ValueError(msg)
        data = exponent._data_dev()
    elif isinstance(exponent, np.ndarray) and exponent.ndim > 0:
        data = D.upload(np.ascontiguousarray(exponent).reshape(-1))
    elif D.is_device_tensor(exponent):
        data = exponent.reshape(-1)
    else:
        if exponent < 0:
            raise ValueError(msg)
        return
    if data.shape[0] == 0:
        return
    _, negative = Kn.ew_map(_BINARY[np.less], 0, Kn.cast(data, T), T.type(0), False, np.bool_)
    if Kn.scan_flags(negative)[1]:
        raise ValueError(msg)


def _fill_of(func, *fills):
    """func(fill values) the way the reference evaluates it (_umath.py:516-527): NumPy values go through the ARRAY
    loop as 1-element arrays, Python scalars stay weak scalars.  NumPy's scalar and array loops are not bit-identical
    everywhere (float16 transcendental results, fmin / fmax of +0.0 and -0.0), and the fill value decides what is
    pruned, so the same loop has to run."""
    with np.errstate(all="ignore"):
        res = func(*[np.atleast_1d(f) if isinstance(f, (np.generic, np.ndarray)) else f for f in fills])
    return np.asarray(res).reshape(-1)[0]


class _Elemwise:
    def __init__(self, func, *args, **kwargs):
        from ._gcxs import GCXS

        processed = []
        sparse_args = [arg for arg in args if isinstance(arg, SparseArray)]
        if len(sparse_args) == 0:
            raise ValueError(f"None of the args is sparse: {args}")
        out_type, out_kwargs = _out_format(sparse_args)
        self.args = None
        for arg in args:
            if _is_scipy_sparse(arg):
                processed.append(COO.from_scipy_sparse(arg))
            elif isscalar(arg) or isinstance(arg, np.ndarray) or D.is_device_tensor(arg):
                processed.append(arg)
            elif isinstance(arg, SparseArray):
                if not isinstance(arg, COO):
                    arg = arg.asformat(COO)
                if arg.ndim == 0:
                    arg = arg.todense()
                processed.append(arg)
            else:
                return
        self.out_type, self.out_kwargs = out_type, out_kwargs
        self.args = tuple(processed)
        self.func = func
        self.dtype = kwargs.pop("dtype", None)
        kwargs.pop("casting", None)
        kwargs.pop("where", None) if kwargs.get("where", True) is True else None
        if kwargs:
            raise TypeError(f"sparse_b200.elemwise: unsupported keyword arguments {sorted(kwargs)}")
        self.shape = _get_nary_broadcast_shape(*tuple(tuple(a.shape) if hasattr(a, "shape") else np.shape(a)
                                                      for a in self.args))

    def get_result(self):
        if self.args is None:
            return NotImplemented
        n = len(self.args)
        if not any(isinstance(a, COO) for a in self.args):
            # every sparse operand was 0-D and became a scalar (_umath.py:438-439): the result is the 0-D array
            # whose fill value is func(scalars) -- host scalar arithmetic, no data path involved
            # Python scalars stay Python scalars (weak promotion: clip(float32, -1, 2) is float32); NumPy values go
            # through the ARRAY loop as in the reference (np.atleast_1d, _umath.py:516-527 -- for float16 results it
            # is not the scalar loop bit for bit)
            host = [D.download(a) if D.is_device_tensor(a) else a for a in self.args]

            def call(*args):
                # `dtype=` selects the loop (operands are cast BEFORE the operation); functions that do not take it
                # are called without and the result is cast (_umath.py:521-524, 612-620)
                if self.dtype is not None:
                    try:
                        return self.func(*args, dtype=self.dtype)
                    except TypeError:
                        pass
                return self.func(*args)

            with np.errstate(all="ignore"):
                if all(np.ndim(h) == 0 for h in host):
                    res = np.asarray(call(*[np.atleast_1d(h) if isinstance(h, (np.generic, np.ndarray)) else h
                                            for h in host])).reshape(())
                else:
                    res = np.asarray(call(*host))
            if self.dtype is not None:
                res = res.astype(self.dtype)
            if res.ndim:
                # 0-D sparse operands next to a dense array: dense, unless func(fills, ndarray) is one constant --
                # then that constant is the fill value of an array without stored entries (_umath.py:536-546); with
                # a zero-length axis the constant is func(fills, zero of the ndarray's dtype) (:529-534)
                from ._utils import equivalent

                if res.size == 0:
                    with np.errstate(all="ignore"):
                        # upstream substitutes the zero of the dtype for EVERY ndarray here, the densified 0-D
                        # sparse operands included (:531-533)
                        const = np.asarray(self.func(*[_zero_of_dtype(h.dtype) if isinstance(h, (np.ndarray, np.generic))
                                                       else h for h in host])).astype(res.dtype)[()]
                elif equivalent(res.reshape(-1)[0], res, loose=True).all():
                    const = res.reshape(-1)[0]
                else:
                    return res
                return COO(np.empty((res.ndim, 0), dtype=np.intp), np.empty(0, dtype=res.dtype), shape=res.shape,
                           has_duplicates=False, sorted=True, fill_value=const) if res.size == 0 else COO(
                    np.empty((res.ndim, 0), dtype=np.intp), np.empty(0, dtype=res.dtype), shape=res.shape,
                    has_duplicates=False, sorted=True, fill_value=const).asformat(self.out_type, **self.out_kwargs)
            # no stored entry, the value is the fill value, and the operands' format is kept (_umath.py:480-503)
            return COO(np.empty((0, 0), dtype=np.intp), np.empty(0, dtype=res.dtype), shape=(), has_duplicates=False,
                       sorted=True, fill_value=res[()]).asformat(self.out_type, **self.out_kwargs)
        from . import _complex as C

        if isinstance(self.func, np.ufunc) and builtins_any(C.is_complex(a) for a in self.args) \
                or (self.dtype is not None and np.dtype(self.dtype).kind == "c"):
            out = C.elemwise_complex(self.func, self.args)
            if out is NotImplemented:
                raise TypeError(f"sparse_b200: {getattr(self.func, '__name__', self.func)} on complex operands is "
                                "outside the CUDA op set (add, subtract, multiply, divide, negative, conjugate, "
                                "absolute, square, equal, not_equal, isnan, isinf, isfinite)")
            if isinstance(out, SparseArray):
                if self.dtype is not None and np.dtype(self.dtype) != out.dtype:
                    out = out.astype(self.dtype)
                return out.asformat(self.out_type, **self.out_kwargs)
            return out
        if self.dtype is not None and isinstance(self.func, np.ufunc):
            # ufunc(..., dtype=T) (what `out=` turns into, _sparse_array.py:344) selects the T loop: array operands
            # are cast to T BEFORE the operation.  Predicates (bool result whatever the input) keep their operands.
            dt = np.dtype(self.dtype)
            code = _BINARY.get(self.func, 0) if n == 2 else _UNARY.get(self.func, 0)
            if dt != np.bool_ and code < (32 if n == 2 else 64):
                self.args = tuple(a.astype(dt) if isinstance(a, (COO, np.ndarray)) and getattr(a, "ndim", 0) > 0
                                  and a.dtype != dt else a for a in self.args)
        composite = not isinstance(self.func, np.ufunc) and self.func not in _BINARY and self.func not in _UNARY
        if composite:
            out = self._composite()
        elif n == 1:
            out = self._unary()
        elif n == 2:
            out = self._binary()
        else:
            out = self._composite()
        if isinstance(out, COO):
            if self.dtype is not None and np.dtype(self.dtype) != out.dtype:
                out = out.astype(self.dtype)
            if any(s == 0 for s in self.shape):
                return out  # a zero-length axis: the reference returns the empty COO as it is (_umath.py:467-477)
            return out.asformat(self.out_type, **self.out_kwargs)
        return out

    # ------------------------------------------------------------------------------------------------------
    def _composite(self):
        """n-ary / user-defined `func` (e.g. `lambda x, y, z: (x + y) * z`, tests/test_elemwise.py:252-305 upstream).

        The reference evaluates `func` with NumPy on the matched data of every mask combination (_umath.py:576-654).
        A Python callable cannot run inside a CUDA kernel, so it is evaluated ONCE on the sparse operands themselves:
        every operator / ufunc inside it dispatches back to the unary / binary device kernels through
        `__array_ufunc__`, and the intermediate results stay canonical COO arrays on the device.  Element for element
        the same IEEE operations run in the same order as in the reference, so values and the final fill value are
        identical; a `func` that leaves the ufunc protocol (or an n-ary ufunc, n > 2) raises."""
        if isinstance(self.func, np.ufunc):
            raise TypeError(f"sparse_b200: {self.func.__name__} with {len(self.args)} operands is not in the CUDA op "
                            "set; there is no CPU fallback.")
        from ._utils import equivalent

        def is_dense(a):
            return (isinstance(a, np.ndarray) and a.ndim > 0) or D.is_device_tensor(a)

        # Next to ndarrays (or with a zero-length axis) upstream decides sparse-or-dense, the error and the fill value
        # on ONE probe of func(fill values | ndarrays) (_umath.py:505-546); evaluating `func` operator by operator
        # decides per operator, which differs (an intermediate that happens to be constant, ndarrays of different
        # shapes, 0-D operands).  The probe is host arithmetic on fill values and the ndarrays, as upstream's.
        probe = None
        dense_args = [a for a in self.args if is_dense(a)]
        shape = tuple(self.shape)
        if dense_args or any(s == 0 for s in shape):
            def stand_in(a, zeros=False):
                if isinstance(a, COO):
                    return a.fill_value if zeros else np.atleast_1d(a.fill_value)
                if D.is_device_tensor(a):
                    a = D.download(a)
                if isinstance(a, (np.ndarray, np.generic)):
                    return _zero_of_dtype(a.dtype) if zeros else np.atleast_1d(a)
                return a

            with np.errstate(all="ignore"):
                fva = np.asarray(self.func(*[stand_in(a) for a in self.args]))
                fv = fva.reshape(-1)[0] if fva.size else np.asarray(
                    self.func(*[stand_in(a, zeros=True) for a in self.args])).reshape(-1)[0]
            const = bool(equivalent(fv, fva, loose=True).all()) if fva.size else True
            if not const:
                nd_shape = _get_nary_broadcast_shape(*[tuple(a.shape) for a in dense_args])
                if shape != tuple(nd_shape):
                    raise ValueError("Performing a mixed sparse-dense operation that would result in a dense array. "
                                     "Please make sure that func(sparse_fill_values, ndarrays) is a constant array.")
            probe = (fv, const)
        if probe is None:
            out = self.func(*self.args)
        else:
            # next to ndarrays every operator would take its own sparse-or-dense decision (and a sparse (x) dense
            # product keeps ONE zero for +0.0 and -0.0): evaluate with every ndarray as a COO of its non-zero entries
            # instead -- the sparse kernels then compute the exact value at every position, the probe above decides
            # what the result looks like
            from ._coo import as_coo

            out = self.func(*[as_coo(D.download(a) if D.is_device_tensor(a) else a) if is_dense(a) else a
                              for a in self.args])
        if out is NotImplemented or not (isinstance(out, (SparseArray, np.ndarray)) or isscalar(out)
                                         or D.is_device_tensor(out)):
            raise TypeError("sparse_b200.elemwise: the function did not evaluate to an array through the NumPy ufunc "
                            "protocol; only compositions of the supported ufuncs run on the CUDA path")
        if isscalar(out):
            out = COO.from_numpy(np.asarray(out))
        if isinstance(out, SparseArray) and tuple(out.shape) != shape:
            out = broadcast_to(out.asformat("coo"), shape)
        if probe is None:
            return out.asformat("coo") if isinstance(out, SparseArray) else out
        fv, const = probe
        host = out.todense() if isinstance(out, SparseArray) and (not const or not any(s == 0 for s in shape)) else out
        if not const:  # dense result (_umath.py:463-465)
            host = D.download(host) if D.is_device_tensor(host) else np.asarray(host)
            return np.broadcast_to(host, shape).copy() if tuple(host.shape) != shape else host
        dt = np.dtype(out.dtype) if isinstance(out, (SparseArray, np.ndarray)) else D.np_dtype(out)
        fv = np.asarray(fv).astype(dt)[()]
        if any(s == 0 for s in shape):
            return self._empty(dt, fv)
        if prod(shape) > (1 << 27):  # too large to reconcile through a dense copy: the operator-by-operator result
            return out.asformat("coo") if isinstance(out, SparseArray) else out
        # Sparse by the probe.  Upstream stores, among the positions some sparse operand has an entry at (the only
        # ones it visits), those whose value differs from the fill value by bit pattern (_umath.py:627-633); the
        # operator-by-operator evaluation can store more (positions only an ndarray is non-zero at, -0.0 there) or be
        # relative to another fill value.  Rebuild exactly that set: visited positions = union of the operands'
        # stored coordinates, broadcast to the result.
        host = D.download(host) if D.is_device_tensor(host) else np.asarray(host)
        host = np.broadcast_to(host, shape) if tuple(host.shape) != shape else host
        visited = None
        for a in self.args:
            if isinstance(a, COO):
                m = COO(a.coords, np.ones(a.nnz, dtype=np.bool_), shape=a.shape, has_duplicates=False, sorted=True)
                m = broadcast_to(m, shape) if tuple(m.shape) != shape else m
                visited = m if visited is None else np.logical_or(visited, m)
        coords = np.asarray(visited.coords)
        vals = host[tuple(coords)].astype(dt, copy=False)
        keep = ~np.asarray(equivalent(vals, fv), dtype=bool).reshape(-1) if vals.size else np.zeros(0, dtype=bool)
        return COO(coords[:, keep], vals[keep], shape=shape, has_duplicates=False, sorted=True, fill_value=fv)

    def _unary(self):
        (a,) = self.args
        func = self.func
        if func is np.conjugate and a.dtype.kind in "fiu":
            func = np.positive  # conj of a real array is the array itself
        if a.dtype == np.bool_ and func in (np.invert, np.absolute, np.conjugate):
            if func is np.absolute:
                return a.copy()  # |bool| is the array itself (NumPy keeps bool)
            if func is np.conjugate:
                return a.astype(np.int8)  # NumPy has no bool loop for conjugate: the int8 one runs
            func = np.logical_not  # ~bool
        op = _op_code(func, _UNARY, "unary")
        out_dt, T = _resolve(func, _stand_in(a))
        if T in _WIDE_FOR and func not in _NOT_VIA_WIDE:
            return self._via_wide(func, T, out_dt)
        _check_compute_dtype(T, func)
        fill = np.asarray(_fill_of(func, a.fill_value)).astype(out_dt)[()]
        data = a._data_dev()
        if any(s == 0 for s in self.shape):
            return COO(np.empty((len(self.shape), 0), dtype=np.intp), np.empty(0, dtype=out_dt), shape=self.shape,
                       has_duplicates=False, sorted=True, fill_value=fill)
        vals, flags = Kn.ew_map(op, 2, Kn.cast(data, T), None, fill, out_dt)
        return self._keep(a, vals, flags, fill)

    def _via_wide(self, func, T, out_dt):
        """Narrow / unsigned integer operands: compute in the wider signed type, then cast back (the cast prunes the
        entries that wrap around to the fill value)."""
        W = _WIDE_FOR[T]

        def widen(v):
            if isinstance(v, COO):
                return v.astype(W) if v.dtype != W else v
            if isinstance(v, np.ndarray) and v.ndim > 0:
                return v.astype(W)
            if D.is_device_tensor(v):
                return Kn.cast(v, W)
            return W.type(v)

        out = _Elemwise(func, *[widen(a) for a in self.args]).get_result()
        if out_dt == np.bool_ or not hasattr(out, "astype"):
            return out
        if isinstance(out, np.ndarray):
            return out.astype(out_dt)
        return out.asformat("coo").astype(out_dt, _raw=True)

    def _keep(self, a, vals, flags, fill):
        pos, total = Kn.scan_flags(flags)
        if total == a.nnz:  # nothing pruned: coordinates (materialised or lazy) are shared with the operand
            return COO._from_device(a._coords, vals, a.shape, fill,
                                    keys=a._keys if a._coords is not None else a.sorted_keys())
        keys = Kn.compact(a.sorted_keys(), flags, pos, total)
        return COO._from_device(None, Kn.compact(vals, flags, pos, total), a.shape, fill, keys=keys)

    # ------------------------------------------------------------------------------------------------------
    def _binary(self):
        a, b = self.args
        func = self.func
        a_sp, b_sp = isinstance(a, COO), isinstance(b, COO)
        a_dn = (isinstance(a, np.ndarray) and a.ndim > 0) or D.is_device_tensor(a)
        b_dn = (isinstance(b, np.ndarray) and b.ndim > 0) or D.is_device_tensor(b)
        # bool bitwise ops are the logical ops
        la, lb = _stand_in(a), _stand_in(b)
        if func in _BOOL_BITWISE and all(getattr(x, "dtype", np.dtype(type(x))) == np.bool_ for x in (la, lb)):
            func = _BOOL_BITWISE[func]
        op = _op_code(func, _BINARY, "binary")
        out_dt, T = _resolve(func, la, lb)
        if T in _WIDE_FOR and func not in _NOT_VIA_WIDE:
            return self._via_wide(func, T, out_dt)
        _check_compute_dtype(T, func)
        if func is np.power and T.kind == "i":
            _refuse_negative_exponent(b, T)
        if op < 32 and out_dt == np.bool_:
            raise TypeError(f"sparse_b200: {func.__name__} with boolean output is outside the CUDA dtype matrix")
        shape = self.shape
        empty = any(s == 0 for s in shape)

        def fv(x):
            return x.fill_value if isinstance(x, COO) else x

        if a_sp and b_sp:
            fill = np.asarray(_fill_of(func, a.fill_value, b.fill_value)).astype(out_dt)[()]
            if empty:
                return self._empty(out_dt, fill)
            ka, da, Ra = _stream(a, shape)
            kb, db, Rb = _stream(b, shape)
            _, vals, keys = Kn.ew_merge_fused(op, ka, Kn.cast(da, T), Ra, kb, Kn.cast(db, T), Rb,
                                              T.type(a.fill_value), T.type(b.fill_value), fill, out_dt, shape,
                                              want_coords=False)
            return COO._from_device(None, vals, shape, fill, keys=keys)

        if (a_sp and not b_dn) or (b_sp and not a_dn):  # sparse (x) scalar
            sp, sc, mode = (a, b, 0) if a_sp else (b, a, 1)
            weak = sc if type(sc) in (bool, int, float) else np.asarray(sc)[()]  # a Python scalar promotes weakly
            sc = np.asarray(sc)[()]
            fill = np.asarray(_fill_of(func, a.fill_value, weak) if a_sp else _fill_of(func, weak, b.fill_value)
                              ).astype(out_dt)[()]
            if empty:
                return self._empty(out_dt, fill)
            data = sp._data_dev()
            vals, flags = Kn.ew_map(op, mode, Kn.cast(data, T), T.type(sc), fill, out_dt)
            return self._keep(sp, vals, flags, fill)

        # sparse (x) dense ndarray: mask (True, None) of the reference
        sp, dn, swap = (a, b, False) if a_sp else (b, a, True)
        dense = D.upload(np.ascontiguousarray(dn)) if isinstance(dn, np.ndarray) else dn.contiguous()
        dense = Kn.cast(dense, T)
        dshape = tuple(dense.shape)
        flat = dense.reshape(-1)
        # _get_fill_value (:505-555): func(fill, ndarray) must be constant, else the result is dense
        g, _ = Kn.ew_map(op, 1 if not swap else 0, flat, T.type(sp.fill_value), 0, out_dt)
        if flat.shape[0] == 0:
            # nothing to test for constancy: func(fill, zero of the dense dtype) (_umath.py:529-534)
            z = _zero_of_dtype(np.dtype(dn.dtype) if isinstance(dn, np.ndarray) else D.np_dtype(dn))
            with np.errstate(all="ignore"):
                f0 = func(z, sp.fill_value) if swap else func(sp.fill_value, z)
            return self._empty(out_dt, np.asarray(f0).astype(out_dt)[()])
        fill = D.download(g[:1])[0]
        if fill != fill:
            _, nflags = Kn.ew_map(_UNARY[np.isnan], 2, Kn.cast(g, T) if out_dt != T else g, None, True, np.bool_)
        else:
            _, nflags = Kn.ew_map(_BINARY[np.not_equal], 0, Kn.cast(g, T) if out_dt != T else g, T.type(fill), False,
                                  np.bool_)
        _, n_diff = Kn.scan_flags(nflags)
        if n_diff != 0:
            if tuple(shape) != dshape:
                raise ValueError("Performing a mixed sparse-dense operation that would result in a dense array. "
                                 "Please make sure that func(sparse_fill_values, ndarrays) is a constant array.")
            return self._dense_result(sp, dense, swap, op, T, out_dt)
        if empty:
            return self._empty(out_dt, fill)
        ks, ds, Rs = _stream(sp, shape)
        keys, vals, flags = Kn.ew_dense(op, swap, ks, Kn.cast(ds, T), Rs, dense, shape,
                                        _dense_strides_over(shape, dshape), fill, out_dt)
        return _finish(keys, vals, flags, shape, fill)

    def _dense_result(self, sp, dense, swap, op, T, out_dt):
        """func(sparse.todense(), ndarray) when the fill value is not constant (_umath.py:463-465)."""
        if tuple(sp.shape) != tuple(self.shape):  # a sparse row / column / scalar against a dense array
            sp = broadcast_to(sp.asformat("coo"), self.shape)
        full = Kn.cast(sp.todense_device().reshape(-1), T)
        keys = Kn.iota(int(full.shape[0]))
        _, vals, _ = Kn.ew_dense(op, swap, keys, full, 1, dense, self.shape,
                                 _dense_strides_over(self.shape, tuple(dense.shape)), 0, out_dt)
        return D.download(vals.reshape(self.shape))

    def _empty(self, out_dt, fill):
        return COO(np.empty((len(self.shape), 0), dtype=np.intp), np.empty(0, dtype=out_dt), shape=self.shape,
                   has_duplicates=False, sorted=True, fill_value=fill)


def elemwise(func, *args, **kwargs):
    """Apply a function to any number of arguments (reference: _umath.py:13-50)."""
    return _Elemwise(func, *args, **kwargs).get_result()


def where(condition, x=None, y=None):
    """numpy.where for sparse operands (reference: _coo/common.py:533-579).

    One argument: the coordinates of the non-zero entries.  Three arguments: `elemwise(np.where, condition, x, y)` in
    the reference; here two selections and one OR of raw bit patterns, each a pass of the binary coiteration kernel:
    `(c ? x : +0) | (c ? +0 : y)` -- exact for every value (signed zeros, NaN payloads, infinities), and the fill
    value of the result is `where(fill_c, fill_x, fill_y)` by the same formula."""
    from ._utils import check_zero_fill_value

    x_given, y_given = x is not None, y is not None
    if not (x_given or y_given):
        if not isinstance(condition, SparseArray) and not _is_scipy_sparse(condition):
            raise ValueError(f"Performing this operation would produce a dense result: {np.where!s}")
        check_zero_fill_value(condition)
        c = condition.asformat("coo") if isinstance(condition, SparseArray) else COO.from_scipy_sparse(condition)
        return tuple(c.coords)
    if x_given != y_given:
        raise ValueError("either both or neither of x and y should be given")
    # one three-way broadcast check up front: the error names all three shapes, as upstream's single elemwise call does
    _get_nary_broadcast_shape(*[tuple(v.shape) if hasattr(v, "shape") else np.shape(v) for v in (condition, x, y)])
    sparse_ops = [v for v in (condition, x, y) if isinstance(v, SparseArray)]
    if sparse_ops and all(v.ndim == 0 for v in sparse_ops):
        # every sparse operand is 0-D: they are scalars to upstream (_umath.py:438-439) and the call is host arithmetic
        return _Elemwise(np.where, condition, x, y).get_result()
    with np.errstate(all="ignore"):
        T = np.result_type(_stand_in(x), _stand_in(y))
    work = np.dtype("int32") if T == np.bool_ else T
    _check_compute_dtype(work, np.where)

    def as_t(v):
        if isinstance(v, SparseArray):
            return v.astype(work) if v.dtype != work else v
        if D.is_device_tensor(v):
            return Kn.cast(v, work)
        if isinstance(v, np.ndarray) and v.ndim > 0:
            return v.astype(work)
        return work.type(v)

    c = condition
    cdt = c.dtype if hasattr(c, "dtype") else np.asarray(c).dtype
    if cdt != np.bool_:
        c = c != 0  # truth value first: a narrowing cast could flush a tiny non-zero to zero
    c = c.astype(work) if hasattr(c, "astype") else work.type(bool(c))
    def step(func, a, b):
        """One binary pass; two DENSE operands (np.where(dense, dense, sparse)) meet on the device kernel directly."""
        if isinstance(a, SparseArray) or isinstance(b, SparseArray):
            return elemwise(func, a, b)

        def dev(v):
            if D.is_device_tensor(v):
                return v
            v = np.asarray(v, dtype=work)
            return D.upload(np.ascontiguousarray(v)) if v.ndim else Kn.full(1, v[()], work)

        return dense_binary(func, dev(a), dev(b))

    # sparse or dense?  Upstream decides on the INPUTS of its one elemwise call (_umath.py:536-546):
    # where(fill_c, fill_x | ndarray, fill_y | ndarray) must be one constant for the result to stay sparse; otherwise
    # it is dense (or an error when the sparse operands would have to be broadcast up).  Deciding pass by pass would
    # differ (an intermediate that happens to be constant, two ndarrays of different shapes).  The decision is host
    # arithmetic on the fill values and the ndarrays, as upstream's; the values come from the device passes below.
    ops = (condition, x, y)
    dense_ops = [v for v in ops if (isinstance(v, np.ndarray) and v.ndim > 0) or D.is_device_tensor(v)]
    full = _get_nary_broadcast_shape(*[tuple(v.shape) if hasattr(v, "shape") else np.shape(v) for v in ops])

    def densified(v):
        return Kn.cast(v.asformat("coo").todense_device(), work) if isinstance(v, SparseArray) else v

    def dense_passes():
        """The three passes on densified operands (device kernels throughout); host array of the full shape."""
        cd, xd, yd = densified(c), densified(as_t(x)), densified(as_t(y))
        res = D.download(step(_bitor_raw, step(_sel_x, cd, xd), step(_sel_y, cd, yd)))
        res = np.broadcast_to(res, full) if tuple(res.shape) != tuple(full) else res
        return res.astype(np.bool_) if T == np.bool_ else res

    fv = None
    if dense_ops or any(s == 0 for s in full):
        from ._utils import equivalent

        def stand_in(v, zeros=False):
            """What upstream feeds its fill-value probe (_umath.py:516-534): the fill value of a sparse operand, the
            whole array for an ndarray (a 0-D sparse operand IS an ndarray by then); `zeros`: the zero of the dtype
            instead of the array, the fallback when the probe comes out empty."""
            if isinstance(v, SparseArray) and v.ndim:
                return np.atleast_1d(v.fill_value)
            if isinstance(v, SparseArray):
                v = v.todense()
            elif D.is_device_tensor(v):
                v = D.download(v)
            if isinstance(v, (np.ndarray, np.generic)):
                return _zero_of_dtype(v.dtype) if zeros else np.atleast_1d(v)
            return v

        def probe(zeros=False):
            h = [stand_in(v, zeros) for v in ops]
            with np.errstate(all="ignore"):
                return np.asarray(np.where(np.asarray(h[0]) != 0, h[1], h[2]))

        fva = probe()
        fv = fva.reshape(-1)[0] if fva.size else probe(zeros=True).reshape(-1)[0]
        if fva.size and not equivalent(fv, fva, loose=True).all():
            nd_shape = _get_nary_broadcast_shape(*[tuple(v.shape) for v in dense_ops])
            if tuple(full) != tuple(nd_shape):
                raise ValueError("Performing a mixed sparse-dense operation that would result in a dense array. "
                                 "Please make sure that func(sparse_fill_values, ndarrays) is a constant array.")
            return dense_passes()
        if any(s == 0 for s in full):  # nothing to compute: the empty COO (_umath.py:467-477)
            return COO(np.empty((len(full), 0), dtype=np.intp), np.empty(0, dtype=T), shape=tuple(full),
                       has_duplicates=False, sorted=True, fill_value=np.asarray(fv).astype(T)[()])
    cast_back = T == np.bool_
    try:
        out = step(_bitor_raw, step(_sel_x, c, as_t(x)), step(_sel_y, c, as_t(y)))
    except ValueError:
        # a single pass can need a dense intermediate that the whole expression does not (the probe above said
        # "sparse"): compute the passes on densified operands instead -- only when the result is small enough to hold
        if fv is None or prod(full) > (1 << 27):
            raise
        out, cast_back = dense_passes(), False
    if D.is_device_tensor(out):  # every step was dense (only reachable through the np.where dispatch)
        out = D.download(out)
    out = out.astype(np.bool_) if cast_back else out
    if sparse_ops and fv is not None and not isinstance(out, SparseArray):
        # the probe said "sparse" (constant fill) but the passes went through a dense intermediate (a 0-D sparse
        # operand next to an ndarray): same values, stored relative to the probed fill value
        out = np.asarray(out)
        out = COO.from_numpy(np.broadcast_to(out, full) if tuple(out.shape) != tuple(full) else out,
                             fill_value=np.asarray(fv).astype(out.dtype)[()])
    if isinstance(out, SparseArray) and sparse_ops and not any(s == 0 for s in out.shape):
        fmt, kw = _out_format(sparse_ops)  # the format of ONE elemwise call over the three operands
        out = out.asformat("coo").asformat(fmt, **kw)
    return out


def broadcast_to(x, shape):
    """numpy.broadcast_to for COO (reference: _umath.py:344-389); returns a new canonical COO."""
    shape = tuple(int(s) for s in shape)
    if shape == x.shape:
        return x
    result_shape = _get_broadcast_shape(x.shape, shape, is_result=True)
    if any(s == 0 for s in result_shape):  # a length-1 axis stretched to length 0: nothing is left
        return COO(np.empty((len(result_shape), 0), dtype=np.intp), np.empty(0, dtype=x.dtype), shape=result_shape,
                   has_duplicates=False, sorted=True, fill_value=x.fill_value)
    keys, data, R = _stream(x, result_shape)
    if R > 1:
        # materialise the virtual trailing expansion: key = k*R + r
        coords, _ = x._dev()
        nd, off = len(result_shape), len(result_shape) - x.ndim
        bc = [not (d >= off and x.shape[d - off] == result_shape[d]) and result_shape[d] > 1 for d in range(nd)]
        src_row = [(d - off if (d >= off and not bc[d]) else -1) for d in range(nd)]
        is_b = [1 if (bc[d] or src_row[d] < 0) else 0 for d in range(nd)]
        keys, src = Kn.ew_expand(coords, result_shape, is_b, src_row)
        data = Kn.gather(data, src)
    return COO._from_device(None, data, result_shape, x.fill_value, keys=keys)
