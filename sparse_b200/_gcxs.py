"""GCXS container (generalised CSR/CSC) with device-resident data / indices / indptr.

Mirrors sparse/numba_backend/_compressed/compressed.py: `_from_coo` (:25-77), constructor (:135-187),
`tocoo` (:425-460), `change_compressed_axes` (:388-423), O(1) 2-D transpose (:743-768), `_prune` (:816-842).
An N-D array is stored as the 2-D CSR of its (compressed axes ; remaining axes) flattening.
"""
from __future__ import annotations

from collections.abc import Iterable

import numpy as np

from . import _device as D
from . import _kernels as Kn
from ._coo import COO, _is_scipy_sparse
from ._sparse_array import SparseArray
from ._utils import _zero_of_dtype, c_strides, can_store, check_compressed_axes, check_linear_range, key_bits, normalize_axis, prod


class GCXS(SparseArray):
    def __init__(self, arg, shape=None, compressed_axes=None, prune=False, fill_value=None, idx_dtype=None):
        self._data_np = self._indices_np = self._indptr_np = None
        self._data = self._indices = self._indptr = None
        self._idx_vis = None  # index dtype shown to the caller when it is not the device one (int32 / int64)
        if _is_scipy_sparse(arg):
            arg = GCXS.from_scipy_sparse(arg)
        if isinstance(arg, np.ndarray):
            arg = GCXS.from_coo(COO.from_numpy(arg, fill_value=fill_value), compressed_axes)
        elif isinstance(arg, COO):
            arg = GCXS.from_coo(arg, compressed_axes, idx_dtype)
        if isinstance(arg, GCXS):
            if compressed_axes is not None and arg.compressed_axes != tuple(compressed_axes):
                arg = arg.change_compressed_axes(compressed_axes)
            self._adopt(arg)
            if fill_value is not None:
                self.fill_value = self._dtype.type(fill_value)
            if prune:
                self._prune()
            return
        if shape is None:
            raise ValueError("missing `shape` argument")
        shape = tuple(int(s) for s in shape) if isinstance(shape, Iterable) else (int(shape),)
        check_compressed_axes(len(shape), compressed_axes)
        if len(shape) == 1:
            compressed_axes = None
        data, indices, indptr = arg
        dev_in = D.is_device_tensor(data)
        if dev_in:
            self._data, self._indices = data, indices
            self._indptr = indptr if D.is_device_tensor(indptr) else None
            if self._indptr is None:
                self._indptr_np = np.asarray(indptr)
            self._dtype = D.np_dtype(data)
            if data.dim() != 1:
                raise ValueError("data must be a scalar or 1-dimensional.")
        else:
            self._data_np = np.asarray(data)
            self._indices_np = np.asarray(indices)
            self._indptr_np = np.asarray(indptr)
            if self._indices_np.dtype.kind in "iu" and D.device_index_dtype(self._indices_np.dtype) != self._indices_np.dtype:
                self._idx_vis = self._indices_np.dtype
            if self._data_np.ndim != 1:
                raise ValueError("data must be a scalar or 1-dimensional.")
            self._dtype = self._data_np.dtype
        SparseArray.__init__(self, shape, fill_value=None)
        if fill_value is None:
            fill_value = _zero_of_dtype(self._dtype)
        self._compressed_axes = tuple(int(a) for a in compressed_axes) if isinstance(compressed_axes, Iterable) else None
        self.fill_value = self._dtype.type(fill_value)
        if prune:
            self._prune()

    # mode streams of mttkrp_mode ({(mode, int32 indices): (coordinate rows, values)}); belong to the current contents
    _mode_streams = None

    def _adopt(self, o):
        SparseArray.__init__(self, o.shape, fill_value=None)
        self._mode_streams = None
        self._data_np, self._indices_np, self._indptr_np = o._data_np, o._indices_np, o._indptr_np
        self._data, self._indices, self._indptr = o._data, o._indices, o._indptr
        self._idx_vis = o._idx_vis
        self._dtype = o._dtype
        self._compressed_axes = o._compressed_axes
        self.fill_value = o.fill_value

    # ---- pickling: the state is the host mirror -----------------------------------------------------------------------
    def __getstate__(self):
        return {"data": self.data, "indices": self.indices, "indptr": self.indptr, "shape": self.shape,
                "compressed_axes": self.compressed_axes, "fill_value": self.fill_value, "cls": type(self).__name__}

    def __setstate__(self, state):
        GCXS.__init__(self, (state["data"], state["indices"], state["indptr"]), shape=state["shape"],
                      compressed_axes=state["compressed_axes"], fill_value=state["fill_value"])

    def __sizeof__(self):
        return self.nbytes

    def _make_shallow_copy_of(self, other):
        """`out=` target of a ufunc (compressed.py:_make_shallow_copy_of)."""
        self._adopt(other if isinstance(other, GCXS) else GCXS.from_coo(other.asformat("coo"), self.compressed_axes))

    @classmethod
    def _from_device(cls, data, indices, indptr, shape, compressed_axes, fill_value=None):
        self = cls.__new__(cls)
        SparseArray.__init__(self, tuple(int(s) for s in shape), fill_value=None)
        self._data_np = self._indices_np = self._indptr_np = None
        self._data, self._indices, self._indptr = data, indices, indptr
        self._idx_vis = None
        self._dtype = D.np_dtype(data)
        self._compressed_axes = tuple(int(a) for a in compressed_axes) if compressed_axes is not None else None
        self.fill_value = self._dtype.type(0 if fill_value is None else fill_value)
        return self

    # ---- layout metadata (compressed.py:221-262) -----------------------------------------------------------
    @property
    def compressed_axes(self):
        return self._compressed_axes

    @property
    def _axis_order(self):
        axis_order = list(self.compressed_axes)
        axis_order.extend(a for a in range(self.ndim) if a not in set(self.compressed_axes))
        return axis_order

    @property
    def _axisptr(self):
        return len(self.compressed_axes)

    @property
    def _reordered_shape(self):
        return tuple(self.shape[i] for i in self._axis_order)

    @property
    def _compressed_shape(self):
        rs = self._reordered_shape
        return (prod(rs[: self._axisptr]), prod(rs[self._axisptr:]))

    @property
    def dtype(self):
        return self._dtype

    @property
    def nnz(self):
        return int(self._data.shape[0]) if self._data is not None else int(self._data_np.shape[0])

    @property
    def format(self):
        return "gcxs"

    @property
    def nbytes(self):
        isz = self._indices.element_size() if self._indices is not None else self._indices_np.itemsize
        nptr = (self._indptr.shape[0] if self._indptr is not None else len(self._indptr_np))
        return self.nnz * (self._dtype.itemsize + isz) + nptr * isz

    # ---- mirrors ---------------------------------------------------------------------------------------------
    def to_device(self, device=None, /, *, stream=None):
        """Move the arrays to HBM now (they stay resident); returns self."""
        from ._creation import _check_device

        _check_device(device, method=True)
        self._dev()
        return self

    def _dev(self):
        if self._data is None:
            D.require_device()
            self._data = D.upload(self._data_np)
            self._indices = D.upload_index(self._indices_np)
        if self._indptr is None:
            ip = np.asarray(self._indptr_np)
            if ip.size == 0:
                ip = np.zeros(0, dtype=np.int64)
            self._indptr = D.upload_index(ip.astype(D.np_dtype(self._indices)) if ip.dtype != D.np_dtype(self._indices) else ip)
        if self._indptr.dtype != self._indices.dtype:
            self._indptr = Kn.cast(self._indptr, D.np_dtype(self._indices))
        return self._data, self._indices, self._indptr

    @property
    def data(self):
        if self._data_np is None:
            self._data_np = D.download(self._data)
        return self._data_np

    @property
    def indices(self):
        if self._indices_np is None:
            a = D.download(self._indices)
            self._indices_np = a.astype(self._idx_vis) if self._idx_vis is not None else a
        return self._indices_np

    @property
    def indptr(self):
        if self._indptr_np is None:
            a = D.download(self._indptr)
            self._indptr_np = a.astype(self._idx_vis) if self._idx_vis is not None else a
        return self._indptr_np

    def _has_long_rows(self):
        """Is the row-length distribution skewed -- longest compressed row > max(512, 8 x the mean)?  (cached; one device
        reduction per matrix.)  Enables K1's nnz-balanced mode: rows are drawn dynamically by persistent warps and rows
        longer than max(512, 4 x mean) go to the shared-memory-ring kernel (csrc/spmm_skew.cu).  Uniform matrices (the
        C2 headline: Poisson(100) rows, longest ~150) keep the static row-split grid."""
        if getattr(self, "_long_rows_flag", None) is None:
            _, _, indptr = self._dev()
            rows = self._compressed_shape[0]
            self._long_rows_flag = False
            if self.ndim >= 2 and self.nnz > 4096 and rows >= 4096:
                longest = Kn.csr_max_row_nnz(indptr, rows)
                self._long_rows_flag = longest > max(512, 8 * (self.nnz // max(rows, 1)))
        return self._long_rows_flag

    def _rows_sorted(self):
        """Are the indices of every compressed row sorted?  (cached; decides whether K1 may use its panel passes)"""
        if getattr(self, "_rows_sorted_flag", None) is None:
            data, indices, indptr = self._dev()
            self._rows_sorted_flag = Kn.csr_rows_sorted(indices, indptr, self._compressed_shape[0]) if self.ndim >= 2 else True
        return self._rows_sorted_flag

    # ---- COO <-> GCXS ----------------------------------------------------------------------------------------
    @classmethod
    def from_coo(cls, x, compressed_axes=None, idx_dtype=None):
        """_from_coo (compressed.py:25-77) on the device."""
        if x.ndim == 0:
            if compressed_axes is not None:
                raise ValueError("no axes to compress for 0d array")
            _, data = x._dev()
            return cls._from_device(data, x._coords, D.torch().zeros(0, dtype=x._coords.dtype, device=data.device),
                                    x.shape, None, x.fill_value)
        if x.ndim == 1:
            if compressed_axes is not None:
                raise ValueError("no axes to compress for 1d array")
            coords, data = x._dev()
            return cls._from_device(data, coords[0].contiguous(),
                                    D.torch().zeros(0, dtype=coords.dtype, device=data.device), x.shape, None,
                                    x.fill_value)
        if idx_dtype is not None and not can_store(idx_dtype, max(x.shape)):
            raise ValueError(f"cannot cast array with shape {x.shape} to dtype {idx_dtype}.")
        compressed_axes = normalize_axis(compressed_axes, x.ndim)
        if compressed_axes is None:
            compressed_axes = (int(np.argmin(x.shape)),)
        if isinstance(compressed_axes, int):
            compressed_axes = (compressed_axes,)
        check_compressed_axes(x.shape, compressed_axes)
        axis_order = list(compressed_axes)
        axisptr = len(compressed_axes)
        axis_order.extend(a for a in range(x.ndim) if a not in set(compressed_axes))
        reordered_shape = tuple(x.shape[i] for i in axis_order)
        row_size, col_size = prod(reordered_shape[:axisptr]), prod(reordered_shape[axisptr:])
        check_linear_range(x.shape)
        data = x._data_dev()
        # index dtype (compressed.py:52-61): the caller's, else the COO's unless it cannot hold max(rows, cols, nnz)
        need = max(row_size, col_size, x.nnz)
        if idx_dtype is not None:
            idt = np.dtype(idx_dtype)
            if not can_store(idt, need):
                raise ValueError(f"cannot store array with the compressed shape {(row_size, col_size)} and nnz "
                                 f"{x.nnz} with dtype {idt}.")
        else:
            idt = np.dtype(x._idx_dtype())
            if not can_store(idt, need):
                idt = np.dtype(np.min_scalar_type(need))
        vis, idt = idt, D.device_index_dtype(idt)
        if axis_order == list(range(x.ndim)):
            keys = x.sorted_keys()
        else:
            coords = x._dev()[0]
            st = c_strides(reordered_shape)
            strides = [0] * x.ndim
            for pos, a in enumerate(axis_order):
                strides[a] = st[pos]
            keys = Kn.linearize(coords, strides)
            unsorted, _ = Kn.keys_flags(keys)
            if unsorted:
                keys, perm = Kn.sort_keys(keys, key_bits(x.size))
                data = Kn.gather(data, perm)
        _, indices, indptr = Kn.csr_from_keys(keys, row_size, col_size, idt)
        out = cls._from_device(data, indices, indptr, x.shape, compressed_axes, x.fill_value)
        out._idx_vis = vis if vis != idt else None
        return out

    def tocoo(self):
        """compressed.py:425-460: rows from indptr, then undo the axis reordering (COO rebuild + sort)."""
        data, indices, indptr = self._dev()
        if self.ndim == 0:
            return COO._from_device(indices.reshape(0, int(data.shape[0])), data, self.shape, self.fill_value)
        if self.ndim == 1:
            return COO(indices[None, :], data, shape=self.shape, fill_value=self.fill_value)
        nrows, ncols = self._compressed_shape
        idt = D.np_dtype(indices)
        rows = Kn.rows_from_indptr(indptr, self.nnz, idt)
        t = D.torch()
        coords2 = t.stack([rows, indices])
        keys2 = Kn.linearize(coords2, [ncols, 1])
        axis_order = self._axis_order
        if axis_order == list(range(self.ndim)):
            keys = keys2
        else:
            # key over the reordered shape -> key over the original shape
            re_coords = Kn.unravel(keys2, self._reordered_shape, np.int64)
            st = c_strides(self.shape)
            keys = Kn.linearize(re_coords, [st[a] for a in axis_order])
        unsorted, _ = Kn.keys_flags(keys)
        if unsorted:
            keys, perm = Kn.sort_keys(keys, key_bits(self.size))
            data = Kn.gather(data, perm)
        return COO._from_device(None, data, self.shape, self.fill_value, keys=keys)  # coordinates derived lazily

    @classmethod
    def from_iter(cls, x, shape=None, compressed_axes=None, fill_value=None, idx_dtype=None):
        """compressed.py:221-227: through COO.from_iter."""
        return cls.from_coo(COO.from_iter(x, shape, fill_value), compressed_axes, idx_dtype)

    @classmethod
    def from_numpy(cls, x, compressed_axes=None, fill_value=None, idx_dtype=None):
        return cls.from_coo(COO.from_numpy(x, fill_value=fill_value, idx_dtype=idx_dtype), compressed_axes)

    @classmethod
    def from_scipy_sparse(cls, x, /, *, fill_value=None):
        """compressed.py:210-219: CSC input stays column-compressed, anything else goes through CSR; non-canonical
        input (duplicates, explicit zeros, unsorted rows) is canonicalised by SciPy on the host before the upload."""
        is_csc = x.format == "csc"
        ca = (1,) if is_csc else (0,)
        if not is_csc:
            x = x.asformat("csr")
        if not x.has_canonical_format:
            x = x.copy()
            x.eliminate_zeros()
            x.sum_duplicates()
        return cls((x.data, x.indices, x.indptr), shape=x.shape, compressed_axes=ca, fill_value=fill_value)

    def todense(self):
        return self.tocoo().todense()

    def todense_device(self):
        return self.tocoo().todense_device()

    def copy(self, deep=True):
        """compressed.py:copy -- deep: the three arrays are cloned (device clone and host mirrors alike)."""
        out = type(self).__new__(type(self))
        out._adopt(self)
        if deep:
            for name in ("_data", "_indices", "_indptr"):
                dev, host = getattr(self, name), getattr(self, name + "_np")
                setattr(out, name, dev.clone() if dev is not None else None)
                setattr(out, name + "_np", host.copy() if host is not None else None)
        return out

    def to_scipy_sparse(self, accept_fv=None):
        """compressed.py:495-525: csr_array when axis 0 is compressed, else csc_array."""
        import scipy.sparse

        from ._utils import check_fill_value

        check_fill_value(self, accept_fv=accept_fv)
        if self.ndim != 2:
            raise ValueError("Can only convert a 2-dimensional array to a Scipy sparse matrix.")
        cls = scipy.sparse.csr_array if 0 in self.compressed_axes else scipy.sparse.csc_array
        return cls((self.data, self.indices, self.indptr), shape=self.shape)

    def asformat(self, format, **kwargs):
        """compressed.py:asformat -- "gcxs" / "csr" / "csc" / "coo" / "dense" (names or classes)."""
        from ._dok import DOK

        if isinstance(format, str):
            format = {"gcxs": GCXS, "csr": CSR, "csc": CSC, "coo": COO, "dok": DOK, "dense": np.ndarray}.get(format,
                                                                                                              format)
        if isinstance(format, type) and issubclass(format, DOK):
            if kwargs:
                raise ValueError(f"Extra kwargs found: {kwargs}")
            return DOK.from_coo(self.tocoo())
        if isinstance(format, type) and issubclass(format, (CSR, CSC)):
            if kwargs:
                raise ValueError(f"Extra kwargs found: {kwargs}")
            return format(self)
        if format is GCXS or (isinstance(format, type) and issubclass(format, GCXS)):
            ca = kwargs.pop("compressed_axes", None)
            if kwargs:
                raise ValueError(f"Extra kwargs found: {kwargs}")
            if ca is None:
                return self if type(self) is GCXS else GCXS(self)
            return GCXS(self).change_compressed_axes(ca) if type(self) is not GCXS else self.change_compressed_axes(ca)
        if kwargs:
            raise ValueError(f"Extra kwargs found: {kwargs}")
        if format is COO or (isinstance(format, type) and issubclass(format, COO)):
            return self.tocoo()
        if format is np.ndarray:
            return self.todense()
        raise NotImplementedError(f"The given format is not supported: {format}")

    def astype(self, dtype, casting="unsafe", copy=True, _keep_format=False):
        """Cast; entries that become equal to the fill value are pruned, as upstream's elemwise-based astype does.
        (`_keep_format`: internal casts of intermediate results stay GCXS also when the array is empty.)"""
        dtype = np.dtype(dtype)
        if self.dtype == dtype and not copy:
            return self
        if not np.can_cast(self.dtype, dtype, casting=casting):
            raise TypeError(f"Cannot cast array data from {self.dtype!r} to {dtype!r} according to the rule {casting!r}")
        if self.ndim == 0 and not _keep_format:
            return self.tocoo().astype(dtype, casting=casting, copy=copy).asformat("gcxs")  # value-as-fill, see COO
        if any(s == 0 for s in self.shape) and not _keep_format:
            # upstream's astype is an elemwise call, and elemwise hands back the empty COO as it is (_umath.py:467-477)
            return self.tocoo().astype(dtype, casting=casting, copy=copy)
        data, indices, indptr = self._dev()
        if dtype != self.dtype and (self.dtype.kind == "c" or dtype.kind == "c"):
            from ._complex import cast_values

            data = cast_values(data, self.dtype, dtype)
        out = GCXS._from_device(Kn.cast(data, dtype) if dtype != D.np_dtype(data) else
                                (data.clone() if dtype == self.dtype else data), indices, indptr,
                                self.shape, self.compressed_axes, np.asarray(self.fill_value).astype(dtype)[()])
        out._prune()  # always: upstream's elemwise-based astype also drops fill values that were stored explicitly
        return out

    def change_compressed_axes(self, new_compressed_axes):
        """compressed.py:388-423."""
        if new_compressed_axes is not None:
            new_compressed_axes = tuple(normalize_axis(a, self.ndim) for a in new_compressed_axes)
        if new_compressed_axes == self.compressed_axes:
            return self
        if self.ndim == 1:
            raise NotImplementedError("no axes to compress for 1d array")
        if len(new_compressed_axes) >= len(self.shape):
            raise ValueError("cannot compress all axes")
        if len(set(new_compressed_axes)) != len(new_compressed_axes):
            raise ValueError("repeated axis in compressed_axes")
        return GCXS.from_coo(self.tocoo(), new_compressed_axes)

    # ---- transpose ---------------------------------------------------------------------------------------------
    def _2d_transpose(self):
        """O(1): CSR of (m, n) is CSC of (n, m) (compressed.py:743-768)."""
        ca = [(self.compressed_axes[0] + 1) % 2]
        data, indices, indptr = self._dev()
        return GCXS._from_device(data, indices, indptr, self.shape[::-1], ca, self.fill_value)

    def transpose(self, axes=None, compressed_axes=None):
        if axes is None:
            axes = tuple(reversed(range(self.ndim)))
        axes = tuple(int(a) + self.ndim if int(a) < 0 else int(a) for a in axes)
        if self.ndim == 2 and axes == (1, 0) and compressed_axes is None:
            return self._2d_transpose()
        if axes == tuple(range(self.ndim)):
            return self
        if self.ndim == 1:
            return self
        out = self.tocoo().transpose(axes)
        return GCXS.from_coo(out, compressed_axes)

    @property
    def T(self):
        return self.transpose()

    @property
    def mT(self):
        if self.ndim < 2:
            raise ValueError("Cannot compute matrix transpose if `ndim < 2`.")
        axes = list(range(self.ndim))
        axes[-1], axes[-2] = axes[-2], axes[-1]
        return self.transpose(axes)

    def reshape(self, shape, order="C", compressed_axes=None):
        """compressed.py:622-682."""
        shape = tuple(shape) if isinstance(shape, Iterable) else (shape,)
        if order not in {"C", None}:
            raise NotImplementedError("The 'order' parameter is not supported")
        shape = tuple(int(s) for s in shape)
        if any(d == -1 for d in shape):
            extra = int(self.size / np.prod([d for d in shape if d != -1]))
            shape = tuple(d if d != -1 else extra for d in shape)
        if self.shape == shape:
            return self
        if self.size != prod(shape):
            raise ValueError(f"cannot reshape array of size {self.size} into shape {shape}")
        if len(shape) == 0:
            return GCXS.from_coo(self.tocoo().reshape(shape))
        if compressed_axes is None:
            if len(shape) == self.ndim:
                compressed_axes = self.compressed_axes
            elif len(shape) == 1:
                compressed_axes = None
            else:
                compressed_axes = (int(np.argmin(shape)),)
        return GCXS.from_coo(self.tocoo().reshape(shape), compressed_axes)

    def flatten(self, order="C"):
        return self.reshape(-1)

    def __getitem__(self, index):
        """Integers, slices, None, Ellipsis (_compressed/indexing.py:14-174); see _indexing.py."""
        from ._indexing import gcxs_getitem

        return gcxs_getitem(self, index)

    # ---- prune (compressed.py:816-842) ---------------------------------------------------------------------------
    def _prune(self):
        data, indices, indptr = self._dev()
        if self.nnz == 0:
            return
        flags = Kn.flag_not_fill(data, self.fill_value)
        pos, total = Kn.scan_flags(flags)
        if total == self.nnz:
            return
        self._mode_streams = None
        self._data = Kn.compact(data, flags, pos, total)
        self._indices = Kn.compact(indices, flags, pos, total)
        if self.ndim > 1:
            self._indptr = Kn.indptr_remap(indptr, pos, int(flags.shape[0]), total)
        self._data_np = self._indices_np = self._indptr_np = None

    # ---- products ---------------------------------------------------------------------------------------------------
    def dot(self, other):
        from ._dot import dot

        return dot(self, other)

    def __matmul__(self, other):
        from ._dot import matmul

        try:
            return matmul(self, other)
        except NotImplementedError:
            return NotImplemented

    def __rmatmul__(self, other):
        from ._dot import matmul

        try:
            return matmul(other, self)
        except NotImplementedError:
            return NotImplemented


class _Compressed2d(GCXS):
    """2-D specialisations (compressed.py:851-949): fixed compressed axis, O(1) transpose into the sibling class."""

    class_compressed_axes = None

    def __init__(self, arg, shape=None, compressed_axes=None, prune=False, fill_value=None):
        if compressed_axes is None:
            compressed_axes = self.class_compressed_axes
        if tuple(compressed_axes) != self.class_compressed_axes:
            what = "rows" if self.class_compressed_axes == (0,) else "columns"
            raise ValueError(f"{type(self).__name__} only accepts {what} as compressed axis but got: {compressed_axes}")
        if not hasattr(arg, "shape") and shape is None:
            raise ValueError("missing `shape` argument")
        if shape is not None and hasattr(arg, "shape"):
            raise NotImplementedError("Cannot change shape in constructor")
        nd = len(shape if shape is not None else arg.shape)
        if nd != 2:
            raise ValueError(f"{type(self).__name__} must be 2-d, passed {nd}-d shape.")
        super().__init__(arg, shape=shape, compressed_axes=self.class_compressed_axes, prune=prune,
                         fill_value=fill_value)

    @property
    def ndim(self):
        return 2

    @classmethod
    def from_numpy(cls, x, fill_value=0, idx_dtype=None):
        return cls(GCXS.from_coo(COO.from_numpy(x, fill_value=fill_value, idx_dtype=idx_dtype),
                                 cls.class_compressed_axes, idx_dtype))

    @classmethod
    def from_coo(cls, x, compressed_axes=None, idx_dtype=None):
        return cls(GCXS.from_coo(x, cls.class_compressed_axes, idx_dtype))

    @classmethod
    def from_scipy_sparse(cls, x, /, *, fill_value=None):
        fmt = "csr" if cls.class_compressed_axes == (0,) else "csc"
        x = x.asformat(fmt, copy=False)
        if not x.has_canonical_format:
            x = x.copy()
            x.eliminate_zeros()
            x.sum_duplicates()
        return cls((x.data, x.indices, x.indptr), shape=x.shape, fill_value=fill_value)

    def transpose(self, axes=None, copy=False, compressed_axes=None):
        """compressed.py:915-923: CSR of (m, n) IS the CSC of (n, m) -- the three arrays are shared, not copied."""
        axes = normalize_axis(axes, self.ndim) if axes is not None else None
        if axes not in [(0, 1), (1, 0), None]:
            raise ValueError(f"Invalid transpose axes: {axes}")
        src = self.copy() if copy else self
        if axes == (0, 1):
            return src
        if not copy and src.nbytes <= (64 << 20):
            src.data, src.indices, src.indptr  # small arrays: both views hand out the SAME host mirrors
        other = CSC if isinstance(self, CSR) else CSR
        out = other.__new__(other)
        out._adopt(src)
        out.shape = src.shape[::-1]
        out._compressed_axes = other.class_compressed_axes
        return out


class CSR(_Compressed2d):
    """2-D GCXS with compressed_axes=(0,)."""

    class_compressed_axes = (0,)


class CSC(_Compressed2d):
    """2-D GCXS with compressed_axes=(1,)."""

    class_compressed_axes = (1,)
