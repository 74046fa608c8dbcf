"""COO container with device-resident coordinates and data.

Mirrors sparse/numba_backend/_coo/core.py: constructor normalisation (sort / sum duplicates / prune,
:198-291, :1294-1371), transpose (:725-807), reshape (:1034-1111), linear_loc, todense, asformat.
The arrays live in HBM as torch CUDA tensors (moved there once); `.coords` / `.data` materialise NumPy
mirrors lazily.  Every data-path step runs in libsparse_b200 kernels -- there is no CPU fallback: a COO
whose construction needs work (unsorted input, duplicates, pruning) requires a CUDA device.
"""
from __future__ import annotations

from collections.abc import Iterable

import numpy as np

from . import _device as D
from . import _kernels as Kn
from ._sparse_array import SparseArray
from ._utils import _zero_of_dtype, c_strides, can_store, check_linear_range, key_bits, normalize_axis, prod


def _segment_sum(data, heads, pos, total):
    """Kn.segment_sum for the compute dtypes, per plane for complex values (sparse_b200/_complex.py)."""
    if data.is_complex():
        from ._complex import segment_sum

        return segment_sum(data, heads, pos, total)
    dt = D.np_dtype(data)
    if dt not in D._CODES and dt.kind in "iu":
        # storage-only integer widths: sum in int64, cast back (two's-complement wrap = NumPy's reduceat in that dtype)
        return Kn.cast(Kn.segment_sum(Kn.cast(data, np.int64), heads, pos, total), dt)
    return Kn.segment_sum(data, heads, pos, total)


def _is_scipy_sparse(x):
    mod = type(x).__module__
    return mod.startswith("scipy.sparse") and hasattr(x, "tocoo")


class COO(SparseArray):
    """N-D sparse array in coordinate format: ``coords[ndim, nnz]`` + ``data[nnz]``."""

    def __init__(self, coords, data=None, shape=None, has_duplicates=True, sorted=False, prune=False, cache=False,
                 fill_value=None, idx_dtype=None):
        self._coords_np = None
        self._data_np = None
        self._coords = None  # device [ndim, nnz]
        self._data = None    # device [nnz]
        self._keys = None    # device sorted linear keys (cache)
        self._cache = {} if cache else None  # opt-in result cache of transpose / reshape / tocsr / tocsc
        self._idx_vis = None  # index dtype shown to the caller when it is not the device one (int32 / int64)

        if isinstance(coords, COO):
            if data is not None or shape is not None:
                raise ValueError("If `coords` is `COO`, then no other arguments should be provided.")
            self._copy_from(coords)
            if fill_value is not None:
                self.fill_value = self.dtype.type(fill_value)
            return

        if data is None:
            arr = as_coo(coords, shape=shape, fill_value=fill_value, idx_dtype=idx_dtype)
            self._copy_from(arr)
            if idx_dtype is not None and self.ndim:
                if not can_store(idx_dtype, max(self.shape)):
                    raise ValueError(f"cannot cast array with shape {self.shape} to dtype {idx_dtype}.")
            return

        dev_in = D.is_device_tensor(coords) or D.is_device_tensor(data)
        if dev_in:
            t = D.torch()
            if not D.is_device_tensor(coords):
                coords = D.upload_index(np.asarray(coords))
            if not D.is_device_tensor(data):
                data = D.upload(np.asarray(data))
            if coords.dim() == 1:
                coords = coords[None, :]
            if data.dim() == 0:
                data = data.expand(coords.shape[1]).contiguous()
            self._coords, self._data = coords, data
            nnz, ndim_c = int(coords.shape[1]), int(coords.shape[0])
            self._dtype = D.np_dtype(data)
            if data.dim() != 1:
                raise ValueError("`data` must be a scalar or 1-dimensional.")
        else:
            data = np.asarray(data)
            coords = np.asarray(coords)
            if coords.ndim == 1:
                if coords.size == 0 and shape is not None:
                    coords = coords.reshape((len(shape) if isinstance(shape, Iterable) else 1, len(data)))
                else:
                    coords = coords[None, :]
            if data.ndim == 0:
                data = np.broadcast_to(data, coords.shape[1])
            if data.ndim != 1:
                raise ValueError("`data` must be a scalar or 1-dimensional.")
            if coords.dtype.kind not in "iu":
                coords = coords.astype(np.intp)
            if D.device_index_dtype(coords.dtype) != coords.dtype:
                self._idx_vis = coords.dtype
            self._coords_np, self._data_np = coords, data
            nnz, ndim_c = int(coords.shape[1]), int(coords.shape[0])
            self._dtype = data.dtype

        if shape is None:
            raise ValueError("`shape` was not provided.")
        if not isinstance(shape, Iterable):
            shape = (shape,)
        shape = tuple(int(s) for s in shape)
        if shape and nnz == 0 and not dev_in:
            self._coords_np = np.zeros((len(shape), 0), dtype=np.intp)
            ndim_c = len(shape)
        super().__init__(shape, fill_value=None)
        if fill_value is None:
            fill_value = _zero_of_dtype(self._dtype)
        self.fill_value = self._dtype.type(fill_value)

        if idx_dtype:
            if not can_store(idx_dtype, max(shape) if shape else 0):
                raise ValueError(f"cannot cast array with shape {shape} to dtype {idx_dtype}.")
            idx_dtype = np.dtype(idx_dtype)
            dev_dt = D.device_index_dtype(idx_dtype)
            self._idx_vis = idx_dtype if dev_dt != idx_dtype else None
            if self._coords_np is not None:
                self._coords_np = self._coords_np.astype(idx_dtype)
            else:
                self._coords = Kn.cast(self._coords, dev_dt)
        if self.shape:
            dlen = int(self._data.shape[0]) if self._data is not None else len(self._data_np)
            if dlen != nnz:
                raise ValueError("The data length does not match the coordinates given.\n"
                                 f"len(data) = {dlen}, but {nnz} coords specified.")
            if len(self.shape) != ndim_c:
                raise ValueError("Shape specified by `shape` doesn't match the shape of `coords`; "
                                 f"len(shape)={len(shape)} != coords.shape[0]={ndim_c}")
        check_linear_range(self.shape)
        from . import _settings

        if _settings.WARN_ON_TOO_DENSE and self.nbytes >= self.size * self._dtype.itemsize:
            import warnings

            warnings.warn("Attempting to create a sparse array that takes no less memory than than an equivalent "
                          "dense array. You may want to use a dense array here instead.", RuntimeWarning, stacklevel=1)
        if (not sorted) or has_duplicates or prune:
            self._canonicalise(check_sort=not sorted, sum_dups=has_duplicates, prune=prune)

    # ---- construction helpers ------------------------------------------------------------------------
    # mode streams of mttkrp_mode ({(mode, int32 indices): (coordinate rows, values)}) and fiber streams of ttm_mode
    # ({("fiber", mode, int32 indices): ...}); belong to the current contents
    _mode_streams = None

    def _copy_from(self, other):
        SparseArray.__init__(self, other.shape, fill_value=None)
        self._mode_streams = None
        self._coords_np, self._data_np = other._coords_np, other._data_np
        self._coords, self._data, self._keys = other._coords, other._data, other._keys
        self._idx_vis = other._idx_vis
        self._dtype = other._dtype
        self.fill_value = other.fill_value

    def _make_shallow_copy_of(self, other):
        """`out=` target of a ufunc (_coo/core.py:_make_shallow_copy_of): adopt the result's arrays."""
        self._copy_from(other.asformat("coo") if not isinstance(other, COO) else other)
        # results cached for the OLD contents (enable_caching) are stale now; upstream replaces __dict__, i.e. takes
        # the result's cache (None)
        self._cache = None

    @classmethod
    def _from_device(cls, coords, data, shape, fill_value=None, keys=None):
        """Wrap canonical device arrays without any checks.  coords may be None when `keys` (sorted linear keys over
        `shape`) is given: the coordinate rows are then derived lazily."""
        assert coords is not None or keys is not None
        self = cls.__new__(cls)
        SparseArray.__init__(self, tuple(int(s) for s in shape), fill_value=None)
        self._coords_np = self._data_np = None
        self._coords, self._data, self._keys = coords, data, keys
        self._idx_vis = None
        self._dtype = D.np_dtype(data)
        self.fill_value = self._dtype.type(0 if fill_value is None else fill_value)
        return self

    @classmethod
    def from_iter(cls, x, shape=None, fill_value=None, dtype=None):
        """COO from `{(i, j): v}`, `[((i, j), v), ...]`, `(data, (row, col))` or an iterator of the second form
        (_coo/core.py:469-560): host-side parsing of the input into coordinate / value arrays, then the constructor."""
        from collections.abc import Sized

        if isinstance(x, dict):
            if shape is None:
                raise TypeError("`shape` must be given when converting a dictionary to COO.")
            x = list(x.items())
        if not isinstance(x, Sized):
            x = list(x)
        if len(x) != 2 and not all(len(item) == 2 for item in x):
            raise ValueError("Invalid iterable to convert to COO.")
        if not x:
            ndim = 0 if shape is None else len(shape)
            coords = np.empty((ndim, 0), dtype=np.intp)
            data = np.empty((0,), dtype=dtype)
            shape = () if shape is None else shape
        elif not isinstance(x[0][0], Iterable):
            coords = np.stack([np.asarray(c) for c in x[1]], axis=0)
            data = np.asarray(x[0], dtype=dtype)
        else:
            coords = np.array([item[0] for item in x]).T
            data = np.array([item[1] for item in x], dtype=dtype)
        if not (coords.ndim == 2 and data.ndim == 1 and np.issubdtype(coords.dtype, np.integer)
                and np.all(coords >= 0)):
            raise ValueError("Invalid iterable to convert to COO.")
        return cls(coords, data, shape=shape, fill_value=fill_value)

    # ---- pickling: the state is the host mirror (device tensors are re-created lazily on the receiving side) --------
    def __getstate__(self):
        return {"coords": self.coords, "data": self.data, "shape": self.shape, "fill_value": self.fill_value}

    def __setstate__(self, state):
        self.__init__(state["coords"], state["data"], shape=state["shape"], has_duplicates=False, sorted=True,
                      fill_value=state["fill_value"])  # the cache is not part of the state

    def __sizeof__(self):
        return self.nbytes

    _cache = None

    def enable_caching(self):
        """Opt-in result cache (_coo/core.py:`cache=True`): repeated `transpose` / `reshape` / `tocsr` / `tocsc` calls
        with the same arguments hand back the same object; the three most recent results per method are kept."""
        if self._cache is None:
            self._cache = {}
        return self

    def _cached(self, name, key, compute):
        if self._cache is None:
            return compute()
        import collections

        bucket = self._cache.setdefault(name, collections.deque(maxlen=3))
        for k, v in bucket:
            if k == key:
                return v
        v = compute()
        if isinstance(v, COO) and v is not self and v._cache is None:
            v._cache = {}  # results of a caching array cache as well (chains like x.reshape(..).T.tocsr())
        bucket.append((key, v))
        return v

    @classmethod
    def from_numpy(cls, x, fill_value=None, idx_dtype=None):
        """Dense ndarray -> COO (_coo/core.py:from_numpy): entries bitwise different from the fill value."""
        x = np.asanyarray(x).view(type=np.ndarray)
        if idx_dtype is not None and x.ndim and not can_store(idx_dtype, max(x.shape)):
            raise ValueError(f"cannot cast array with shape {x.shape} to dtype {idx_dtype}.")
        if fill_value is None:
            # 0-D: the element itself becomes the fill value (nnz = 0), _coo/core.py:371-372
            fill_value = _zero_of_dtype(x.dtype) if x.shape else x[()]
        fill_value = x.dtype.type(fill_value)
        if x.ndim == 0:
            from ._utils import equivalent

            keep = 0 if bool(equivalent(x, fill_value)) else 1
            return cls(np.empty((0, keep), dtype=np.intp), x.reshape(-1)[:keep], shape=(), has_duplicates=False,
                       sorted=True, fill_value=fill_value)
        D.require_device()
        xd = D.upload(np.ascontiguousarray(x))
        return cls._from_dense_device(xd, x.shape, fill_value, idx_dtype)

    @classmethod
    def _from_dense_device(cls, xd, shape, fill_value, idx_dtype=None):
        n = prod(shape)
        flat = xd.reshape(1, n)
        if D.np_dtype(xd) not in D._CODES:
            # storage-only dtypes (narrow / unsigned integers, float16, complex): element-size generic flag + compact
            flags = Kn.flag_not_fill(flat.reshape(-1), fill_value)
            pos, total = Kn.scan_flags(flags)
            keys = Kn.compact(Kn.iota(n), flags, pos, total)
            data = Kn.compact(flat.reshape(-1), flags, pos, total)
        elif np.dtype(D.np_dtype(xd)).type(fill_value).tobytes() == b"\0" * xd.element_size():
            _, keys, data, _ = Kn.dense_to_csr(flat, mode=1, want_indptr=False)
        else:
            flags = Kn.flag_not_fill(flat.reshape(-1), fill_value)
            _, keys, data, _ = Kn.dense_to_csr(flat, flags=flags.reshape(1, n), want_indptr=False)
        dev_dt = D.device_index_dtype(idx_dtype or np.int64)
        out = cls._from_device(Kn.unravel(keys, shape, dev_dt), data, shape, fill_value, keys=keys)
        if idx_dtype is not None and np.dtype(idx_dtype) != dev_dt:
            out._idx_vis = np.dtype(idx_dtype)
        return out

    @classmethod
    def from_scipy_sparse(cls, x, /, *, fill_value=None):
        """_coo/core.py:424-467; non-canonical input is canonicalised by SciPy on the host before the upload."""
        x = x.asformat("coo")
        if not x.has_canonical_format:
            x = x.copy()
            x.eliminate_zeros()
            x.sum_duplicates()
        coords = np.stack([x.row, x.col]) if not hasattr(x, "coords") else np.stack(x.coords)
        return cls(coords, x.data, shape=x.shape, has_duplicates=not x.has_canonical_format,
                   sorted=x.has_canonical_format, fill_value=fill_value)

    # ---- device / host mirrors -----------------------------------------------------------------------
    def to_device(self, device=None, /, *, stream=None):
        """Move the arrays to HBM now (they stay resident); returns self."""
        from ._creation import _check_device

        _check_device(device, method=True)
        self._dev()
        return self

    def _dev(self):
        """(coords, data) on the device.  Coordinates are LAZY: results of device operations carry only their sorted
        linear keys (8 B/entry instead of 8*ndim B); the coordinate rows are unravelled the first time they are asked
        for (a user reading `.coords`, or an axis permutation)."""
        if self._data is None:
            D.require_device()
            self._coords = D.upload_index(self._coords_np)
            self._data = D.upload(self._data_np)
        if self._coords is None:
            self._coords = Kn.unravel(self._keys, self.shape, np.int64)
        return self._coords, self._data

    def _data_dev(self):
        """Device data only (does not materialise lazy coordinates)."""
        if self._data is None:
            self._dev()
        return self._data

    def _idx_dtype(self):
        if self._idx_vis is not None:
            return self._idx_vis
        if self._coords is not None:
            return D.np_dtype(self._coords)
        if self._coords_np is not None:
            return self._coords_np.dtype
        return np.dtype(np.int64)

    @property
    def coords(self):
        if self._coords_np is None:
            c = D.download(self._dev()[0])
            self._coords_np = c.astype(self._idx_vis) if self._idx_vis is not None else c
        return self._coords_np

    @property
    def data(self):
        if self._data_np is None:
            self._data_np = D.download(self._data)
        return self._data_np

    @property
    def dtype(self):
        return self._dtype

    @property
    def nnz(self):
        if self._data is not None:
            return int(self._data.shape[0])
        return int(self._data_np.shape[0])

    @property
    def nbytes(self):
        c_item = self._idx_dtype().itemsize
        return self.nnz * (self._dtype.itemsize + self.ndim * c_item)

    @property
    def format(self):
        return "coo"

    # ---- canonicalisation (COO.__init__ tail, _coo/core.py:283-291) -----------------------------------
    def sorted_keys(self):
        """Device linear keys (C order over self.shape) of the canonical entries; cached."""
        if self._keys is None:
            coords, _ = self._dev()
            self._keys = Kn.linearize(coords, c_strides(self.shape))
        return self._keys

    def _canonicalise(self, check_sort=True, sum_dups=True, prune=False):
        coords, data = self._dev()
        nnz = int(data.shape[0])
        if nnz == 0:
            self._keys = None
            return
        keys = Kn.linearize(coords, c_strides(self.shape))
        changed = False
        unsorted, dups = Kn.keys_flags(keys)
        if check_sort and unsorted:
            keys, perm = Kn.sort_keys(keys, key_bits(self.size))
            data = Kn.gather(data, perm)
            changed = True
            _, dups = Kn.keys_flags(keys)
        if sum_dups and dups:
            heads = Kn.flag_heads(keys)
            pos, total = Kn.scan_flags(heads)
            data = _segment_sum(data, heads, pos, total)
            keys = Kn.compact(keys, heads, pos, total)
            changed = True
        if prune:
            flags = Kn.flag_not_fill(data, self.fill_value)
            pos, total = Kn.scan_flags(flags)
            if total != int(data.shape[0]):
                data = Kn.compact(data, flags, pos, total)
                keys = Kn.compact(keys, flags, pos, total)
                changed = True
        if changed:
            self._mode_streams = None
            idt = D.np_dtype(coords)
            # keep the caller's index dtype when it is not int64; otherwise derive coordinates lazily from the keys
            self._coords = Kn.unravel(keys, self.shape, idt) if idt != np.dtype(np.int64) else None
            self._data = data
            self._coords_np = self._data_np = None
        if not (unsorted and not check_sort):
            self._keys = keys  # keys are sorted (or the caller vouched for the order)
        elif self._coords is None:
            self._coords = Kn.unravel(keys, self.shape, np.int64)  # unsorted by request: no key cache

    # ---- conversions ----------------------------------------------------------------------------------
    def todense(self):
        """Dense NumPy array (device scatter into a fill-initialised buffer, then one D2H)."""
        return D.download(self.todense_device())

    def todense_device(self):
        data = self._data_dev()
        out = Kn.full(max(self.size, 1) if self.ndim == 0 else self.size, self.fill_value, self._dtype)
        if self.ndim == 0:
            if self.nnz:
                out[:1] = data[:1]
            return out[:1].reshape(())
        if self.nnz:
            Kn.scatter(data, self.sorted_keys(), out)
        return out.reshape(self.shape)

    def tocoo(self):
        return self

    def copy(self, deep=True):
        """Shallow: the same arrays; deep: clones (device tensors and host mirrors alike).  The cache is not copied."""
        out = COO.__new__(COO)
        out._copy_from(self)
        out._cache = None
        if deep:
            for name in ("_coords", "_data", "_keys"):
                v = getattr(self, name)
                setattr(out, name, v.clone() if v is not None else None)
            for name in ("_coords_np", "_data_np"):
                v = getattr(self, name)
                setattr(out, name, v.copy() if v is not None else None)
        elif self.nbytes <= (64 << 20):
            out.coords, out.data  # small arrays: materialise the host mirrors once, both objects hand out the same arrays
            self._coords_np, self._data_np = out._coords_np, out._data_np
        return out

    def asformat(self, format, **kwargs):
        """_coo/core.py:asformat -- "coo" / "gcxs" / "csr" / "csc" / "dense" (names or classes)."""
        from ._gcxs import CSC, CSR, GCXS

        from ._dok import DOK

        if isinstance(format, str):
            format = {"coo": COO, "gcxs": GCXS, "csr": CSR, "csc": CSC, "dok": DOK, "dense": np.ndarray}.get(format,
                                                                                                              format)
        if isinstance(format, type) and issubclass(format, DOK):
            if kwargs:
                raise ValueError(f"Extra kwargs found: {kwargs}")
            return DOK.from_coo(self)
        if isinstance(format, type) and issubclass(format, (CSR, CSC)):
            if kwargs:
                raise ValueError(f"Extra kwargs found: {kwargs}")
            return format(self)
        if isinstance(format, type) and issubclass(format, GCXS):
            return GCXS.from_coo(self, **kwargs)
        if kwargs:
            raise ValueError(f"Extra kwargs found: {kwargs}")
        if isinstance(format, type) and issubclass(format, COO):
            return self
        if format is np.ndarray:
            return self.todense()
        raise NotImplementedError(f"The given format is not supported: {format}")

    # ---- SciPy interop (_coo/core.py:1166-1260): host objects built from one D2H of the component arrays -------
    def to_scipy_sparse(self, /, *, accept_fv=None):
        import scipy.sparse

        from ._utils import check_fill_value

        check_fill_value(self, accept_fv=accept_fv)
        result = scipy.sparse.coo_array((self.data, tuple(self.coords)), shape=self.shape)  # n-D with SciPy >= 1.13
        result.has_canonical_format = True
        return result

    def tocsr(self):
        """scipy.sparse.csr_array (row pointer built on the device by the CSR conversion kernels)."""
        import scipy.sparse

        from ._utils import check_zero_fill_value

        check_zero_fill_value(self)
        if self.ndim != 2:
            raise ValueError("This array must be two-dimensional for this conversion to work.")
        def build():
            g = self.asformat("gcxs", compressed_axes=(0,))
            return scipy.sparse.csr_array((g.data, g.indices, g.indptr), shape=self.shape)

        return self._cached("tocsr", (), build)

    def tocsc(self):
        import scipy.sparse

        from ._utils import check_zero_fill_value

        check_zero_fill_value(self)
        if self.ndim != 2:
            raise ValueError("This array must be two-dimensional for this conversion to work.")
        def build():
            g = self.asformat("gcxs", compressed_axes=(1,))
            return scipy.sparse.csc_array((g.data, g.indices, g.indptr), shape=self.shape)

        return self._cached("tocsc", (), build)

    def astype(self, dtype, casting="unsafe", copy=True, _raw=False):
        """Cast of the stored values and the fill value (`_raw`: internal casts of intermediate results keep a 0-D
        array's stored entry / fill value structure).  Upstream routes this through `elemwise`
        (_sparse_array.py:626-643), so values that BECOME equal to the fill value under the cast (0.4 -> int 0, a
        double that underflows to float32 0) are dropped from the result; same here (flag, scan, compact)."""
        dtype = np.dtype(dtype)
        if self.dtype == dtype and not copy:
            return self
        if not np.can_cast(self.dtype, dtype, casting=casting):
            raise TypeError(f"Cannot cast array data from {self.dtype!r} to {dtype!r} according to the rule {casting!r}")
        if self.ndim == 0 and not _raw:
            # a 0-D operand is a scalar to upstream's elemwise (_umath.py:438-439): the cast VALUE comes back as the
            # fill value of an array without stored entries, whatever was stored before
            return COO(np.empty((0, 0), dtype=np.intp), np.empty(0, dtype=dtype), shape=(), has_duplicates=False,
                       sorted=True, fill_value=np.asarray(self.todense()).astype(dtype)[()])
        data = self._data_dev()
        fill = np.asarray(self.fill_value).astype(dtype)[()]
        if self.dtype == dtype:
            vals = data.clone()
        elif self.dtype.kind == "c" or dtype.kind == "c":
            from ._complex import cast_values

            vals = cast_values(data, self.dtype, dtype)
        else:
            vals = Kn.cast(data, dtype)
        if self.nnz:  # always: upstream's elemwise-based astype also drops fill values that were stored explicitly
            flags = Kn.flag_not_fill(vals, fill)
            pos, total = Kn.scan_flags(flags)
            if total != self.nnz:
                return COO._from_device(None, Kn.compact(vals, flags, pos, total), self.shape, fill,
                                        keys=Kn.compact(self.sorted_keys(), flags, pos, total))
        out = COO._from_device(self._coords, vals, self.shape, fill,
                               keys=self.sorted_keys() if self._coords is None else self._keys)
        out._idx_vis = self._idx_vis
        return out

    def linear_loc(self):
        return D.download(self.sorted_keys())

    # ---- transpose / reshape (reference: :725-807, :1034-1111) -----------------------------------------
    def transpose(self, axes=None):
        if axes is None:
            axes = tuple(reversed(range(self.ndim)))
        if not isinstance(axes, Iterable) or any(isinstance(a, Iterable) for a in axes):
            raise ValueError(f"axes must be a sequence of integers, got {axes!r}")
        axes = normalize_axis(tuple(axes), self.ndim)
        if len(np.unique(axes)) < len(axes):
            raise ValueError("repeated axis in transpose")
        if not len(axes) == self.ndim:
            raise ValueError("axes don't match array")
        if axes == tuple(range(self.ndim)):
            return self
        return self._cached("transpose", axes,
                            lambda: self._permute_reshape(axes, tuple(self.shape[a] for a in axes)))

    @property
    def T(self):
        return self.transpose(tuple(range(self.ndim))[::-1])

    @property
    def mT(self):
        if self.ndim < 2:
            raise ValueError("Cannot compute matrix transpose if `ndim < 2`.")
        axes = list(range(self.ndim))
        axes[-1], axes[-2] = axes[-2], axes[-1]
        return self.transpose(axes)

    def reshape(self, shape, order="C"):
        shape = tuple(shape) if isinstance(shape, Iterable) else (shape,)
        if order not in {"C", None}:
            raise NotImplementedError("The `order` parameter is not supported")
        shape = tuple(int(s) for s in shape)
        if any(d == -1 for d in shape):
            extra = int(self.size / np.prod([d for d in shape if d != -1]))
            shape = tuple(d if d != -1 else extra for d in shape)
        if self.size != prod(shape):
            raise ValueError(f"cannot reshape array of size {self.size} into shape {shape}")
        if self.shape == shape:
            return self
        return self._cached("reshape", shape, lambda: self._reshape(shape))

    def _reshape(self, shape):
        check_linear_range(shape)
        # linear index is invariant under a C-order reshape: only the coordinates are re-derived
        if self.nnz == 0 and self._data is None:
            return COO(np.zeros((len(shape), 0), dtype=np.intp), self._data_np[:0], shape=shape, has_duplicates=False,
                       sorted=True, fill_value=self.fill_value)
        # only the (lazy) coordinates change; keys and data are shared
        out = COO._from_device(None, self._data_dev(), shape, self.fill_value, keys=self.sorted_keys())
        if self._idx_vis is not None:  # upstream keeps the index dtype, widened when the new extents need it
            out._idx_vis = self._idx_vis if can_store(self._idx_vis, max(shape) if shape else 0) \
                else np.dtype(np.min_scalar_type(max(shape)))
        return out

    def _permute_reshape(self, axes, new_shape):
        """transpose(axes) followed by reshape(new_shape) in one pass: linearise with permuted strides,
        stable sort, unravel (COO rebuild + mergesort of the reference, _coo/core.py:796-803)."""
        coords, data = self._dev()
        perm_shape = tuple(self.shape[a] for a in axes)
        st_perm = c_strides(perm_shape)
        strides = [0] * self.ndim
        for pos, a in enumerate(axes):
            strides[a] = st_perm[pos]
        if self.nnz == 0:
            t = D.torch()
            return COO._from_device(t.zeros((len(new_shape), 0), dtype=coords.dtype, device=coords.device), data,
                                    new_shape, self.fill_value)
        keys = Kn.linearize(coords, strides)
        unsorted, _ = Kn.keys_flags(keys)
        if unsorted:
            keys, perm = Kn.sort_keys(keys, key_bits(self.size))
            data = Kn.gather(data, perm)
        return COO._from_device(None, data, new_shape, self.fill_value, keys=keys)

    def _permuted_keys(self, axes):
        """(sorted linear keys over the permuted shape, matching data) without building coordinates."""
        coords, data = self._dev()
        axes = tuple(axes)
        if axes == tuple(range(self.ndim)):
            return self.sorted_keys(), data
        perm_shape = tuple(self.shape[a] for a in axes)
        st_perm = c_strides(perm_shape)
        strides = [0] * self.ndim
        for pos, a in enumerate(axes):
            strides[a] = st_perm[pos]
        keys = Kn.linearize(coords, strides)
        unsorted, _ = Kn.keys_flags(keys)
        if unsorted:
            keys, perm = Kn.sort_keys(keys, key_bits(self.size))
            data = Kn.gather(data, perm)
        return keys, data

    def broadcast_to(self, shape):
        from ._elemwise import broadcast_to

        return broadcast_to(self, shape)

    # ---- indexing ---------------------------------------------------------------------------------------
    def __getitem__(self, index):
        """Integers, slices (any step), None and Ellipsis -- one streaming kernel over the linear keys
        (_coo/indexing.py:12-133); see _indexing.py."""
        from ._indexing import coo_getitem

        return coo_getitem(self, index)

    def _take_leading(self, i):
        if i < 0:
            i += self.shape[0]
        if not 0 <= i < self.shape[0]:
            raise IndexError("index out of range")
        coords, data = self._dev()
        self.sorted_keys()  # validates / caches the canonical order
        lead = coords[0] if coords[0].is_contiguous() else coords[0].contiguous()
        ip = D.download(Kn.indptr_from_sorted(lead, self.shape[0]))
        lo, hi = int(ip[i]), int(ip[i + 1])
        sub_coords = coords[1:, lo:hi].contiguous()
        return COO._from_device(sub_coords, data[lo:hi].contiguous(), self.shape[1:], self.fill_value)

    # ---- products ---------------------------------------------------------------------------------------
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


def as_coo(x, shape=None, fill_value=None, idx_dtype=None):
    """_coo/common.py:as_coo."""
    from ._gcxs import GCXS

    from ._sparse_array import SparseArray

    if hasattr(x, "shape") and shape is not None:
        raise ValueError("Cannot provide a shape in combination with something that already has a shape.")
    if hasattr(x, "fill_value") and fill_value is not None:
        raise ValueError("Cannot provide a fill-value in combination with something that already has a fill-value.")
    if isinstance(x, COO):
        return x
    if isinstance(x, SparseArray):
        return x.tocoo()
    if _is_scipy_sparse(x):
        return COO.from_scipy_sparse(x)
    if isinstance(x, np.ndarray) or np.isscalar(x):
        if idx_dtype is not None and np.ndim(x) and not can_store(idx_dtype, max(np.shape(x))):
            raise ValueError(f"cannot cast array with shape {np.shape(x)} to dtype {idx_dtype}.")
        return COO.from_numpy(np.asarray(x), fill_value=fill_value, idx_dtype=idx_dtype)
    if isinstance(x, Iterable) and not isinstance(x, (str, bytes)):
        try:
            return COO.from_iter(x, shape=shape, fill_value=fill_value)
        except (ValueError, TypeError, IndexError):
            if isinstance(x, (list, tuple)):
                return COO.from_numpy(np.asarray(x), fill_value=fill_value, idx_dtype=idx_dtype)
            raise
    raise NotImplementedError(f"Format not supported for conversion. Supplied type is {type(x)}, "
                              "see help(sparse.as_coo) for supported formats.")
