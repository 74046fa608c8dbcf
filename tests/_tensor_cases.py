"""Inputs and small helpers shared by the tests of the sparse-tensor ops (mttkrp_mode, ttmc_mode, tttp, ttm_mode and
cp_completion_mode): shapes and storage layouts, random and chunk-structured tensors, the float64 einsum references and
the full-size GPU tensor.  Each op's test file picks the orders and layouts it runs; nothing here is parametrised."""
import string

import numpy as np

# orders 2..8, small extents so the dense einsum stays small
SHAPES = {2: (37, 29), 3: (23, 17, 11), 4: (9, 7, 6, 5), 5: (6, 5, 4, 3, 5), 6: (4, 3, 3, 2, 3, 2),
          7: (3, 2, 3, 2, 2, 3, 2), 8: (3, 2, 3, 2, 2, 3, 2, 2)}
# (format, compressed axes); "last" is the tensor's last axis
LAYOUTS = [("coo", None), ("gcxs", (0,)), ("gcxs", "last"), ("gcxs", (0, 1))]


def layout_id(i):
    return LAYOUTS[i][0] + str(LAYOUTS[i][1] or "")


def layout(X, fmt, ca):
    """X in storage layout (fmt, ca) of LAYOUTS."""
    if fmt == "coo":
        return X
    return X.asformat("gcxs", compressed_axes=(X.ndim - 1,) if ca == "last" else ca)


def chunk(sp):
    return sp._kernels.mttkrp_mode_chunk()


def dev(sp, a):
    return sp._device.upload(np.asarray(a))


def host(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def rand_tensor(sp, rng, shape, nnz, dtype, fmt="coo", ca=None, signed=False):
    size = int(np.prod(shape))
    lin = np.sort(rng.choice(size, size=min(nnz, size), replace=False))
    coords = np.stack(np.unravel_index(lin, shape)).astype(np.int64)
    vals = rng.random(len(lin)) + 0.1
    if signed:
        vals = vals * rng.choice([-1.0, 1.0], len(lin))
    X = sp.COO(coords, vals.astype(dtype), shape=shape, has_duplicates=False, sorted=True)
    return X if fmt == "coo" else X.asformat("gcxs", compressed_axes=ca)


def entries(X):
    """(coordinates N x nnz, values) of X's entries in its stored order."""
    if X.format == "coo":
        return np.asarray(X.coords, np.int64), np.asarray(X.data)
    ca = list(X.compressed_axes)
    order = ca + [a for a in range(X.ndim) if a not in ca]
    rs = [X.shape[a] for a in order]
    rows = np.repeat(np.arange(len(X.indptr) - 1), np.diff(X.indptr))
    parts = list(np.unravel_index(rows, rs[:len(ca)])) + list(np.unravel_index(X.indices, rs[len(ca):]))
    coords = np.zeros((X.ndim, X.nnz), np.int64)
    for pos, a in enumerate(order):
        coords[a] = parts[pos]
    return coords, np.asarray(X.data)


def plant_specials(rng, U):
    """Put +inf, -inf, NaN and -0.0 at random places of each factor (in place); returns U."""
    for u in U:
        flat = u.reshape(-1)
        k = min(4, flat.size)
        flat[rng.choice(flat.size, k, replace=False)] = [np.inf, -np.inf, np.nan, -0.0][:k]
    return U


def chunk_structured(sp, rng, dtype, R):
    """Order-3 tensor whose mode-0 slices are: inside one chunk, empty, crossing one chunk boundary, and one slice of
    more than 3 chunks that starts and ends mid-chunk; stored -0.0 values and +-inf / NaN in the factors."""
    ch = chunk(sp)
    lengths = [5, 0, 17, ch - 30, 60, 0, 3 * ch + 77, 9, 0, 2, ch // 2 + 3, 1, 40]
    J, K = 48, max(48, -(-(3 * ch + 77) // 48))
    coords, vals = [], []
    for i, L in enumerate(lengths):
        lin = np.sort(rng.choice(J * K, size=L, replace=False))
        coords.append(np.stack([np.full(L, i), lin // K, lin % K]))
        vals.append(rng.standard_normal(L))
    coords = np.concatenate(coords, axis=1).astype(np.int64)
    vals = np.concatenate(vals).astype(dtype)
    vals[rng.choice(len(vals), 25, replace=False)] = -0.0
    X = sp.COO(coords, vals, shape=(len(lengths), J, K), has_duplicates=False, sorted=True)
    U = [rng.standard_normal((s, R)).astype(dtype) for s in X.shape]
    return X, plant_specials(rng, U)


def edge_rows(sp, rng, dtype, R):
    """Order-3 tensor whose mode-0 rows have 511, 512 and 513 entries around the chunk edges, short rows between them,
    two empty rows, stored -0.0, +-inf and NaN values in a few rows."""
    ch = chunk(sp)
    lengths = [3, ch - 1, ch, 0, ch + 1, 7, 1, ch - 3, 0, 2 * ch, 40]
    J, K = 40, 60
    coords, vals = [], []
    for i, L in enumerate(lengths):
        lin = np.sort(rng.choice(J * K, size=L, replace=False))
        coords.append(np.stack([np.full(L, i), lin // K, lin % K]))
        vals.append(rng.standard_normal(L))
    coords = np.concatenate(coords, axis=1).astype(np.int64)
    vals = np.concatenate(vals).astype(dtype)
    vals[rng.choice(len(vals), 25, replace=False)] = -0.0
    vals[[2, 100]] = [np.inf, np.nan]  # row 0 becomes non-finite, row 1 NaN
    X = sp.COO(coords, vals, shape=(len(lengths), J, K), has_duplicates=False, sorted=True)
    U = [rng.standard_normal((s, R)).astype(dtype) for s in X.shape]
    return X, U


def mttkrp_einsum(X, factors, mode):
    """float64 mttkrp_mode: einsum over every mode but `mode` of X and the other modes' factors, (I_mode, R)."""
    N = X.ndim
    letters = string.ascii_lowercase[:N]
    terms = [letters] + [letters[m] + "z" for m in range(N) if m != mode]
    ops = [X.todense().astype(np.float64)] + [np.asarray(factors[m], np.float64) for m in range(N) if m != mode]
    return np.einsum(",".join(terms) + "->" + letters[mode] + "z", *ops)


def ttmc_einsum(X, U, mode):
    """float64 ttmc_mode: einsum with output subscripts "i" + "abc...", flattened to (I_mode, W)."""
    N = X.ndim
    lo, hi = string.ascii_lowercase[:N], string.ascii_uppercase[:N]
    others = [m for m in range(N) if m != mode]
    terms = [lo] + [lo[m] + hi[m] for m in others]
    ops = [X.todense().astype(np.float64)] + [np.asarray(U[m], np.float64) for m in others]
    out = np.einsum(",".join(terms) + "->" + lo[mode] + "".join(hi[m] for m in others), *ops)
    return out.reshape(X.shape[mode], -1)


def model_dense(U):
    """float64 CP model [[U_0, ..., U_{N-1}]] as a dense array."""
    N = len(U)
    lo = string.ascii_lowercase[:N]
    return np.einsum(",".join(c + "z" for c in lo) + "->" + lo, *[np.asarray(u, np.float64) for u in U])


FULL_SHAPE = (1_000_000, 1_000_000, 100)


def full_size_tensor(seed, signed=False):
    """The full-size GPU workload: FULL_SHAPE with 1e8 uniform positions drawn (duplicates merged), values in
    [0.1, 1.1), with a random sign each when `signed` (so no value is zero).  Returns (X, coords, vals, generator); the
    generator continues for the caller's factors."""
    import torch

    import sparse_b200 as spm

    devc = torch.device("cuda")
    shape = FULL_SHAPE
    g = torch.Generator(device=devc).manual_seed(seed)
    lin = torch.unique(torch.randint(0, shape[0] * shape[1] * shape[2], (100_000_000,), generator=g, device=devc))
    coords = torch.stack(torch.unravel_index(lin, shape))
    del lin
    if signed:
        sign = torch.randint(0, 2, (coords.shape[1],), generator=g, device=devc) * 2 - 1
        vals = (torch.rand(coords.shape[1], generator=g, device=devc) + 0.1) * sign
        del sign
    else:
        vals = torch.rand(coords.shape[1], generator=g, device=devc) + 0.1
    X = spm.COO(coords, vals, shape=shape, has_duplicates=False, sorted=True)
    return X, coords, vals, g
