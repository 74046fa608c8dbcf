"""tttp(X, factors): a sparse tensor of order 2..8 times a CP model at its stored entries (X * [[U_0, ..., U_{N-1}]]).

Parity with float64 dense `X * einsum(...)` and with the reference's unfused broadcast expression (golden fixture), bit
equality with a CPU restatement of the fixed order of operations (tests/_tensor_order.py) on both column paths with
special values, order 2 against sddmm, the result's pattern and format, the absence of sorts, identities with
mttkrp_mode, edge cases and the `None` factor.  Determinism across calls, factor locations and layouts, index widths and
the shared argument errors are in tests/test_tensor_ops_contract.py.  Every body runs on the NumPy mock without a GPU
and on the CUDA kernels with `-m gpu`."""
import string

import numpy as np
import pytest

import _tensor_order as TO
from _api import dec, sp  # noqa: F401
from _golden import load
from _tensor_cases import (LAYOUTS, SHAPES, dev, entries, full_size_tensor, layout, layout_id, model_dense,
                           rand_tensor)

TOL = {"float32": 2e-5, "float64": 1e-12}
same_bits = TO.same_bits


def positive_zero(z):
    w = {4: np.uint32, 8: np.uint64}[z.dtype.itemsize]
    return np.ascontiguousarray(z).view(w) == 0


def check_exact(sp, got, X, U, dtype):
    """got holds X's entries, in X's stored order, minus those whose z is bitwise +0, with the bits of _tensor_order."""
    dtype = np.dtype(dtype)
    coords, vals = entries(X)
    z = TO.values(coords, vals, U, dtype)
    keep = ~positive_zero(z)
    assert got.format == X.format and got.shape == X.shape and got.dtype == dtype
    assert same_bits(np.asarray(got.fill_value), np.asarray(dtype.type(0)))
    if X.format == "gcxs":
        assert got.compressed_axes == X.compressed_axes
    gc, gv = entries(got)
    assert np.array_equal(gc, coords[:, keep])
    assert same_bits(gv, z[keep])
    return keep


# R = 1, 3 and 37 take the scalar path in both dtypes; 32 and 300 the vector path (300 is ten f32 or 19 f64 r-tiles)
@pytest.mark.parametrize("R", [1, 3, 32, 37, 300])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("order", [2, 3, 4, 5, 6, 8])
@pytest.mark.parametrize("lay", range(len(LAYOUTS)), ids=layout_id)
def test_fp64_parity(sp, lay, order, dtype, R):
    shape = SHAPES[order]
    fmt, ca = LAYOUTS[lay]
    if ca == (0, 1) and order == 2:
        pytest.skip("an order-2 tensor cannot compress two axes")
    rng = np.random.default_rng(100 * order + R)
    X = rand_tensor(sp, rng, shape, max(int(np.prod(shape)) // 4, 5), dtype, fmt,
                    (order - 1,) if ca == "last" else ca)
    U = [rng.random((s, R)).astype(dtype) + np.asarray(0.05, dtype) for s in shape]
    got = sp.tttp(X, U)
    assert got.format == fmt and got.dtype == np.dtype(dtype) and got.nnz == X.nnz
    want = X.todense().astype(np.float64) * model_dense(U)
    np.testing.assert_allclose(got.todense(), want, rtol=TOL[dtype], atol=0)


GOLDEN = [c for c in load("tttp_api") if c["op"] == "tttp"]


@pytest.mark.parametrize("c", GOLDEN, ids=lambda c: f"{c['dtype']}-order{c['order']}-R{c['R']}")
@pytest.mark.parametrize("fmt", ["coo", "gcxs"])
def test_golden_parity(sp, c, fmt):
    X = dec(sp, c, "X_", fmt)
    U = [np.array(c.arr[f"U{m}"]) for m in range(int(c["order"]))]
    got = sp.tttp(X, U)
    w = c.sub("out_")
    want = sp.COO(np.array(w["coords"]), np.array(w["data"]), shape=tuple(int(s) for s in w["shape"])).todense()
    tol = TOL[c["dtype"]]
    assert got.dtype == want.dtype and got.shape == want.shape
    np.testing.assert_allclose(got.todense(), want, rtol=tol, atol=tol)


def special_inputs(sp, rng, shape, nnz, R, dtype):
    """Signed values with stored -0.0; signed factors with +-inf, NaN and -0.0; and mode-0 rows whose products cancel
    exactly (q_{R-2} = -q_{R-1}, every other q_r a signed zero), so m = +0 and z = +-0 on both signs of v."""
    X = rand_tensor(sp, rng, shape, nnz, dtype, signed=True)
    coords, vals = np.asarray(X.coords), np.array(X.data)
    vals[rng.choice(len(vals), max(len(vals) // 20, 1), replace=False)] = -0.0
    X = sp.COO(coords, vals, shape=shape, has_duplicates=False, sorted=True)
    U = [rng.standard_normal((s, R)).astype(dtype) for s in shape]
    cancel = rng.choice(shape[0], max(shape[0] // 3, 1), replace=False)
    if R >= 2:
        for u in U[1:]:
            u[:, R - 1] = u[:, R - 2]
        U[0][cancel, : R - 2] = rng.choice(np.array([0.0, -0.0], dtype), (len(cancel), R - 2))
        U[0][cancel, R - 1] = -U[0][cancel, R - 2]
    else:
        U[0][cancel] = 0.0
    for m, u in enumerate(U):
        flat = u.reshape(-1)
        live = np.flatnonzero(~np.isin(np.arange(u.shape[0]), cancel)) if m == 0 else np.arange(u.shape[0])
        pick = rng.choice(live, min(4, len(live)), replace=False) * R + rng.integers(0, R, min(4, len(live)))
        flat[pick] = [np.inf, -np.inf, np.nan, -0.0][: len(pick)]
    return X, U


# f32 packs hold 4 columns and f64 ones 2: R = 8 and 40 take the vector path in both dtypes, 5 and 37 the scalar path
@pytest.mark.parametrize("R", [1, 5, 8, 37, 40])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_exact_order_both_paths(sp, dtype, R):
    rng = np.random.default_rng(50 + R)
    X, U = special_inputs(sp, rng, (30, 20, 12), 2500, R, dtype)
    for fmt, ca in LAYOUTS:
        Y = layout(X, fmt, ca)
        keep = check_exact(sp, sp.tttp(Y, U), Y, U, dtype)
        _, vals = entries(Y)
        z = TO.values(entries(Y)[0], vals, U, dtype)
        assert (~keep).sum() > 0 and np.signbit(z[~keep]).sum() == 0
        assert (np.signbit(z) & (z == 0)).any()  # stored -0.0 results
        assert np.isnan(z).any()
    # device factors that are column-sliced views (unaligned rows): the scalar path, the same bits
    wide = [dev(sp, np.concatenate([np.zeros((u.shape[0], 1), dtype), u], axis=1))[:, 1:] for u in U]
    mixed = [U[0], wide[1], dev(sp, U[2])]
    want = sp.tttp(X, U)
    for variant in (wide, mixed):
        got = sp.tttp(X, variant)
        assert np.array_equal(got.coords, want.coords) and same_bits(got.data, want.data)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_order2_matches_sddmm(sp, dtype):
    rng = np.random.default_rng(8)
    X = rand_tensor(sp, rng, (60, 45), 900, dtype, signed=True)
    U0, U1 = (rng.random((s, 24)).astype(dtype) + np.asarray(0.05, dtype) for s in X.shape)
    got = sp.tttp(X, [U0, U1])
    want = sp.sddmm(X, U0, U1, b_transposed=True)
    np.testing.assert_allclose(got.todense(), want.todense(), rtol=TOL[dtype], atol=0)
    G = X.asformat("gcxs", compressed_axes=(1,))
    np.testing.assert_allclose(sp.tttp(G, [U0, U1]).todense(), want.todense(), rtol=TOL[dtype], atol=0)


def test_pattern_and_format(sp):
    rng = np.random.default_rng(9)
    X = rand_tensor(sp, rng, (12, 10, 8, 6), 800, "float32", signed=True)
    U = [rng.random((s, 7)).astype(np.float64) + 0.05 for s in X.shape]  # positive model, f64 factors
    for fmt, ca in LAYOUTS:
        Y = layout(X, fmt, ca)
        got = sp.tttp(Y, U)
        assert got.dtype == np.float64 and got.shape == X.shape and got.format == fmt
        assert same_bits(np.asarray(got.fill_value), np.asarray(np.float64(0)))
        assert got.nnz == X.nnz  # a positive model prunes nothing
        if fmt == "gcxs":
            assert got.compressed_axes == Y.compressed_axes
            assert np.array_equal(got.indices, Y.indices) and np.array_equal(got.indptr, Y.indptr)
        check_exact(sp, got, Y, U, np.float64)
    # a negative model corner: the unfused fill value would be -0.0; tttp keeps +0
    Un = [-u for u in U[:1]] + U[1:]
    got = sp.tttp(X, Un)
    assert not np.signbit(got.fill_value)
    assert got.nnz == X.nnz and np.all(got.todense() * X.todense() <= 0)
    # a model that is zero on some mode-1 slices prunes those entries with v >= 0 (v < 0 gives a stored -0.0)
    Uz = [u.copy() for u in U]
    Uz[1][::2] = 0.0
    for fmt, ca in LAYOUTS:
        Y = layout(X, fmt, ca)
        got = sp.tttp(Y, Uz)
        c, v = entries(Y)
        assert got.nnz == int(((c[1] % 2 == 1) | np.signbit(v)).sum()) < X.nnz
        check_exact(sp, got, Y, Uz, np.float64)


def test_gcxs_with_repeated_indices(sp):
    """A GCXS built by hand whose rows repeat an index: one product per stored entry, in stored order."""
    data = np.array([1.5, -2.0, 3.0, 0.5, 4.0])
    indices = np.array([2, 2, 0, 1, 1])
    indptr = np.array([0, 3, 3, 5])
    G = sp.GCXS((data, indices, indptr), shape=(3, 4), compressed_axes=(0,))
    rng = np.random.default_rng(12)
    U = [rng.random((3, 5)), rng.random((4, 5))]
    got = sp.tttp(G, U)
    assert got.nnz == 5 and np.array_equal(got.indices, indices) and np.array_equal(got.indptr, indptr)
    check_exact(sp, got, G, U, np.float64)


def test_no_sort(sp, monkeypatch):
    rng = np.random.default_rng(13)
    X = rand_tensor(sp, rng, (25, 18, 9), 1200, "float64", signed=True)
    Ys = [layout(X, fmt, ca) for fmt, ca in LAYOUTS]
    U = [rng.standard_normal((s, 6)) for s in X.shape]

    def no_sort(*a, **k):
        raise AssertionError("tttp sorted the entries")

    monkeypatch.setattr(sp._kernels, "sort_keys", no_sort)
    for Y in Ys:
        check_exact(sp, sp.tttp(Y, U), Y, U, np.float64)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_identities_with_mttkrp_mode(sp, dtype):
    rng = np.random.default_rng(15)
    X = rand_tensor(sp, rng, (20, 16, 12, 6), 1500, dtype, signed=True)
    U = [rng.standard_normal((s, 5)).astype(dtype) for s in X.shape]
    fit = float(sp.tttp(X, U).sum())
    for n in range(X.ndim):
        other = float((U[n].astype(np.float64) * sp.mttkrp_mode(X, U, n)).sum())
        assert fit == pytest.approx(other, rel=50 * TOL[dtype])
    # completion gradient: mttkrp_mode(tttp(P, U) - X, U, n) with P X's pattern with ones
    P = sp.COO(X.coords, np.ones(X.nnz, dtype), shape=X.shape, has_duplicates=False, sorted=True)
    resid = sp.tttp(P, U) - X
    mask = X.todense() != 0
    dres = mask * model_dense(U) - X.todense().astype(np.float64)
    lo = string.ascii_lowercase[:X.ndim]
    for n in range(X.ndim):
        others = [m for m in range(X.ndim) if m != n]
        want = np.einsum(",".join([lo] + [lo[m] + "z" for m in others]) + "->" + lo[n] + "z", dres,
                         *[U[m].astype(np.float64) for m in others])
        got = sp.mttkrp_mode(resid, U, n)
        np.testing.assert_allclose(got, want, rtol=100 * TOL[dtype], atol=100 * TOL[dtype] * np.abs(want).max())


def test_edge_cases(sp):
    rng = np.random.default_rng(16)
    U = [rng.random((s, 3)) for s in (5, 6, 7)]
    empty = sp.COO(np.zeros((3, 0), np.int64), np.zeros(0), shape=(5, 6, 7))
    for fmt, ca in LAYOUTS:
        got = sp.tttp(layout(empty, fmt, ca), U)
        assert got.nnz == 0 and got.shape == (5, 6, 7) and got.format == fmt
    X = rand_tensor(sp, rng, (5, 6, 7), 60, "float64", signed=True)
    vals = np.array(X.data)
    vals[:3] = [np.inf, -0.0, np.nan]
    X = sp.COO(X.coords, vals, shape=X.shape, has_duplicates=False, sorted=True)
    U0 = [np.zeros((s, 0)) for s in X.shape]
    for fmt, ca in LAYOUTS:
        Y = layout(X, fmt, ca)
        got = sp.tttp(Y, U0)  # R = 0: z = v * +0, stored where that is -0.0 or NaN
        check_exact(sp, got, Y, U0, np.float64)
        assert got.nnz == int(np.signbit(vals).sum() + np.isnan(vals).sum() + np.isinf(vals).sum() - np.isneginf(vals).sum())
    zero_ext = sp.COO(np.zeros((3, 0), np.int64), np.zeros(0), shape=(5, 0, 7))
    got = sp.tttp(zero_ext, [np.ones((5, 2)), np.ones((0, 2)), np.ones((7, 2))])
    assert got.shape == (5, 0, 7) and got.nnz == 0
    one = sp.COO(np.array([[4], [5], [6]]), np.array([2.0]), shape=(5, 6, 7))
    for fmt, ca in LAYOUTS:
        got = sp.tttp(layout(one, fmt, ca), U)
        assert got.nnz == 1
        assert same_bits(got.data, TO.values([[4], [5], [6]], [2.0], U, np.float64))


def test_errors(sp):
    rng = np.random.default_rng(17)
    X = rand_tensor(sp, rng, (5, 6, 7), 40, "float64")
    U = [rng.random((s, 3)) for s in X.shape]
    with pytest.raises(ValueError, match="None"):
        sp.tttp(X, [None, U[1], U[2]])


@pytest.mark.gpu
def test_full_size():
    """(1e6, 1e6, 100) with 1e8 uniform entries, R = 32, f32: every entry within 2e-5 of a float64 restatement on the
    device, and 10,000 sampled entries bit-equal to the CPU restatement of the order."""
    import torch

    import sparse_b200 as spm

    X, coords, vals, g = full_size_tensor(79, signed=True)  # no zero value: nothing is pruned
    R = 32
    U = [torch.rand((s, R), generator=g, device=coords.device) + 0.05 for s in X.shape]
    got = spm.tttp(X, U)
    assert got.nnz == coords.shape[1]
    gv = got._data_dev()
    step = 10_000_000
    for s in range(0, coords.shape[1], step):
        c = coords[:, s:s + step]
        m = (U[0][c[0]].double() * U[1][c[1]].double() * U[2][c[2]].double()).sum(1)
        want = vals[s:s + step].double() * m
        assert torch.allclose(gv[s:s + step].double(), want, rtol=2e-5, atol=0), s
    rng = np.random.default_rng(6)
    pick = torch.from_numpy(np.sort(rng.choice(coords.shape[1], 10_000, replace=False))).to(coords.device)
    c = coords[:, pick].cpu().numpy()
    want = TO.values(c, vals[pick].cpu().numpy(), [u.cpu().numpy() for u in U], np.float32)
    assert same_bits(gv[pick].cpu().numpy(), want)
