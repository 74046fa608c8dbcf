"""masked_matmul(mask, a, b): the value of mask * (a @ b) at mask's stored positions, for sparse a and b.

Parity with the reference's unfused expression (golden fixture, restricted to the mask's pattern, and in full where
a @ b is non-negative and finite), bit equality with the package's own unfused expression across dtypes, layouts,
special values, long and hub rows, the segment path and the int64 index path, the unsorted-row rule, the triangle count
against SciPy, determinism and errors.  Every body runs on the NumPy mock without a GPU and on the CUDA kernels with
`-m gpu`."""
import itertools

import numpy as np
import pytest
import scipy.sparse as ss

from _api import dec, sp  # noqa: F401
from _golden import load

LAYOUTS = [("coo", None), ("gcxs", (0,)), ("gcxs", (1,))]


def fmt(x, layout):
    kind, ca = LAYOUTS[layout] if isinstance(layout, int) else layout
    return x if kind == "coo" else x.asformat("gcxs", compressed_axes=ca)


def coo_parts(x):
    c = x.tocoo() if x.format == "gcxs" else x
    return np.asarray(c.coords), np.asarray(c.data)


def same(x, y):
    """Equal bit for bit, except that any NaN matches any NaN (the sign and payload of a NaN produced by an invalid
    operation differ between the host CPU and the GPU)."""
    x, y = np.asarray(x), np.asarray(y)
    if x.shape != y.shape or x.dtype != y.dtype:
        return False
    if x.dtype.kind != "f":
        return np.array_equal(x, y)
    nan = np.isnan(x) & np.isnan(y)
    return np.array_equal(x[~nan].view(np.uint8), y[~nan].view(np.uint8)) and np.array_equal(np.isnan(x), np.isnan(y))


def restrict(coords, data, mask_coords, shape):
    """The entries of (coords, data) at positions stored in the mask."""
    keys = np.ravel_multi_index(tuple(coords), shape) if coords.shape[1] else np.zeros(0, np.int64)
    mkeys = np.ravel_multi_index(tuple(mask_coords), shape) if mask_coords.shape[1] else np.zeros(0, np.int64)
    keep = np.isin(keys, mkeys)
    return coords[:, keep], data[keep]


def check_against(got, want_coords, want_data):
    gc, gd = coo_parts(got)
    assert np.array_equal(gc, want_coords), "coordinates differ"
    assert gd.dtype == want_data.dtype, (gd.dtype, want_data.dtype)
    assert same(gd, want_data), "values differ"


def check_unfused(sp, mask, a, b):
    """masked_matmul equals the package's own unfused mask * (a @ b) restricted to mask's pattern; returns it."""
    got = sp.masked_matmul(mask, a, b)
    assert got.format == mask.format
    if mask.format == "gcxs":
        assert got.compressed_axes == mask.compressed_axes
    ref = mask * (a @ b)
    rc, rd = coo_parts(ref)
    mc, _ = coo_parts(mask)
    check_against(got, *restrict(rc, rd, mc, mask.shape))
    return got, ref


def rand(sp, rng, shape, nnz, dtype, signed=True):
    size = int(np.prod(shape))
    lin = np.sort(rng.choice(size, size=min(nnz, size), replace=False)) if size else np.zeros(0, np.int64)
    coords = np.stack(np.unravel_index(lin, shape)).astype(np.int64)
    if np.dtype(dtype).kind == "f":
        vals = rng.random(len(lin)) + 0.25
        if signed:
            vals = vals * rng.choice([-1.0, 1.0], len(lin))
    else:
        vals = rng.integers(1, 6, len(lin)) * (rng.choice([-1, 1], len(lin)) if signed else 1)
    return sp.COO(coords, vals.astype(dtype), shape=shape, has_duplicates=False, sorted=True)


def from_scipy(sp, m, dtype):
    m = ss.coo_matrix(m)
    m.sum_duplicates()
    order = np.lexsort((m.col, m.row))
    coords = np.stack([m.row[order], m.col[order]]).astype(np.int64)
    return sp.COO(coords, m.data[order].astype(dtype), shape=m.shape, has_duplicates=False, sorted=True)


# ---- golden fixture: the reference's unfused expression ----------------------------------------------------------
GOLDEN = load("masked_matmul_api")


@pytest.mark.parametrize("c", GOLDEN, ids=lambda c: f"{c['op']}-{c['dtype']}-{'x'.join(map(str, c['shape']))}"
                                                    f"{'-special' if c['special'] else ''}")
def test_golden_parity(sp, c):
    base = [dec(sp, c, p) for p in ("mask_", "a_", "b_")]
    w = c.sub("out_")
    shape = tuple(int(s) for s in w["shape"])
    want_c, want_d = np.asarray(w["coords"]), np.asarray(w["data"])
    in_c, in_d = restrict(want_c, want_d, np.asarray(c.arr["mask_coords"]), shape)
    for lm, la, lb in itertools.product(range(3), repeat=3):
        mask, a, b = fmt(base[0], lm), fmt(base[1], la), fmt(base[2], lb)
        got = sp.masked_matmul(mask, a, b)
        assert got.format == mask.format and got.shape == shape
        if mask.format == "gcxs":
            assert got.compressed_axes == mask.compressed_axes
        check_against(got, in_c, in_d)
        if c["full_equal"]:
            check_against(got, want_c, want_d)
    if c["op"] == "triangles":
        assert float(sp.masked_matmul(*base).sum()) / 6 == c["triangles"]


def test_golden_has_outside_entries():
    """The special-value cases do store entries outside the mask in the unfused result (-0.0 / NaN), so the
    restriction above is what makes the fused and unfused results comparable there."""
    n_out = 0
    for c in GOLDEN:
        w = c.sub("out_")
        shape = tuple(int(s) for s in w["shape"])
        n_out += w["data"].shape[0] - restrict(np.asarray(w["coords"]), w["data"], c.arr["mask_coords"], shape)[1].size
    assert n_out > 0


# ---- host logic ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dts", [("float32", "float32", "float32"), ("int32", "float32", "float32"),
                                 ("float32", "int32", "int64"), ("int64", "int32", "int32"),
                                 ("int32", "int32", "int32"), ("float64", "float32", "int64"),
                                 ("float32", "float32", "float64"), ("int64", "int64", "float32")])
def test_dtype_promotion(sp, dts):
    rng = np.random.default_rng(7)
    mask, a, b = rand(sp, rng, (20, 25), 150, dts[0]), rand(sp, rng, (20, 18), 120, dts[1]), \
        rand(sp, rng, (18, 25), 140, dts[2])
    got, _ = check_unfused(sp, mask, a, b)
    assert got.dtype == np.result_type(dts[0], np.result_type(dts[1], dts[2]))


@pytest.mark.parametrize("layouts", list(itertools.product(range(3), repeat=3)))
def test_layouts_match_unfused(sp, layouts):
    rng = np.random.default_rng(11)
    mask, a, b = rand(sp, rng, (30, 35), 300, "float64"), rand(sp, rng, (30, 40), 400, "float64"), \
        rand(sp, rng, (40, 35), 420, "float64")
    check_unfused(sp, *(fmt(x, lay) for x, lay in zip((mask, a, b), layouts)))


@pytest.mark.parametrize("bad", ["float16", "complex128", "bool", "int16", "uint32"])
def test_dtype_errors(sp, bad):
    """Both result_type(a, b) and result_type(mask, result_type(a, b)) must be float32, float64, int32 or int64."""
    odd = sp.COO.from_numpy((np.eye(4) * 2).astype(bad))
    with pytest.raises(TypeError, match="float32, float64, int32, int64"):
        sp.masked_matmul(odd, odd, odd)
    f32 = sp.COO.from_numpy(np.eye(4, dtype=np.float32))
    if bad == "complex128":
        with pytest.raises(TypeError, match="float32, float64, int32, int64"):
            sp.masked_matmul(odd, f32, f32)  # the product is float32, the masked result complex
    if bad == "bool":
        got = sp.masked_matmul(odd, f32, f32)  # a boolean mask promotes into the matrix
        assert got.dtype == np.float32


def test_shape_and_type_errors(sp):
    rng = np.random.default_rng(4)
    m, a, b = rand(sp, rng, (5, 6), 8, "float64"), rand(sp, rng, (5, 7), 8, "float64"), \
        rand(sp, rng, (7, 6), 8, "float64")
    with pytest.raises(ValueError):
        sp.masked_matmul(m, a, rand(sp, rng, (6, 6), 8, "float64"))
    with pytest.raises(ValueError):
        sp.masked_matmul(rand(sp, rng, (5, 5), 8, "float64"), a, b)
    with pytest.raises(ValueError):
        sp.masked_matmul(m, rand(sp, rng, (4, 7), 8, "float64"), b)
    with pytest.raises(TypeError):
        sp.masked_matmul(m.todense(), a, b)
    with pytest.raises(TypeError):
        sp.masked_matmul(m, a, b.todense())
    with pytest.raises(TypeError):
        sp.masked_matmul(m, rand(sp, rng, (5, 7, 2), 8, "float64"), b)
    with pytest.raises(ValueError):
        sp.masked_matmul(m, sp.COO.from_numpy(np.ones((5, 7)), fill_value=1.0), b)


def test_empty_cases(sp):
    rng = np.random.default_rng(5)
    for M, K, N, nm in ((6, 0, 7, 12), (6, 5, 7, 0), (0, 5, 7, 0), (6, 5, 0, 0)):
        mask = rand(sp, rng, (M, N), nm, "float64")
        a, b = rand(sp, rng, (M, K), 10, "float64"), rand(sp, rng, (K, N), 10, "float64")
        for lm in range(3):
            got, _ = check_unfused(sp, fmt(mask, lm), a, b)
            if K == 0:
                # every c' is +0: only the negative mask values survive, as -0.0
                d = coo_parts(got)[1]
                assert np.all(np.signbit(d)) and np.all(d == 0)


def test_unsorted_rows_follow_unfused(sp):
    """A GCXS built by hand with an unsorted row: the call is computed as the unfused expression restricted to the
    mask, so it follows the stored order of the unfused product."""
    big = np.float32(1e8)
    # row 0 of a: k = 2, 0, 1 with values 1, 1e8, -1e8 -- stored order sums to 0, ascending k to 1
    a = sp.GCXS((np.array([1, big, -big, 1], np.float32), np.array([2, 0, 1, 0]), np.array([0, 3, 4])),
                shape=(2, 3), compressed_axes=(0,))
    b = sp.COO.from_numpy(np.ones((3, 2), np.float32))
    mask = sp.COO.from_numpy(np.ones((2, 2), np.float32))
    got, ref = check_unfused(sp, mask, a, b)
    # the canonical order (ascending k) gives a different value, so the rule is observable
    canon = sp.masked_matmul(mask, a.tocoo(), b)
    assert coo_parts(canon)[1].shape != coo_parts(got)[1].shape or not same(coo_parts(canon)[1], coo_parts(got)[1])
    bt = sp.GCXS((np.array([1, 1, 1, 1, 1, 1], np.float32), np.array([2, 0, 1, 0, 1, 2]), np.array([0, 3, 6])),
                 shape=(3, 2), compressed_axes=(1,))  # b by columns, column 0 unsorted
    check_unfused(sp, mask, a.tocoo(), bt)


def test_repeated_calls_identical(sp):
    rng = np.random.default_rng(9)
    mask, a, b = rand(sp, rng, (60, 70), 900, "float32"), rand(sp, rng, (60, 50), 800, "float32"), \
        rand(sp, rng, (50, 70), 900, "float32")
    first = sp.masked_matmul(mask, a, b)
    for _ in range(3):
        again = sp.masked_matmul(mask, a, b)
        assert np.array_equal(coo_parts(first)[0], coo_parts(again)[0])
        assert same(coo_parts(first)[1], coo_parts(again)[1])


# ---- kernel paths: long rows, segments, hubs, power law, int64 indices ------------------------------------------
def skewed(sp, rng, n, nnz, dtype, alpha=1.3):
    """Power-law rows and columns (Zipf-like degrees)."""
    w = 1.0 / np.arange(1, n + 1) ** (alpha / 2)
    p = w / w.sum()
    r, c = rng.choice(n, nnz, p=p), rng.choice(n, nnz, p=p)
    m = ss.coo_matrix((rng.random(nnz) + 0.1, (rng.permutation(n)[r], c)), shape=(n, n))
    return from_scipy(sp, m, dtype)


@pytest.mark.parametrize("dtype", ["float32", "float64", "int64"])
def test_power_law_rows(sp, dtype):
    rng = np.random.default_rng(21)
    a = skewed(sp, rng, 600, 9000, dtype)
    check_unfused(sp, a, a, a)
    check_unfused(sp, fmt(a, 1), fmt(a, 1), fmt(a, 2))


def test_hub_columns(sp):
    """A few dense columns of b (long B^T rows) against short rows of a: the kernel searches B^T_j instead."""
    rng = np.random.default_rng(22)
    M, K, N = 300, 4000, 50
    a = rand(sp, rng, (M, K), 1500, "float64")
    bd = np.zeros((K, N))
    bd[:, :3] = rng.random((K, 3)) - 0.5
    bd[rng.random((K, N)) < 0.01] = 1.0
    b = sp.COO.from_numpy(bd)
    mask = rand(sp, rng, (M, N), 3000, "float64")
    for lb in range(3):
        check_unfused(sp, mask, a, fmt(b, lb))


@pytest.mark.parametrize("cap", [1, 3, 17])
def test_forced_segments(sp, cap):
    """Rows of a longer than the staging capacity are processed in ascending-k segments; the running sums carry over."""
    rng = np.random.default_rng(30 + cap)
    M, K, N = 40, 300, 45
    a = rand(sp, rng, (M, K), 6000, "float32")
    b = rand(sp, rng, (K, N), 5000, "float32")
    mask = rand(sp, rng, (M, N), 900, "float32")
    plain = sp.masked_matmul(mask, a, b)
    sp._kernels.masked_spgemm_set_stage(cap)
    try:
        for lm in range(3):
            got, _ = check_unfused(sp, fmt(mask, lm), a, b)
        seg = sp.masked_matmul(mask, a, b)
    finally:
        sp._kernels.masked_spgemm_set_stage(0)
    assert np.array_equal(coo_parts(seg)[0], coo_parts(plain)[0]) and same(coo_parts(seg)[1], coo_parts(plain)[1])


def test_forced_int64_index(sp, monkeypatch):
    from sparse_b200 import _fused

    rng = np.random.default_rng(31)
    mask, a, b = rand(sp, rng, (50, 60), 700, "float64"), rand(sp, rng, (50, 40), 600, "float64"), \
        rand(sp, rng, (40, 60), 700, "float64")
    narrow = sp.masked_matmul(mask, a, b)
    monkeypatch.setattr(_fused, "_FORCE_WIDE_INDEX_MASKED", True)
    for lm in range(3):
        check_unfused(sp, fmt(mask, lm), fmt(a, lm), fmt(b, 2 - lm))
    wide = sp.masked_matmul(mask, a, b)
    assert same(coo_parts(wide)[1], coo_parts(narrow)[1])


def test_special_values_and_empty_intersections(sp):
    rng = np.random.default_rng(33)
    M, K, N = 25, 30, 28
    ad = np.where(rng.random((M, K)) < 0.2, rng.random((M, K)) - 0.5, 0)
    bd = np.where(rng.random((K, N)) < 0.2, rng.random((K, N)) - 0.5, 0)
    ad[0, :5] = [np.inf, -np.inf, np.nan, 2.0, -3.0]
    bd[:5, 1] = [1.0, 1.0, 1.0, np.inf, -0.0]
    bd[10:, 2] = 0  # column 2 meets rows of a that are zero there: empty intersections
    md = np.where(rng.random((M, N)) < 0.4, rng.random((M, N)) - 0.5, 0)
    md[0, :4] = [-0.0, np.nan, -1.0, np.inf]
    a, b, mask = (sp.COO.from_numpy(x) for x in (ad, bd, md))
    mask = sp.COO(mask.coords, np.where(mask.coords[1] == 0, -0.0, mask.data), shape=mask.shape,
                  has_duplicates=False, sorted=True)
    for lm, la, lb in itertools.product(range(3), repeat=3):
        check_unfused(sp, fmt(mask, lm), fmt(a, la), fmt(b, lb))


def test_full_equality_non_negative(sp):
    rng = np.random.default_rng(34)
    mask, a, b = rand(sp, rng, (40, 45), 500, "float64", signed=False), \
        rand(sp, rng, (40, 30), 400, "float64", signed=False), rand(sp, rng, (30, 45), 400, "float64", signed=False)
    got, ref = check_unfused(sp, mask, a, b)
    rc, rd = coo_parts(ref)
    check_against(got, rc, rd)


def test_triangle_count_matches_scipy(sp):
    rng = np.random.default_rng(35)
    n = 3000
    u = ss.triu(ss.random(n, n, density=4e-3, random_state=rng, format="csr"), 1)
    adj = ((u + u.T) > 0).astype(np.float64)
    want = (adj @ adj).multiply(adj).sum() / 6
    A = from_scipy(sp, adj, "float64")
    got = float(sp.masked_matmul(A, A, A).sum()) / 6
    assert got == want and want > 0
    G = fmt(A, 1)
    assert float(sp.masked_matmul(G, G, G.T).sum()) / 6 == want
