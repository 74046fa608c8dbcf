"""sptc(X, Y, axes): sparse x sparse tensor contraction with a sparse COO result, on compressed rows.

Bit identity with ``tensordot(X, Y, axes, return_type=COO)`` wherever tensordot fits (orders 1..8, one to all-but-one
contracted axes, axes paired out of order, negative and integer axes, X is Y, GCXS operands, narrow integers), golden
parity with the reference's own tensordot (tests/golden/sptc_api.npz), special values and the sentinel row, shapes far
beyond tensordot's size limit against a CPU restatement of the contract (tests/_sptc_order.py), both index widths, the
cached compressed rows, K4's row paths through compressed rows, the join kernel alone, edge cases, errors and the argument
checks of the two C entry points.  The cases are `check_*` functions; the two tests at the end run them in turn, one
over the values (against tensordot and the reference) and one over the compressed rows, the kernels and the errors, and
name the case in a note when one fails.  Both run on the NumPy mock without a GPU (the two new wrappers' stand-ins are
tests/_mock_sptc.py, installed by a fixture here) and on the CUDA kernels with `-m gpu`."""
import itertools

import numpy as np
import pytest

import _mock_sptc
import _sptc_order as SO
from _api import dec, sp  # noqa: F401
from _golden import load
from _tensor_cases import SHAPES, dev, host, rand_tensor

same_bits = SO.same_bits


@pytest.fixture(autouse=True)
def _mock_stand_ins(request):
    """On the NumPy mock backend, the stand-ins of tests/_mock_sptc.py in place of the real wrappers."""
    if "sp" not in request.fixturenames:
        yield
        return
    sp = request.getfixturevalue("sp")
    if not sp._device._TEST_CPU:
        yield
        return
    real = {name: getattr(sp._kernels, name) for name in _mock_sptc.STAND_INS}
    for name, fn in _mock_sptc.STAND_INS.items():
        setattr(sp._kernels, name, fn)
    yield
    for name, fn in real.items():
        setattr(sp._kernels, name, fn)


def assert_same(got, want):
    """Same canonical COO: shape, dtype, fill value, coordinates and values bit for bit."""
    assert got.format == "coo" and want.format == "coo"
    assert got.shape == want.shape and got.dtype == want.dtype
    assert same_bits(np.asarray(got.fill_value), np.asarray(want.fill_value))
    assert np.array_equal(np.asarray(got.coords, np.int64), np.asarray(want.coords, np.int64))
    assert same_bits(got.data, want.data)


def coo_of(X):
    return X.tocoo() if X.format == "gcxs" else X


def assert_order(sp, got, X, Y, axes):
    """got equals the CPU restatement of the contract on the stored entries."""
    ax, ay = axes
    X, Y = coo_of(X), coo_of(Y)
    keys, vals = SO.result(X.coords, X.data, X.shape, Y.coords, Y.data, Y.shape, ax, ay, got.dtype)
    assert got.format == "coo" and same_bits(np.asarray(got.fill_value), np.asarray(got.dtype.type(0)))
    assert np.array_equal(host(got.sorted_keys()), keys)
    assert same_bits(got.data, vals)


def pair(sp, rng, order, ncon, dtype, perm=True):
    """X of SHAPES[order] and a Y that shares `ncon` of its axes, in shuffled positions, plus two free axes."""
    xs = SHAPES[order]
    ax = [int(a) for a in rng.choice(order, ncon, replace=False)] if perm else list(range(order - ncon, order))
    free = [4, 3][: 8 - ncon]  # Y stays within order 8
    slots = [("c", k) for k in range(ncon)] + [("f", k) for k in range(len(free))]
    if perm:
        slots = [slots[i] for i in rng.permutation(len(slots))]
    ys = tuple(xs[ax[k]] if kind == "c" else free[k] for kind, k in slots)
    ay = [slots.index(("c", k)) for k in range(ncon)]
    ints = np.dtype(dtype).kind == "i"
    X = rand_tensor(sp, rng, xs, max(int(np.prod(xs)) // 3, 5), "float64", signed=True)
    Y = rand_tensor(sp, rng, ys, max(int(np.prod(ys)) // 2, 5), "float64", signed=True)
    if ints:
        X, Y = (X * 10).astype(dtype), (Y * 10).astype(dtype)
    else:
        X, Y = X.astype(dtype), Y.astype(dtype)
    return X, Y, (ax, ay)


def check_tensordot_bit_identity(sp, order, dtype):
    rng = np.random.default_rng(7 * order)
    for ncon in sorted({1, min(2, order - 1), order - 1}):
        X, Y, axes = pair(sp, rng, order, ncon, dtype)
        got = sp.sptc(X, Y, axes)
        assert_same(got, sp.tensordot(X, Y, axes, return_type=sp.COO))
        assert_order(sp, got, X, Y, axes)
        neg = ([a - X.ndim for a in axes[0]], [a - Y.ndim for a in axes[1]])
        assert_same(sp.sptc(X, Y, neg), got)
    X, Y, axes = pair(sp, rng, order, 1, dtype, perm=False)
    Yl = sp.moveaxis(Y, axes[1][0], 0)
    assert_same(sp.sptc(X, Yl, 1), sp.tensordot(X, Yl, 1, return_type=sp.COO))  # integer axes
    assert_same(sp.sptc(X, Yl, (-1, 0)), sp.tensordot(X, Yl, (-1, 0), return_type=sp.COO))  # scalar axes


def check_axes_out_of_order(sp):
    rng = np.random.default_rng(1)
    X = rand_tensor(sp, rng, (6, 5, 7), 90, "float64", signed=True)
    Y = rand_tensor(sp, rng, (4, 7, 3, 6), 200, "float64", signed=True)
    axes = ([2, 0], [1, 3])
    got = sp.sptc(X, Y, axes)
    assert got.shape == (5, 4, 3)
    assert_same(got, sp.tensordot(X, Y, axes, return_type=sp.COO))
    assert_order(sp, got, X, Y, axes)
    np.testing.assert_allclose(got.todense(), np.tensordot(X.todense(), Y.todense(), axes), rtol=1e-12, atol=1e-12)


def check_low_orders_and_narrow_ints(sp, dtype):
    """Order 1 and 2 operands (2 x 2 is a @ b), the outer product (axes=0), the full contraction, X is Y."""
    rng = np.random.default_rng(2)
    mk = lambda shape, n: (rand_tensor(sp, rng, shape, n, "float64", signed=np.dtype(dtype).kind != "u") * 9).astype(dtype)
    A, B, v, w = mk((12, 9), 50), mk((9, 14), 60), mk((9,), 6), mk((12,), 7)
    for X, Y, axes in ((A, B, 1), (A, v, 1), (w, A, 1), (v, v, 1), (A, A, 2), (A, B, ([1], [0])), (v, w, 0),
                       (A, A, ([0], [0])), (A, A, ([1, 0], [1, 0]))):
        got = sp.sptc(X, Y, axes)
        assert_same(got, sp.tensordot(X, Y, axes, return_type=sp.COO))
    assert_same(sp.sptc(A, B, 1), (A @ B))


def check_gcxs_operands(sp):
    rng = np.random.default_rng(3)
    X = rand_tensor(sp, rng, (7, 6, 5), 80, "float64", signed=True)
    Y = rand_tensor(sp, rng, (5, 4, 6), 60, "float64", signed=True)
    axes = ([1, 2], [2, 0])
    want = sp.sptc(X, Y, axes)
    for k in (1, 2):
        for ca in itertools.combinations(range(3), k):
            G, H = X.asformat("gcxs", compressed_axes=ca), Y.asformat("gcxs", compressed_axes=ca)
            assert_same(sp.sptc(G, Y, axes), want)
            assert_same(sp.sptc(X, H, axes), want)
            assert_same(sp.sptc(G, H, axes), want)


def check_special_values(sp, dtype):
    """Sums that cancel exactly to +0 (pruned), products of -0.0 (a sum that starts at +0 cannot end at -0.0: pruned as
    well), stored zeros, +-inf and NaN (0 * inf is stored as NaN), X entries whose C meets no Y row, Y rows no X entry
    uses."""
    t = np.dtype(dtype).type
    # X (4, 6): row 0 cancels against Y column 0; row 1 holds -0.0 and +0; row 2 meets inf / NaN; row 3 meets no Y row
    xc = np.array([[0, 0, 1, 1, 2, 2, 2, 3, 3], [0, 1, 0, 2, 0, 3, 4, 5, 2]])
    xv = np.array([2.0, -2.0, -0.0, 0.0, 0.0, 1.0, 1.0, 7.0, 0.5], dtype)
    # Y (6, 3): row 5 is absent, so X[3, 5] joins nothing; no X entry uses Y's entry (3, 2) but X[2, 3]
    yc = np.array([[0, 1, 0, 1, 3, 4, 2, 3], [0, 0, 1, 1, 1, 1, 2, 2]])
    yv = np.array([3.0, 3.0, 5.0, 1.0, np.inf, -np.inf, 4.0, np.nan], dtype)
    X = sp.COO(xc, xv, shape=(4, 6))
    Y = sp.COO(yc, yv, shape=(6, 3))
    got = sp.sptc(X, Y, 1)
    assert_same(got, sp.tensordot(X, Y, 1, return_type=sp.COO))
    assert_order(sp, got, X, Y, ([1], [0]))
    d = {(int(i), int(j)): v for i, j, v in zip(*np.asarray(got.coords), got.data)}
    assert (0, 0) not in d  # 2 * 3 + (-2) * 3 = +0: pruned
    assert (1, 0) not in d  # +0 + (-0 * 3) is +0: a sum that starts at +0 never ends at -0.0
    assert np.isnan(d[(2, 1)])  # 0 * 5 + 1 * inf + 1 * -inf
    assert np.isnan(d[(2, 2)])
    assert (3, 0) not in d and (3, 1) not in d and d[(3, 2)] == t(2.0)
    # the integer zero: products that wrap to 0 are pruned, too
    Xi = sp.COO(np.array([[0, 0], [0, 1]]), np.array([2**62, 3], np.int64), shape=(1, 2))
    Yi = sp.COO(np.array([[0, 1], [0, 0]]), np.array([4, 0], np.int64), shape=(2, 1))
    assert sp.sptc(Xi, Yi, 1).nnz == 0 and sp.tensordot(Xi, Yi, 1, return_type=sp.COO).nnz == 0


def check_empty_results_and_zero_length_axes(sp):
    rng = np.random.default_rng(4)
    X = rand_tensor(sp, rng, (6, 8), 10, "float64")
    Xl = sp.COO(np.array([[0, 1], [0, 1]]), np.ones(2), shape=(6, 8))
    Yr = sp.COO(np.array([[6, 7], [0, 1]]), np.ones(2), shape=(8, 3))
    got = sp.sptc(Xl, Yr, 1)  # no common contracted key: every X entry joins the sentinel row
    assert got.nnz == 0 and got.shape == (6, 3)
    assert_same(got, sp.tensordot(Xl, Yr, 1, return_type=sp.COO))
    empty = sp.COO(np.zeros((2, 0), np.int64), np.zeros(0, np.float32), shape=(8, 3))
    for a, b in ((X, empty), (empty.T, X.T)):
        got = sp.sptc(a, b, 1)
        assert got.nnz == 0 and got.dtype == np.float64
        assert_same(got, sp.tensordot(a, b, 1, return_type=sp.COO))
    z = sp.COO(np.zeros((3, 0), np.int64), np.zeros(0), shape=(5, 0, 7))
    y = rand_tensor(sp, rng, (7, 4), 9, "float64")
    for a, b, axes, shape in ((z, y, 1, (5, 0, 4)), (z, z, ([1], [1]), (5, 7, 5, 7)), (z, z, ([0, 2], [0, 2]), (0, 0))):
        got = sp.sptc(a, b, axes)
        assert got.shape == shape and got.nnz == 0 and got.format == "coo"
        want = sp.tensordot(a, b, axes, return_type=sp.COO)
        assert want.shape == got.shape and want.dtype == got.dtype


def planted(sp, rng, shape, n, con, dtype, pool):
    """n entries of `shape` whose coordinates on the axes `con` come from `pool` (so that rows share contracted keys);
    duplicates summed, sorted."""
    c = np.stack([rng.integers(0, s, n) for s in shape])
    pick = rng.integers(0, pool.shape[1], n)
    for k, a in enumerate(con):
        c[a] = pool[k, pick]
    free = [a for a in range(len(shape)) if a not in con]
    c[free[0], : n // 2] = c[free[0], n // 2: 2 * (n // 2)]  # rows with more than one entry
    v = (rng.random(n) + 0.1) * rng.choice([-1.0, 1.0], n)
    return sp.COO(c, v.astype(dtype), shape=shape)


BEYOND = [
    # X over (2e5)^3 contracted over its last mode with a (2e5, 3e5) matrix: tensordot's indptr would have 4e10 entries
    ((200_000,) * 3, (200_000, 300_000), ([2], [0])),
    # order 5 x order 5 over three modes: both matricised sides exceed 2^40 rows or columns
    ((3000, 2000, 500, 700, 900), (700, 4000, 900, 500, 6000), ([2, 3, 4], [3, 0, 2])),
    # contracted axes first on X, last on Y: both operands are re-sorted
    ((50_000, 70_000, 90_000), (30_000, 50_000, 70_000), ([0, 1], [1, 2])),
]


def check_beyond_tensordot_size_limit(sp, case, dtype):
    xs, ys, (ax, ay) = BEYOND[case]
    rng = np.random.default_rng(case)
    pool = np.stack([rng.integers(0, xs[a], 300) for a in ax])
    X = planted(sp, rng, xs, 4000, ax, "float64", pool)
    Y = planted(sp, rng, ys, 3000, ay, "float64", pool)
    if dtype == "int64":
        X, Y = (X * 2**40).astype(dtype), (Y * 2**40).astype(dtype)  # products wrap
    else:
        X, Y = X.astype(dtype), Y.astype(dtype)
    got = sp.sptc(X, Y, (ax, ay))
    assert got.nnz > 10_000
    assert_order(sp, got, X, Y, (ax, ay))
    # nothing cached is sized by an extent: every array of both streams has at most nnz + 2 entries
    for T_ in (X, Y):
        for k, stream in T_._mode_streams.items():
            assert k[0] == "sptc" and all(int(a.shape[0]) <= T_.nnz + 2 for a in stream)


def check_index_widths_and_cache(sp, monkeypatch):
    rng = np.random.default_rng(5)
    X = rand_tensor(sp, rng, (25, 18, 9), 1200, "float64", signed=True)
    Y = rand_tensor(sp, rng, (9, 25, 11), 700, "float64", signed=True)
    axes = ([2, 0], [0, 1])
    sorts = []
    real = sp._kernels.sort_keys

    def counting(*a, **k):
        sorts.append(1)
        return real(*a, **k)

    monkeypatch.setattr(sp._kernels, "sort_keys", counting)
    first = sp.sptc(X, Y, axes)
    n = len(sorts)
    assert n == 2  # X re-sorted over (free, contracted), Y's free keys ranked; Y's (contracted, free) is its own order
    assert ("sptc", "x", (2, 0), True) in X._mode_streams and ("sptc", "y", (0, 1), True) in Y._mode_streams
    again = sp.sptc(X, Y, axes)
    assert len(sorts) == n
    assert_same(again, first)
    assert_same(first, sp.tensordot(X, Y, axes, return_type=sp.COO))
    monkeypatch.setattr(sp._fused, "_FORCE_WIDE_INDEX_SPTC", True)
    wide = sp.sptc(X, Y, axes)
    assert ("sptc", "x", (2, 0), False) in X._mode_streams
    assert str(X._mode_streams[("sptc", "x", (2, 0), False)][1].dtype).endswith("int64")
    assert str(X._mode_streams[("sptc", "x", (2, 0), True)][1].dtype).endswith("int32")
    assert_same(wide, first)
    monkeypatch.setattr(sp._fused, "_FORCE_WIDE_INDEX_SPTC", False)
    # X is Y: both sides cached on one array
    Z = rand_tensor(sp, rng, (12, 12, 5), 300, "float64", signed=True)
    zz = sp.sptc(Z, Z, ([1, 2], [0, 2]))
    assert_same(zz, sp.tensordot(Z, Z, ([1, 2], [0, 2]), return_type=sp.COO))
    assert {k[1] for k in Z._mode_streams} == {"x", "y"}
    # replacing X's contents in place drops its cached rows: the next call builds them again, on the new values
    before = len(sorts)
    np.multiply(X, 2, out=X)
    assert not any(k[0] == "sptc" for k in (X._mode_streams or {}))
    after = sp.sptc(X, Y, axes)
    assert len(sorts) == before + 1
    assert np.array_equal(after.coords, first.coords) and same_bits(after.data, 2 * first.data)


def check_k4_row_paths_through_compressed_rows(sp):
    """Rows of a few products, of more than 256, of more than the long-row threshold (moved down so that small inputs
    reach it), and repeated columns inside one 32-product chunk."""
    rng = np.random.default_rng(6)
    K, G = 400, 600
    rows = []
    for f, nk in enumerate([1, 3, 40, 300, 400, 2, 0, 64]):
        ks = np.sort(rng.choice(K, nk, replace=False))
        rows.append(np.stack([np.full(nk, 1000 * f + 7), ks]))
    xc = np.concatenate(rows, axis=1)
    X = sp.COO(xc, rng.standard_normal(xc.shape[1]), shape=(10_000, K))
    # every Y row k holds columns {0, 1, 2} (repeated across the products of one X row) and a few spread ones
    yc = [np.stack([np.full(3, k), np.arange(3)]) for k in range(K)]
    yc += [np.stack([np.full(4, k), 3 + np.sort(rng.choice(G - 3, 4, replace=False))]) for k in range(K)]
    yc = np.concatenate(yc, axis=1)
    Y = sp.COO(yc, rng.standard_normal(yc.shape[1]), shape=(K, G))
    want = sp.tensordot(X, Y, 1, return_type=sp.COO)
    assert_same(sp.sptc(X, Y, 1), want)
    try:
        for t0, t1 in ((1, 1), (8, 16), (64, 256)):
            sp._kernels.spgemm_set_thresholds(t0, t1)
            X._mode_streams = None
            got = sp.sptc(X, Y, 1)
            assert_same(got, want)
    finally:
        sp._kernels.spgemm_set_thresholds()
    assert_order(sp, got, X, Y, ([1], [0]))


def join_ref(q, s):
    pos = np.searchsorted(s, q)
    hit = (pos < len(s)) & (s[np.minimum(pos, max(len(s) - 1, 0))] == q if len(s) else False)
    return np.where(hit, pos, len(s))


def check_join_alone(sp, ns):
    """Queries before the first and after the last set element, runs of equal queries, absent and present ones, in
    ascending and in shuffled order, every count modulo the four queries a thread takes; both widths."""
    rng = np.random.default_rng(ns)
    s = np.sort(rng.choice(10 * ns + 10, ns, replace=False)).astype(np.int64) + 5
    Kn = sp._kernels
    for nq in (1, 2, 3, 4, 1021, 4096):
        q = np.sort(rng.integers(0, 10 * ns + 30, nq)).astype(np.int64)
        q[: nq // 3] = np.sort(rng.choice(s, nq // 3)) if ns else q[: nq // 3]  # present, with repeats
        q = np.sort(q)
        q[nq // 2: nq // 2 + 5] = q[nq // 2]  # a run of equal queries
        for qq in (q, rng.permutation(q), np.concatenate([q[nq // 2:], q[: nq // 2]])):
            for idt in (np.int32, np.int64):
                got = host(Kn.sptc_join(dev(sp, qq), dev(sp, s), idt))
                assert got.dtype == idt and np.array_equal(got, join_ref(qq, s))
    rows, cols = rng.integers(0, 7, 1001), rng.integers(0, 9, 1001)
    xr, yc = np.sort(rng.choice(2**40, 7, replace=False)), np.sort(rng.choice(2**20, 9, replace=False))
    for n in (1, 2, 1000, 1001):
        keys = host(Kn.sptc_keys(dev(sp, rows[:n]), dev(sp, cols[:n]), dev(sp, xr), dev(sp, yc), 2**20 + 3))
        assert np.array_equal(keys, xr[rows[:n]] * (2**20 + 3) + yc[cols[:n]])


def check_errors(sp):
    rng = np.random.default_rng(8)
    X = rand_tensor(sp, rng, (5, 6, 7), 40, "float64")
    Y = rand_tensor(sp, rng, (7, 6, 4), 40, "float64")
    for axes in (([2], [1]), ([2, 1], [0]), 1 + 2, ([2, 2], [0, 0])):
        with pytest.raises(ValueError, match="shape-mismatch for sum"):
            sp.sptc(X, Y, axes)
    with pytest.raises(ValueError, match="shape-mismatch for sum"):
        sp.tensordot(X, Y, ([2], [1]))
    s = sp.COO(np.zeros((0, 1), np.int64), np.ones(1), shape=())
    with pytest.raises(ValueError, match="Input 0 operand does not have enough dimensions"):
        sp.sptc(s, Y, 1)
    with pytest.raises(ValueError, match="Input 1 operand does not have enough dimensions"):
        sp.sptc(X, s, 1)
    with pytest.raises(IndexError):
        sp.sptc(X, Y, ([3], [0]))
    with pytest.raises(TypeError, match="COO or GCXS"):
        sp.sptc(X, Y.todense(), 1)
    with pytest.raises(TypeError, match="outside the CUDA dtype matrix"):
        sp.sptc(X, Y.astype(np.complex128), 1)
    with pytest.raises(TypeError, match="outside the CUDA dtype matrix"):
        sp.sptc(X.astype(bool), Y.astype(bool), 1)
    with pytest.raises(TypeError, match="outside the CUDA dtype matrix"):
        sp.sptc(X.astype(np.uint64), Y.astype(np.uint64), 1)
    bad = sp.COO(np.asarray(X.coords), np.asarray(X.data), shape=X.shape, fill_value=1.0)
    with pytest.raises(ValueError, match="requires zero fill values"):
        sp.sptc(bad, Y, 1)
    big = sp.COO(np.zeros((3, 1), np.int64), np.ones(1), shape=(2**31, 2**30, 2))
    with pytest.raises(ValueError, match="2\\*\\*63"):
        sp.sptc(big, big, ([2], [2]))
    assert sp.sptc(big, big, ([0, 1], [0, 1])).shape == (2, 2)  # the same operands with a small result fit
    nine = sp.COO(np.zeros((9, 1), np.int64), np.ones(1), shape=(2,) * 9)
    with pytest.raises(ValueError, match="outside 1..8"):
        sp.sptc(nine, nine, 1)


def check_golden_parity(sp, c):
    """One case of tests/golden/sptc_api.npz: the reference's own tensordot(COO, COO, axes, return_type=COO)."""
    X, Y = dec(sp, c, "X_"), dec(sp, c, "Y_")
    got = sp.sptc(X, Y, c["axes"])
    w = c.sub("out_")
    assert got.shape == tuple(int(s) for s in w["shape"]) and got.dtype == w["data"].dtype
    assert same_bits(np.asarray(got.fill_value), np.asarray(w["fill"]))
    assert np.array_equal(np.asarray(got.coords, np.int64), np.asarray(w["coords"], np.int64))
    assert same_bits(got.data, w["data"])


def check_abi_argument_validation(sp):
    """The two entry points exist, and bad arguments come back as B2S_ERR_INVALID with a message (no GPU needed: the
    checks come before any launch)."""
    import ctypes

    from sparse_b200 import _lib

    lib = _lib.load()
    assert {"b2s_sptc_join", "b2s_sptc_keys"} <= set(_lib.header_symbols())
    i64, i32, vp = ctypes.c_int64, ctypes.c_int, ctypes.c_void_p
    INVALID = -1  # B2S_ERR_INVALID
    buf = (ctypes.c_int64 * 8)()
    p = ctypes.addressof(buf)
    assert p % 16 == 0 or (p + 8) % 16 == 0
    al = p if p % 16 == 0 else p + 8
    bad_join = [
        (i32(2), i64(4), vp(al), i64(4), vp(al), vp(al), vp(0)),        # idx_bytes
        (i32(4), i64(-1), vp(al), i64(4), vp(al), vp(al), vp(0)),       # negative size
        (i32(4), i64(4), vp(al), i64(2**31), vp(al), vp(al), vp(0)),    # set too long for 4-byte indices
        (i32(8), i64(4), vp(0), i64(4), vp(al), vp(al), vp(0)),         # NULL pointer
        (i32(8), i64(4), vp(al + 8), i64(4), vp(al), vp(al), vp(0)),    # misaligned queries
    ]
    for args in bad_join:
        assert lib.b2s_sptc_join(*args) == INVALID
        assert b"sptc_join" in lib.b2s_last_error()
    bad_keys = [
        (i64(-1), vp(al), vp(al), vp(al), vp(al), i64(1), vp(al), vp(0)),
        (i64(2), vp(al), vp(al), vp(al), vp(al), i64(0), vp(al), vp(0)),      # g_ext < 1
        (i64(2), vp(al), vp(0), vp(al), vp(al), i64(1), vp(al), vp(0)),       # NULL pointer
        (i64(2), vp(al), vp(al), vp(al), vp(al), i64(1), vp(al + 8), vp(0)),  # misaligned keys
    ]
    for args in bad_keys:
        assert lib.b2s_sptc_keys(*args) == INVALID
        assert b"sptc_keys" in lib.b2s_last_error()
    assert lib.b2s_sptc_join(i32(4), i64(0), vp(0), i64(0), vp(0), vp(0), vp(0)) == 0  # nothing to do


def run_cases(cases):
    """Run (label, callable) pairs in order; a failure carries the label of its case."""
    for label, fn in cases:
        try:
            fn()
        except BaseException as e:
            e.add_note(f"sptc case: {label}")
            raise


def test_sptc_equals_tensordot(sp):
    """The values: bit identity with tensordot and the CPU restatement over orders 2..8 x dtypes, the axes forms, low
    orders and narrow integers, GCXS operands, special values, empty results, and the golden fixture."""
    cases = [(f"bit identity order {o} {dt}", lambda o=o, dt=dt: check_tensordot_bit_identity(sp, o, dt))
             for o in sorted(SHAPES) for dt in ("float32", "float64", "int64")]
    cases.append(("axes out of order", lambda: check_axes_out_of_order(sp)))
    cases += [(f"low orders {dt}", lambda dt=dt: check_low_orders_and_narrow_ints(sp, dt))
              for dt in ("float32", "int32", "int8", "uint16")]
    cases.append(("gcxs operands", lambda: check_gcxs_operands(sp)))
    cases += [(f"special values {dt}", lambda dt=dt: check_special_values(sp, dt)) for dt in ("float32", "float64")]
    cases.append(("empty results", lambda: check_empty_results_and_zero_length_axes(sp)))
    cases += [(f"golden {c['dtype']} case {c['case']}", lambda c=c: check_golden_parity(sp, c))
              for c in load("sptc_api")]
    run_cases(cases)


def test_sptc_compressed_rows_kernels_and_errors(sp, monkeypatch):
    """The structure: shapes beyond tensordot's limit, index widths and the cache, K4's row paths, the join and key
    kernels alone, the errors of the public call and of the C entry points."""
    cases = [(f"beyond tensordot case {k} {dt}", lambda k=k, dt=dt: check_beyond_tensordot_size_limit(sp, k, dt))
             for k in range(len(BEYOND)) for dt in ("float32", "int64")]
    cases.append(("index widths and cache", lambda: check_index_widths_and_cache(sp, monkeypatch)))
    cases.append(("K4 row paths", lambda: check_k4_row_paths_through_compressed_rows(sp)))
    cases += [(f"join alone, set of {ns}", lambda ns=ns: check_join_alone(sp, ns)) for ns in (0, 1, 31, 32, 33, 5000)]
    cases.append(("errors", lambda: check_errors(sp)))
    cases.append(("ABI argument validation", lambda: check_abi_argument_validation(sp)))
    run_cases(cases)
