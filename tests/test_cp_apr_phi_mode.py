"""cp_apr_phi_mode(X, factors, mode, eps): the ratio MTTKRP Phi of Poisson CP (CP-APR).

Parity with a float64 NumPy evaluation and with the reference's unfused model, ratio and MTTKRP expressions (golden
fixture), bit equality with the CPU restatement of the fixed order of operations (tests/_tensor_order.py) at chunk
edges and with special values (tests/_cp_apr_order.py), the identity with mttkrp_mode of the ratios, bit-identical results across calls,
copies, storage layouts, factor layouts and locations and both index widths, the mode-stream cache shared with the
other mode-stream ops, edge cases, errors, and a CP-APR multiplicative-update run against a dense NumPy one.  Every body
runs on the NumPy mock without a GPU (the op's stand-in is tests/_mock_cp_apr.py, installed by a fixture here) and on
the CUDA kernels with `-m gpu`."""
import numpy as np
import pytest

import _cp_apr_order as CA
import _mock_cp_apr
import _tensor_order as TO
from _api import dec, sp  # noqa: F401
from _golden import load
from _tensor_cases import LAYOUTS, SHAPES, chunk, chunk_structured, dev, edge_rows, host, layout, rand_tensor

TOL = {"float32": 2e-4, "float64": 1e-11}
same_bits = TO.same_bits


@pytest.fixture(autouse=True)
def _mock_stand_in(request):
    """On the NumPy mock backend, the op's stand-in (tests/_mock_cp_apr.py) in place of the real wrapper."""
    if "sp" not in request.fixturenames:
        yield
        return
    sp = request.getfixturevalue("sp")
    if not sp._device._TEST_CPU:
        yield
        return
    real = sp._kernels.cp_apr_phi_mode
    sp._kernels.cp_apr_phi_mode = _mock_cp_apr.cp_apr_phi_mode
    yield
    sp._kernels.cp_apr_phi_mode = real


def stored(X):
    c = X.tocoo() if X.format == "gcxs" else X
    return np.asarray(c.coords, np.int64), np.asarray(c.data)


def phi64(X, U, mode, eps):
    """float64: sum over row i's stored entries of v / max(m, eps) times the other factors' rows, m the model of every
    factor at the entry."""
    coords, vals = stored(X)
    g = [np.asarray(u, np.float64)[coords[m]] for m, u in enumerate(U)]
    m = np.prod(g, axis=0).sum(axis=1)
    w = vals.astype(np.float64) / np.maximum(m, eps)
    h = np.prod([g[k] for k in range(X.ndim) if k != mode], axis=0)
    out = np.zeros((X.shape[mode], h.shape[1]))
    np.add.at(out, coords[mode], w[:, None] * h)
    return out


def order_ref(sp, X, U, mode, dtype, eps):
    coords, vals = stored(X)
    return CA.cp_apr_phi_mode(coords, vals, U, mode, X.shape[mode], chunk(sp), dtype, eps)


def close(got, want, dtype):
    tol = TOL[np.dtype(dtype).name]
    np.testing.assert_allclose(got, want, rtol=tol, atol=tol * max(np.abs(want).max(), 1.0))


# f32 packs hold 4 columns and f64 ones 2: R = 1, 3 and 37 read padded copies of the factors, 4 (f64), 16 and 64 the
# factors themselves.  Each (order, R) pair takes one of the four storage layouts, in turn.
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("order", sorted(SHAPES))
def test_fp64_parity_every_mode(sp, order, dtype):
    shape = SHAPES[order]
    for k, R in enumerate([1, 3, 4, 16, 37, 64]):
        fmt, ca = LAYOUTS[(k + order) % len(LAYOUTS)]
        if ca == (0, 1) and order == 2:
            fmt, ca = "gcxs", (1,)  # an order-2 tensor cannot compress two axes
        rng = np.random.default_rng(20 * order + R)
        X = rand_tensor(sp, rng, shape, max(int(np.prod(shape)) // 4, 5), dtype, fmt,
                        (order - 1,) if ca == "last" else ca)
        U = [rng.random((s, R)).astype(dtype) + np.asarray(0.05, dtype) for s in shape]
        for mode in range(order):
            got = sp.cp_apr_phi_mode(X, U, mode)
            assert isinstance(got, np.ndarray) and got.dtype == np.dtype(dtype) and got.shape == (shape[mode], R)
            close(got, phi64(X, U, mode, 1e-10), dtype)


GOLDEN = load("cp_apr_phi_api")


@pytest.mark.parametrize("c", GOLDEN, ids=lambda c: f"{c['dtype']}-order{c['order']}-mode{c['mode']}")
def test_golden_parity(sp, c):
    N, mode = int(c["order"]), int(c["mode"])
    X = dec(sp, c, "X_", "gcxs" if mode % 2 else "coo")
    U = [np.array(c.arr[f"U{m}"]) for m in range(N)]
    got = sp.cp_apr_phi_mode(X, U, mode, c["eps"])
    want = dec(sp, c, "out_").todense()
    assert got.dtype == np.dtype(c["dtype"]) and got.shape == want.shape
    close(got, want, c["dtype"])


def with_zero_models(U):
    """Rows of the last factor that are +0 and -0: every entry there has the model m = +0 (no entry has m = -0)."""
    U[2][[1, 5]] = 0.0
    U[2][[3, 7]] = -0.0
    return U


@pytest.mark.parametrize("R", [1, 5, 8, 32])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_exact_order(sp, dtype, R):
    """Signed data and factors (so that some models are below eps), +-inf / NaN factors, -0.0 values and zero models,
    at the chunk edges (rows of 511, 512, 513 entries) and on rows over several chunks; eps > 0 and eps = 0."""
    rng = np.random.default_rng(R)
    X, U = edge_rows(sp, rng, dtype, R)
    Y, V = chunk_structured(sp, rng, dtype, R)
    with_zero_models(U)
    with_zero_models(V)
    for T, W in ((X, U), (Y, V)):
        for mode in range(3):
            for eps in (0.5, 0.0):
                assert same_bits(sp.cp_apr_phi_mode(T, W, mode, eps), order_ref(sp, T, W, mode, dtype, eps)), (mode, eps)
    # eps = 0 with m = +0: v / 0 is +-inf or NaN, so the rows of those entries are not finite
    assert not np.isfinite(sp.cp_apr_phi_mode(X, U, 2, 0.0)[[1, 3, 5, 7]]).all()


def test_exact_order_row_over_hundreds_of_chunks(sp):
    """A mode of extent 2: each of its rows spans about 250 chunks."""
    rng = np.random.default_rng(4)
    X = rand_tensor(sp, rng, (500, 500, 2), 256_000, "float32", signed=True)
    U = [rng.standard_normal((s, 6)).astype(np.float32) for s in X.shape]
    assert same_bits(sp.cp_apr_phi_mode(X, U, 2, 0.5), order_ref(sp, X, U, 2, "float32", 0.5))


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_is_mttkrp_mode_of_the_ratios(sp, dtype):
    """cp_apr_phi_mode equals mttkrp_mode of a COO holding the ratios w (formed on the host from tttp's model values)
    bit for bit; and at order 2 it is (X / max(A B^T, eps)) B, the matrix formula."""
    rng = np.random.default_rng(5)
    X = rand_tensor(sp, rng, (30, 20, 10), 1500, dtype)
    U = [rng.random((s, 5)).astype(dtype) for s in X.shape]
    eps = float(np.quantile(TO.values(X.coords, np.ones(X.nnz), U, dtype), 0.3))  # some models are clamped
    P = sp.COO(X.coords, np.ones(X.nnz, dtype), shape=X.shape, has_duplicates=False, sorted=True)
    m = sp.tttp(P, U).data
    assert same_bits(m, TO.values(X.coords, np.ones(X.nnz), U, dtype))
    e = np.asarray(eps, dtype)
    w = X.data / np.where(m < e, e, m)
    W = sp.COO(X.coords, w, shape=X.shape, has_duplicates=False, sorted=True)
    for mode in range(3):
        assert same_bits(sp.cp_apr_phi_mode(X, U, mode, eps), sp.mttkrp_mode(W, U, mode)), mode
    A = rand_tensor(sp, rng, (40, 30), 500, dtype)
    F = [rng.random((40, 4)).astype(dtype), rng.random((30, 4)).astype(dtype)]
    ratio = A.todense().astype(np.float64) / np.maximum(F[0].astype(np.float64) @ F[1].T.astype(np.float64), 0.3)
    close(sp.cp_apr_phi_mode(A, F, 0, 0.3), ratio @ F[1].astype(np.float64), dtype)
    close(sp.cp_apr_phi_mode(A, F, 1, 0.3), ratio.T @ F[0].astype(np.float64), dtype)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_bit_identical_across_calls_copies_layouts_locations_and_index_widths(sp, dtype, monkeypatch):
    """Repeated calls, a copy of X, every storage layout, device, mixed, Fortran-ordered, transposed and offset-view
    (unaligned) factors and forced int64 indices give the first call's bits; a device factor gives a device result."""
    import torch

    rng = np.random.default_rng(11)
    X = rand_tensor(sp, rng, (70, 60, 8), 9000, dtype)
    U = [rng.random((s, 12)).astype(dtype) for s in X.shape]
    Ud = [dev(sp, u) for u in U]
    variants = [[np.asfortranarray(u) for u in U], Ud, [U[0], Ud[1], U[2]], [dev(sp, u.T.copy()).T for u in U],
                [dev(sp, np.concatenate([np.zeros((u.shape[0], 1), dtype), u], axis=1))[:, 1:] for u in U]]
    for mode in range(3):
        first = sp.cp_apr_phi_mode(X, U, mode, 0.25)
        for got in [sp.cp_apr_phi_mode(X, U, mode, 0.25) for _ in range(2)] + [sp.cp_apr_phi_mode(X.copy(), U, mode, 0.25)]:
            assert same_bits(got, first), mode
        for lay in LAYOUTS[1:]:
            assert same_bits(sp.cp_apr_phi_mode(layout(X, *lay), U, mode, 0.25), first), (mode, lay)
        for V in variants:
            got = sp.cp_apr_phi_mode(X, V, mode, 0.25)
            assert isinstance(got, np.ndarray if V is variants[0] else torch.Tensor)
            assert same_bits(host(got), first), mode
        monkeypatch.setattr(sp._fused, "_FORCE_WIDE_INDEX", True)
        wide = sp.cp_apr_phi_mode(X, U, mode, 0.25)
        monkeypatch.setattr(sp._fused, "_FORCE_WIDE_INDEX", False)
        assert same_bits(wide, first), mode
        assert all(c.element_size() == 8 for c in X._mode_streams[(mode, False)][0]), mode
        assert all(c.element_size() == 4 for c in X._mode_streams[(mode, True)][0]), mode


def test_mode_stream_cache(sp, monkeypatch):
    """No sort when mttkrp_mode has built the stream, and none in the other mode-stream ops after cp_apr_phi_mode has;
    new contents (np.multiply(..., out=X)) drop the cache."""
    calls = []
    real = sp._kernels.sort_keys

    def counting(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(sp._kernels, "sort_keys", counting)
    rng = np.random.default_rng(3)
    X = rand_tensor(sp, rng, (30, 20, 10), 1500, "float64")
    U = [rng.random((s, 6)) for s in X.shape]
    sp.mttkrp_mode(X, U, 1)
    assert len(calls) == 1
    before = sp.cp_apr_phi_mode(X, U, 1)
    assert len(calls) == 1
    sp.cp_apr_phi_mode(X, U, 2)
    assert len(calls) == 2
    sp.mttkrp_mode(X, U, 2), sp.ttmc_mode(X, U, 2), sp.cp_completion_mode(X, U, 2, 0.5)
    assert len(calls) == 2
    np.multiply(X, 2, out=X)
    assert same_bits(sp.cp_apr_phi_mode(X, U, 1), 2 * before)  # doubling v doubles w and the sums exactly
    assert len(calls) == 3


def test_edge_cases(sp):
    rng = np.random.default_rng(8)
    U = [rng.random((s, 4)) for s in (5, 6, 7)]
    empty = sp.COO(np.zeros((3, 0), np.int64), np.zeros(0), shape=(5, 6, 7))
    for m in range(3):
        got = sp.cp_apr_phi_mode(empty, U, m)
        assert got.shape == (U[m].shape[0], 4) and not got.any() and not np.signbit(got).any()
    X = rand_tensor(sp, rng, (5, 6, 7), 60, "float64")
    assert sp.cp_apr_phi_mode(X, [np.zeros((s, 0)) for s in X.shape], 1).shape == (6, 0)
    zero_ext = sp.COO(np.zeros((3, 0), np.int64), np.zeros(0), shape=(5, 0, 7))
    assert sp.cp_apr_phi_mode(zero_ext, [np.ones((5, 2)), np.ones((0, 2)), np.ones((7, 2))], 1).shape == (0, 2)
    got = sp.cp_apr_phi_mode(X, U, 1, np.float32(0.5))
    assert same_bits(got, sp.cp_apr_phi_mode(X, U, -2, 0.5))
    assert same_bits(sp.cp_apr_phi_mode(X, U, 0, 0), sp.cp_apr_phi_mode(X, U, 0, 0.0))
    rows = set(np.asarray(X.coords[0]).tolist())
    got = sp.cp_apr_phi_mode(X, U, 0)
    for i in set(range(5)) - rows:  # rows without entries are +0
        assert not got[i].any() and not np.signbit(got[i]).any()


def test_errors(sp, monkeypatch):
    rng = np.random.default_rng(11)
    X = rand_tensor(sp, rng, (5, 6, 7), 40, "float64")
    U = [rng.random((s, 3)) for s in X.shape]
    with pytest.raises(TypeError):
        sp.cp_apr_phi_mode(X.todense(), U, 0)
    for bad in (U[:2], U + [U[0]], [None, U[1], U[2]], [rng.random((4, 3)), U[1], U[2]],
                [rng.random((5, 4)), U[1], U[2]], [rng.random(5), U[1], U[2]]):
        with pytest.raises(ValueError):  # factors[mode] (here 0) is read and checked like the others
            sp.cp_apr_phi_mode(X, bad, 0)
    for bad in (3, -4):
        with pytest.raises(np.exceptions.AxisError):
            sp.cp_apr_phi_mode(X, U, bad)
    for bad in (np.nan, np.inf, -np.inf, -1e-3):
        with pytest.raises(ValueError, match="eps"):
            sp.cp_apr_phi_mode(X, U, 0, bad)
    with pytest.raises(ValueError, match="eps"):  # finite in float64, inf once cast to float32
        sp.cp_apr_phi_mode(X.astype(np.float32), [u.astype(np.float32) for u in U], 0, 1e39)
    for bad in (None, "1", 1j, True):
        with pytest.raises(TypeError):
            sp.cp_apr_phi_mode(X, U, 0, bad)
    with pytest.raises(TypeError, match="outside the CUDA dtype matrix"):
        Xi = sp.COO(X.coords, np.arange(1, X.nnz + 1), shape=X.shape)
        sp.cp_apr_phi_mode(Xi, [np.ones((s, 3), np.int64) for s in X.shape], 1)
    with pytest.raises(ValueError, match="zero fill"):
        sp.cp_apr_phi_mode(sp.COO(X.coords, X.data, shape=X.shape, fill_value=1.0), U, 0)
    nine = sp.COO(np.zeros((9, 1), np.int64), np.ones(1), shape=(2,) * 9)
    with pytest.raises(ValueError, match="order 9"):
        sp.cp_apr_phi_mode(nine, [np.ones((2, 2))] * 9, 0)

    # R above the limit: refused before the mode stream or the result is allocated
    def no_alloc(*a, **k):
        raise AssertionError("allocated before the rank check")

    limit = sp._kernels.cp_apr_phi_max_rank()
    assert limit == 64
    monkeypatch.setattr(sp._fused, "_mode_stream", no_alloc)
    monkeypatch.setattr(sp._kernels, "full", no_alloc)
    with pytest.raises(ValueError, match="exceeds the limit"):
        sp.cp_apr_phi_mode(X, [rng.random((s, limit + 1)) for s in X.shape], 0)


def mu_run(X, U, outer, l_max, eps, phi, nll):
    """CP-APR multiplicative updates (the loop of the cp_apr_phi_mode docstring) with the Phi and negative
    log-likelihood given; returns the factors, the weights and the log-likelihood after every inner iteration."""
    U = [u.copy() for u in U]
    lam = np.ones(U[0].shape[1])
    trace = []
    for _ in range(outer):
        for n in range(X.ndim):
            B = U[n] * lam
            for _ in range(l_max):
                B = B * phi(U[:n] + [B] + U[n + 1:], n)
                trace.append(nll(U[:n] + [B] + U[n + 1:], n))
            lam = B.sum(axis=0)
            U[n] = B / lam
    return U, lam, trace


def test_cp_apr_mu_run_matches_dense(sp):
    """A planted rank-3 Poisson tensor of shape (30, 25, 20) in float64: CP-APR's MU steps with cp_apr_phi_mode and
    tttp never increase the negative log-likelihood, and end at the factors of a dense NumPy MU run to 1e-8."""
    rng = np.random.default_rng(17)
    shape, R, eps = (30, 25, 20), 3, 1e-10
    truth = [rng.gamma(0.5, size=(s, R)) for s in shape]
    M = np.einsum("ir,jr,kr->ijk", *truth) * 2.0
    dense = rng.poisson(M).astype(np.float64)
    coords = np.stack(np.nonzero(dense))
    X = sp.COO(coords, dense[tuple(coords)], shape=shape, has_duplicates=False, sorted=True)
    P = sp.COO(coords, np.ones(X.nnz), shape=shape, has_duplicates=False, sorted=True)
    U0 = [rng.random((s, R)) + 0.1 for s in shape]
    U0 = [u / u.sum(axis=0) for u in U0]

    def nll_sparse(F, n):  # the other factors' columns sum to 1, so the model's total is B's
        return F[n].sum() - float(X.data @ np.log(sp.tttp(P, F).data))

    def phi_dense(F, n):
        letters = "ijk"
        model = np.einsum("ir,jr,kr->ijk", *F)
        ratio = dense / np.maximum(model, eps)
        others = [m for m in range(3) if m != n]
        return np.einsum(f"ijk,{letters[others[0]]}r,{letters[others[1]]}r->{letters[n]}r", ratio,
                         F[others[0]], F[others[1]])

    U_s, lam_s, trace = mu_run(X, U0, 4, 10, eps, lambda F, n: sp.cp_apr_phi_mode(X, F, n, eps), nll_sparse)
    U_d, lam_d, _ = mu_run(X, U0, 4, 10, eps, phi_dense, lambda F, n: 0.0)
    for a, b in zip(trace, trace[1:]):
        assert b <= a + 1e-9 * abs(a), (a, b)
    assert trace[-1] < trace[0]
    np.testing.assert_allclose(lam_s, lam_d, rtol=1e-8)
    for a, b in zip(U_s, U_d):
        np.testing.assert_allclose(a, b, rtol=1e-8, atol=1e-12)


@pytest.mark.gpu
def test_large_f32_against_fp64_and_restatement():
    """About 1e7 float32 entries of a (2000, 1500, 1000) tensor, R = 16, nonnegative factors, eps clamping the
    smallest models: every row against a float64 device evaluation, and sampled rows bit for bit against the CPU
    restatement, at modes 0 and 2."""
    import torch

    import sparse_b200 as spm

    devc = torch.device("cuda")
    shape, R, nnz = (2000, 1500, 1000), 16, 10_000_000
    g = torch.Generator(device=devc).manual_seed(7)
    lin = torch.unique(torch.randint(0, shape[0] * shape[1] * shape[2], (nnz,), generator=g, device=devc))
    coords = torch.stack(torch.unravel_index(lin, shape))
    vals = torch.poisson(torch.full((coords.shape[1],), 1.5, device=devc), generator=g) + 1.0
    X = spm.COO(coords, vals, shape=shape, has_duplicates=False, sorted=True)
    U = [torch.rand((s, R), generator=g, device=devc) for s in shape]
    eps = 1.0  # the models lie in about (0, 4): the smallest are clamped
    h = [u[c].double() for u, c in zip(U, coords)]
    w = vals.double() / (h[0] * h[1] * h[2]).sum(1).clamp_min(eps)
    for mode in (0, 2):
        got = spm.cp_apr_phi_mode(X, U, mode, eps)
        others = [m for m in range(3) if m != mode]
        want = torch.zeros((shape[mode], R), dtype=torch.float64, device=devc)
        want.index_add_(0, coords[mode], w[:, None] * h[others[0]] * h[others[1]])
        err = (got.double() - want).abs().amax(1) / want.abs().amax(1).clamp_min(1e-30)
        assert float(err.max()) < 1e-4, float(err.max())
        rows = np.random.default_rng(mode).choice(shape[mode], 4, replace=False)
        assert CA.sampled_rows_exact(got, coords, vals, U, mode, rows, 512, eps)
