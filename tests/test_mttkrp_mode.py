"""mttkrp_mode(X, factors, mode): mode-n MTTKRP of sparse tensors of order 2..8.

Parity with float64 dense einsum and with the reference's unfused broadcast expression (golden fixtures), bit
equality with a CPU restatement of the fixed order of operations (tests/_mttkrp_order.py), determinism, the mode-stream
cache, factor layouts, edge cases and errors.  Every body runs on the NumPy mock without a GPU and on the CUDA kernels
with `-m gpu`."""
import pickle
import string

import numpy as np
import pytest

import _mttkrp_order as MO
from _api import dec, sp  # noqa: F401
from _golden import load

TOL = {"float32": 2e-5, "float64": 1e-12}


@pytest.fixture(autouse=True)
def _mock_stand_in(request, monkeypatch):
    """On the mock backend, the NumPy stand-in of the K10 wrapper joins the mocked kernel layer."""
    if "sp" in request.fixturenames:
        backend = request.getfixturevalue("sp")
        if backend._device._TEST_CPU:
            import _mock_mttkrp

            monkeypatch.setattr(backend._kernels, "mttkrp_mode", _mock_mttkrp.mttkrp_mode)


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


def einsum_ref(X, factors, mode):
    N = X.ndim
    letters = string.ascii_lowercase[:N]
    terms = [letters] + [letters[m] + "z" for m in range(N) if m != mode]
    ops = [X.todense().astype(np.float64)] + [np.asarray(factors[m], np.float64) for m in range(N) if m != mode]
    return np.einsum(",".join(terms) + "->" + letters[mode] + "z", *ops)


def order_ref(sp, X, factors, mode, dtype):
    c = X.tocoo() if X.format == "gcxs" else X
    return MO.mttkrp_mode(c.coords, c.data, factors, mode, X.shape[mode], chunk(sp), dtype)


# orders 2..8, small extents so the dense einsum stays small; three storage layouts per tensor
SHAPES = {2: (37, 29), 3: (23, 17, 11), 4: (9, 7, 6, 5), 5: (6, 5, 4, 3, 5), 8: (3, 2, 3, 2, 2, 3, 2, 2)}
LAYOUTS = [("coo", None), ("gcxs", (0,)), ("gcxs", "last"), ("gcxs", (0, 1))]


@pytest.mark.parametrize("R", [1, 3, 8, 32, 33, 100, 256])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("order", sorted(SHAPES))
@pytest.mark.parametrize("layout", range(len(LAYOUTS)), ids=lambda i: LAYOUTS[i][0] + str(LAYOUTS[i][1] or ""))
def test_fp64_parity_every_mode(sp, order, dtype, R, layout):
    shape = SHAPES[order]
    fmt, ca = LAYOUTS[layout]
    if ca == "last":
        ca = (order - 1,)
    if ca == (0, 1) and order == 2:
        pytest.skip("an order-2 tensor cannot compress two axes")
    rng = np.random.default_rng(1000 * order + R)
    X = rand_tensor(sp, rng, shape, max(int(np.prod(shape)) // 4, 5), dtype, fmt, ca)
    U = [rng.random((s, R)).astype(dtype) + np.asarray(0.05, dtype) for s in shape]
    for mode in range(order):
        got = sp.mttkrp_mode(X, U, mode)
        assert isinstance(got, np.ndarray) and got.dtype == np.dtype(dtype) and got.shape == (shape[mode], R)
        np.testing.assert_allclose(got, einsum_ref(X, U, mode), rtol=TOL[dtype], atol=0)


GOLDEN = [c for c in load("mttkrp_mode_api") if c["op"] == "mttkrp_mode"]


@pytest.mark.parametrize("c", GOLDEN, ids=lambda c: f"{c['dtype']}-order{c['order']}-mode{c['mode']}")
@pytest.mark.parametrize("fmt", ["coo", "gcxs"])
def test_golden_parity(sp, c, fmt):
    X = dec(sp, c, "X_", fmt)
    U = [np.array(c.arr[f"U{m}"]) for m in range(int(c["order"]))]
    mode = int(c["mode"])
    U[mode] = None
    got = sp.mttkrp_mode(X, U, mode)
    w = c.sub("out_")
    want = sp.COO(np.array(w["coords"]), np.array(w["data"]), shape=tuple(int(s) for s in w["shape"])).todense()
    tol = TOL[c["dtype"]]
    assert got.dtype == want.dtype
    np.testing.assert_allclose(got, want, rtol=tol, atol=tol)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_order3_mode0_matches_mttkrp(sp, dtype):
    rng = np.random.default_rng(5)
    B = rand_tensor(sp, rng, (40, 30, 20), 3000, dtype)
    Dm, Cm = rng.random((20, 16)).astype(dtype), rng.random((30, 16)).astype(dtype)
    got = sp.mttkrp_mode(B, [None, Cm, Dm], 0)
    np.testing.assert_allclose(got, sp.mttkrp(B, Dm, Cm).todense(), rtol=TOL[dtype], atol=0)


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
    for u in U:
        flat = u.reshape(-1)
        flat[rng.choice(flat.size, min(4, flat.size), replace=False)] = [np.inf, -np.inf, np.nan, -0.0][: min(4, flat.size)]
    return X, U


@pytest.mark.parametrize("R", [1, 5, 8, 32])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_exact_order(sp, dtype, R):
    X, U = chunk_structured(sp, np.random.default_rng(R), dtype, R)
    for mode in range(3):
        got = sp.mttkrp_mode(X, U, mode)
        assert MO.same_bits(got, order_ref(sp, X, U, mode, dtype)), mode


def test_exact_order_skewed_mode(sp):
    """A mode with 3 slices of thousands of entries each: every slice spans many chunks."""
    rng = np.random.default_rng(7)
    X = rand_tensor(sp, rng, (60, 50, 3), 6000, "float32", signed=True)
    U = [rng.standard_normal((s, 8)).astype(np.float32) for s in X.shape]
    for mode in (2, -1, 0):
        assert MO.same_bits(sp.mttkrp_mode(X, U, mode), order_ref(sp, X, U, mode % 3, "float32"))


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_determinism(sp, dtype):
    rng = np.random.default_rng(11)
    X = rand_tensor(sp, rng, (70, 60, 8), 9000, dtype, signed=True)
    U = [rng.standard_normal((s, 24)).astype(dtype) for s in X.shape]
    Ud = [dev(sp, u) for u in U]
    for mode in range(3):
        first = sp.mttkrp_mode(X, U, mode)
        for _ in range(3):
            assert MO.same_bits(sp.mttkrp_mode(X, U, mode), first)
        assert MO.same_bits(sp.mttkrp_mode(X.copy(), U, mode), first)  # the copy builds its stream again
        assert MO.same_bits(host(sp.mttkrp_mode(X, Ud, mode)), first)


def test_cache_sorts_once_per_mode_and_follows_new_values(sp, monkeypatch):
    Kn = sp._kernels
    calls = []
    real = Kn.sort_keys

    def counting(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(Kn, "sort_keys", counting)
    rng = np.random.default_rng(3)
    X = rand_tensor(sp, rng, (30, 20, 10), 1500, "float64", signed=True)
    U = [rng.standard_normal((s, 6)) for s in X.shape]
    before = {}
    for mode in (0, 1, 2):
        calls.clear()
        for _ in range(3):
            before[mode] = sp.mttkrp_mode(X, U, mode)
        assert len(calls) == (0 if mode == 0 else 1), mode
    assert X.copy()._mode_streams is None
    assert pickle.loads(pickle.dumps(X))._mode_streams is None
    np.multiply(X, 2, out=X)
    for mode in (0, 1, 2):
        assert MO.same_bits(sp.mttkrp_mode(X, U, mode), 2 * before[mode])

    G = X.asformat("gcxs", compressed_axes=(1,))
    calls.clear()
    for _ in range(2):
        g1 = sp.mttkrp_mode(G, U, 1)
    assert MO.same_bits(g1, sp.mttkrp_mode(X, U, 1))
    n_first = len(calls)
    sp.mttkrp_mode(G, U, 1)
    assert len(calls) == n_first


def test_factor_layouts_and_output_kind(sp):
    import torch

    rng = np.random.default_rng(13)
    R = 12
    X = rand_tensor(sp, rng, (40, 30, 20), 2500, "float32", signed=True)
    U = [rng.standard_normal((s, R)).astype(np.float32) for s in X.shape]
    want = [sp.mttkrp_mode(X, U, m) for m in range(3)]
    fortran = [np.asfortranarray(u) for u in U]
    transposed = [dev(sp, u.T.copy()).T for u in U]  # device, column-major
    wide = [dev(sp, np.concatenate([np.zeros((u.shape[0], 1), np.float32), u], axis=1))[:, 1:] for u in U]
    mixed = [U[0], dev(sp, U[1]), U[2]]
    for m in range(3):
        assert MO.same_bits(sp.mttkrp_mode(X, fortran, m), want[m])
        for variant in (transposed, wide, mixed):
            got = sp.mttkrp_mode(X, variant, m)
            assert isinstance(got, torch.Tensor)
            assert MO.same_bits(host(got), want[m])
    # a float64 factor promotes the result
    U64 = [U[0], U[1].astype(np.float64), U[2]]
    got = sp.mttkrp_mode(X, U64, 0)
    assert got.dtype == np.float64
    np.testing.assert_allclose(got, einsum_ref(X, U64, 0), rtol=1e-12)


def test_edge_cases(sp):
    rng = np.random.default_rng(17)
    U = [rng.random((s, 4)) for s in (5, 6, 7)]
    empty = sp.COO(np.zeros((3, 0), np.int64), np.zeros(0), shape=(5, 6, 7))
    for m in range(3):
        got = sp.mttkrp_mode(empty, U, m)
        assert got.shape == (U[m].shape[0], 4) and not got.any() and not np.signbit(got).any()
    X = rand_tensor(sp, rng, (5, 6, 7), 60, "float64")
    U0 = [np.zeros((s, 0)) for s in (5, 6, 7)]
    assert sp.mttkrp_mode(X, U0, 1).shape == (6, 0)
    one = rand_tensor(sp, rng, (1, 50, 40), 300, "float64")
    Uo = [rng.random((s, 3)) for s in one.shape]
    for m in range(3):
        np.testing.assert_allclose(sp.mttkrp_mode(one, Uo, m), einsum_ref(one, Uo, m), rtol=1e-12)
    sparse_rows = rand_tensor(sp, rng, (500, 4, 3), 20, "float64")  # most rows empty
    Us = [rng.random((s, 2)) for s in sparse_rows.shape]
    got = sp.mttkrp_mode(sparse_rows, Us, 0)
    np.testing.assert_allclose(got, einsum_ref(sparse_rows, Us, 0), rtol=1e-12)
    assert (got == 0).sum() >= 480 and not np.signbit(got[got == 0]).any()
    assert MO.same_bits(sp.mttkrp_mode(X, U, -1), sp.mttkrp_mode(X, U, 2))


def test_int64_index_path(sp, monkeypatch):
    rng = np.random.default_rng(19)
    X = rand_tensor(sp, rng, (50, 40, 9), 4000, "float32", signed=True)
    U = [rng.standard_normal((s, 16)).astype(np.float32) for s in X.shape]
    narrow = [sp.mttkrp_mode(X, U, m) for m in range(3)]
    monkeypatch.setattr(sp._fused, "_FORCE_WIDE_INDEX", True)
    for m in range(3):
        assert MO.same_bits(sp.mttkrp_mode(X, U, m), narrow[m])
    assert all(c.element_size() == 8 for c in X._mode_streams[(1, False)][0])
    assert all(c.element_size() == 4 for c in X._mode_streams[(1, True)][0])


def test_errors(sp):
    rng = np.random.default_rng(23)
    X = rand_tensor(sp, rng, (5, 6, 7), 40, "float64")
    U = [rng.random((s, 3)) for s in X.shape]
    with pytest.raises(TypeError):
        sp.mttkrp_mode(X.todense(), U, 0)
    with pytest.raises(ValueError):
        sp.mttkrp_mode(rand_tensor(sp, rng, (9,), 4, "float64"), [rng.random((9, 2))], 0)
    nine = sp.COO(np.zeros((9, 1), np.int64), np.ones(1), shape=(2,) * 9)
    with pytest.raises(ValueError):
        sp.mttkrp_mode(nine, [np.ones((2, 2))] * 9, 0)
    with pytest.raises(ValueError, match="zero fill"):
        sp.mttkrp_mode(sp.COO(X.coords, X.data, shape=X.shape, fill_value=1.0), U, 0)
    for bad in (3, -4):
        with pytest.raises(np.exceptions.AxisError):
            sp.mttkrp_mode(X, U, bad)
    with pytest.raises(ValueError):
        sp.mttkrp_mode(X, U[:2], 0)
    with pytest.raises(ValueError):
        sp.mttkrp_mode(X, [U[0], rng.random((6, 4)), U[2]], 0)
    with pytest.raises(ValueError):
        sp.mttkrp_mode(X, [U[0], rng.random((5, 3)), U[2]], 0)
    with pytest.raises(TypeError, match="outside the CUDA dtype matrix"):
        Xi = sp.COO(X.coords, np.arange(1, X.nnz + 1), shape=X.shape)
        sp.mttkrp_mode(Xi, [np.ones((s, 3), np.int64) for s in X.shape], 0)


@pytest.mark.gpu
def test_full_size_each_mode():
    """(1e6, 1e6, 100) with 1e8 uniform entries, R = 32, f32: every row within 2e-5 of a float64 restatement on the
    device; 16 sampled rows per mode (two of the 100 slices of mode 2) bit-equal to the CPU order restatement."""
    import torch

    import sparse_b200 as spm

    devc = torch.device("cuda")
    shape, nnz, R = (1_000_000, 1_000_000, 100), 100_000_000, 32
    g = torch.Generator(device=devc).manual_seed(77)
    lin = torch.unique(torch.randint(0, shape[0] * shape[1] * shape[2], (nnz,), generator=g, device=devc))
    coords = torch.stack(torch.unravel_index(lin, shape))
    del lin
    vals = torch.rand(coords.shape[1], generator=g, device=devc) + 0.1
    X = spm.COO(coords, vals, shape=shape, has_duplicates=False, sorted=True)
    U = [torch.rand((s, R), generator=g, device=devc) + 0.05 for s in shape]
    ch = spm._kernels.mttkrp_mode_chunk()
    rng = np.random.default_rng(5)
    for mode in range(3):
        got = spm.mttkrp_mode(X, U, mode)
        want = torch.zeros((shape[mode], R), dtype=torch.float64, device=devc)
        step = 10_000_000
        for s in range(0, coords.shape[1], step):
            c = coords[:, s:s + step]
            p = vals[s:s + step].double()[:, None]
            for m in range(3):
                if m != mode:
                    p = p * U[m][c[m]].double()
            want.index_add_(0, c[mode], p)
        assert torch.allclose(got.double(), want, rtol=2e-5, atol=0), mode
        del want
        rows = rng.choice(shape[mode], 16, replace=False)
        for i in rows:
            sel = torch.nonzero(coords[mode] == int(i)).reshape(-1)  # C order = stream order inside the row
            start = int((coords[mode] < int(i)).sum())
            c = coords[:, sel]
            p = MO.products(vals[sel].cpu().numpy(),
                            [U[m][c[m]].cpu().numpy() for m in range(3) if m != mode], np.float32)
            assert MO.same_bits(got[int(i)].cpu().numpy(), MO.row_result(p, start, ch, np.float32)), (mode, i)
