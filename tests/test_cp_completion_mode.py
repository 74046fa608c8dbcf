"""cp_completion_mode(X, factors, mode, reg): the row-wise regularised least-squares ALS update of CP tensor completion.

Parity with a float64 NumPy solve of (H_i^T H_i + reg I) x = H_i^T v_i and with the reference's unfused Gram and
right-hand-side expressions (golden fixture), bit equality with a CPU restatement of the fixed order of operations
(tests/_tensor_order.py) at chunk edges, on both gather paths and with special values, the identities with
mttkrp_mode, edge cases, errors of `reg` and the rank limit, and ALS convergence.  The mode-stream cache, determinism,
both index widths, factor layouts and the argument errors shared with the other sparse-tensor ops are in
tests/test_tensor_ops_contract.py.  Every body runs on the NumPy mock without a GPU and on the CUDA kernels with
`-m gpu`."""
import numpy as np
import pytest

import _tensor_order as TO
from _api import dec, sp  # noqa: F401
from _golden import load
from _tensor_cases import LAYOUTS, SHAPES, chunk, chunk_structured, dev, edge_rows, host, rand_tensor

TOL = {"float32": 2e-3, "float64": 1e-9}
same_bits = TO.same_bits


def stored(X):
    c = X.tocoo() if X.format == "gcxs" else X
    return np.asarray(c.coords, np.int64), np.asarray(c.data)


def lstsq_ref(X, U, mode, reg, rows=None):
    """float64: row i solves (H_i^T H_i + reg I) x = H_i^T v_i over X's stored entries in row i (`rows`: only
    those, the others 0)."""
    coords, vals = stored(X)
    R = next(np.shape(u)[1] for m, u in enumerate(U) if m != mode)
    h = np.ones((len(vals), R))
    for m in range(X.ndim):
        if m != mode:
            h = h * np.asarray(U[m], np.float64)[coords[m]]
    n = X.shape[mode]
    order = np.argsort(coords[mode], kind="stable")
    h, v, bounds = h[order], vals[order].astype(np.float64), np.searchsorted(coords[mode][order], np.arange(n + 1))
    G = np.stack([h[bounds[i]:bounds[i + 1]].T @ h[bounds[i]:bounds[i + 1]] for i in range(n)])
    b = np.stack([h[bounds[i]:bounds[i + 1]].T @ v[bounds[i]:bounds[i + 1]] for i in range(n)])
    rows = np.arange(n) if rows is None else np.asarray(rows)
    out = np.zeros((n, R))
    out[rows] = np.linalg.solve(G[rows] + reg * np.eye(R), b[rows][..., None])[..., 0]
    return out


def order_ref(sp, X, U, mode, dtype, regs):
    """The restatement's result for each reg in `regs` (the sums once, a solve per reg)."""
    coords, vals = stored(X)
    Gu, b = TO.systems(coords, vals, U, mode, X.shape[mode], chunk(sp), dtype)
    return [TO.solve(Gu, b, reg, dtype) for reg in regs]


def close(got, want, dtype):
    tol = TOL[np.dtype(dtype).name]
    np.testing.assert_allclose(got, want, rtol=tol, atol=tol * max(np.abs(want).max(), 1.0))


# f32 packs hold 4 columns and f64 ones 2: R = 1, 3 and 37 gather scalars, 4 (f64), 16 and 64 16-byte packs.  Each
# (order, R) pair takes one of the four storage layouts, in turn, so every order meets every layout.
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("order", sorted(SHAPES))
def test_fp64_parity_every_mode(sp, order, dtype):
    shape = SHAPES[order]
    for k, R in enumerate([1, 3, 4, 16, 37, 64]):
        fmt, ca = LAYOUTS[(k + order) % len(LAYOUTS)]
        if ca == (0, 1) and order == 2:
            fmt, ca = "gcxs", (1,)  # an order-2 tensor cannot compress two axes
        rng = np.random.default_rng(10 * order + R)
        X = rand_tensor(sp, rng, shape, max(int(np.prod(shape)) // 4, 5), dtype, fmt,
                        (order - 1,) if ca == "last" else ca)
        U = [rng.random((s, R)).astype(dtype) + np.asarray(0.05, dtype) for s in shape]
        reg = 1.0  # every system well conditioned, empty rows included
        for mode in range(order):
            got = sp.cp_completion_mode(X, U, mode, reg)
            assert isinstance(got, np.ndarray) and got.dtype == np.dtype(dtype) and got.shape == (shape[mode], R)
            close(got, lstsq_ref(X, U, mode, reg), dtype)


GOLDEN = [c for c in load("cp_completion_api") if c["op"] == "cp_completion_mode"]


@pytest.mark.parametrize("c", GOLDEN, ids=lambda c: f"{c['dtype']}-order{c['order']}-R{c['R']}-mode{c['mode']}")
def test_golden_parity(sp, c):
    N, R, mode, reg = int(c["order"]), int(c["R"]), int(c["mode"]), 0.5
    X = dec(sp, c, "X_", "gcxs" if mode % 2 else "coo")
    U = [np.array(c.arr[f"U{m}"]) for m in range(N)]
    U[mode] = None
    got = sp.cp_completion_mode(X, U, mode, reg)
    G, b = (c.sub(p) for p in ("G_", "b_"))
    G = sp.COO(np.array(G["coords"]), np.array(G["data"]), shape=tuple(int(s) for s in G["shape"])).todense()
    b = sp.COO(np.array(b["coords"]), np.array(b["data"]), shape=tuple(int(s) for s in b["shape"])).todense()
    want = np.linalg.solve(G.astype(np.float64) + reg * np.eye(R), b.astype(np.float64)[..., None])[..., 0]
    assert got.dtype == np.dtype(c["dtype"]) and got.shape == (X.shape[mode], R)
    close(got, want, c["dtype"])


@pytest.mark.parametrize("R", [1, 5, 8, 32])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_exact_order(sp, dtype, R):
    rng = np.random.default_rng(R)
    X, U = edge_rows(sp, rng, dtype, R)
    Y, V = chunk_structured(sp, rng, dtype, R)
    # R = 32 (four accumulator slots per thread) on the chunk-edge rows only, to keep the restatement quick
    for T, W in ((X, U), (Y, V)) if R <= 8 else ((X, U),):
        for mode in range(3):
            regs = (0.25, 0.0)
            for reg, want in zip(regs, order_ref(sp, T, W, mode, dtype, regs)):
                assert same_bits(sp.cp_completion_mode(T, W, mode, reg), want), (mode, reg)
    got = sp.cp_completion_mode(X, U, 0, 0.25)
    assert (~np.isfinite(got[:2])).any(axis=1).all() and np.isnan(got[1]).all() and np.isfinite(got[2:]).all()
    # device factors that are column-sliced views (unaligned rows): the scalar path, the same bits
    wide = [dev(sp, np.concatenate([np.zeros((u.shape[0], 1), dtype), u], axis=1))[:, 1:] for u in U]
    for mode in range(3):
        want = sp.cp_completion_mode(X, U, mode, 0.25)
        assert same_bits(host(sp.cp_completion_mode(X, wide, mode, 0.25)), want)
        assert same_bits(host(sp.cp_completion_mode(X, [U[0], wide[1], dev(sp, U[2])], mode, 0.25)), want)


def test_exact_order_row_over_hundreds_of_chunks(sp):
    """A mode of extent 2: each of its rows spans about 250 chunks."""
    rng = np.random.default_rng(4)
    X = rand_tensor(sp, rng, (500, 500, 2), 256_000, "float32", signed=True)
    U = [rng.standard_normal((s, 6)).astype(np.float32) for s in X.shape]
    assert same_bits(sp.cp_completion_mode(X, U, 2, 0.5), order_ref(sp, X, U, 2, "float32", [0.5])[0])


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_rhs_is_mttkrp_mode_and_fully_observed_is_cp_als(sp, dtype):
    rng = np.random.default_rng(5)
    shape, R, reg = (9, 8, 7), 5, 0.3
    dense = rng.standard_normal(shape).astype(dtype)
    dense[rng.random(shape) < 0.1] = 0  # stored zeros: every position is observed
    coords = np.stack(np.unravel_index(np.arange(dense.size), shape))
    X = sp.COO(coords, dense.reshape(-1), shape=shape, has_duplicates=False, sorted=True)
    assert X.nnz == dense.size
    U = [rng.standard_normal((s, R)).astype(dtype) for s in shape]
    for mode in range(3):
        # the restatement's right-hand side is mttkrp_mode bit for bit (step 3 of the order)
        _, b = TO.systems(coords, dense.reshape(-1), U, mode, shape[mode], chunk(sp), dtype)
        assert same_bits(b, sp.mttkrp_mode(X, U, mode))
        # fully observed: the CP-ALS update mttkrp_mode @ inv(hadamard of U_m^T U_m + reg I)
        V = np.ones((R, R))
        for m in range(3):
            if m != mode:
                V = V * (U[m].astype(np.float64).T @ U[m].astype(np.float64))
        want = sp.mttkrp_mode(X, U, mode).astype(np.float64) @ np.linalg.inv(V + reg * np.eye(R))
        close(sp.cp_completion_mode(X, U, mode, reg), want, dtype)


def test_stored_zeros_are_observations(sp):
    rng = np.random.default_rng(6)
    X = rand_tensor(sp, rng, (12, 10, 8), 400, "float64")
    vals = np.array(X.data)
    vals[::3] = 0.0
    with_zeros = sp.COO(X.coords, vals, shape=X.shape, has_duplicates=False, sorted=True)
    pruned = sp.COO(X.coords, vals, shape=X.shape, has_duplicates=False, sorted=True, prune=True)
    assert with_zeros.nnz == X.nnz and pruned.nnz < X.nnz
    U = [rng.random((s, 4)) + 0.05 for s in X.shape]
    for mode in range(3):
        a = sp.cp_completion_mode(with_zeros, U, mode, 0.1)
        b = sp.cp_completion_mode(pruned, U, mode, 0.1)
        np.testing.assert_allclose(a, lstsq_ref(with_zeros, U, mode, 0.1), rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(b, lstsq_ref(pruned, U, mode, 0.1), rtol=1e-9, atol=1e-9)
        assert not np.allclose(a, b)


def test_empty_and_rank_deficient_rows(sp):
    rng = np.random.default_rng(7)
    shape, R = (8, 6, 5), 3
    coords = [(i, j, k) for i in (0, 1, 3, 4, 6) for j in range(6) for k in range(5) if rng.random() < 0.7]
    coords += [(2, j, 0) for j in range(6)]  # row 2 sees only k = 0, where U_2 has a zero column
    coords = np.array(sorted(coords)).T
    X = sp.COO(coords, rng.standard_normal(coords.shape[1]), shape=shape, has_duplicates=False, sorted=True)
    U = [rng.random((s, R)) + 0.1 for s in shape]
    U[2][0, 2] = 0.0
    got = sp.cp_completion_mode(X, U, 0, 0.0)
    want = order_ref(sp, X, U, 0, "float64", [0.0])[0]
    assert same_bits(got, want)
    empty = [5, 7]
    assert np.isnan(got[empty]).all() and np.isnan(got[2]).all()
    live = [0, 1, 3, 4, 6]
    np.testing.assert_allclose(got[live], lstsq_ref(X, U, 0, 0.0, live)[live], rtol=1e-8)
    pos = sp.cp_completion_mode(X, U, 0, 0.5)
    assert np.all(pos[empty] == 0) and not np.signbit(pos[empty]).any() and np.isfinite(pos).all()


def test_edge_cases(sp):
    rng = np.random.default_rng(8)
    U = [rng.random((s, 4)) for s in (5, 6, 7)]
    empty = sp.COO(np.zeros((3, 0), np.int64), np.zeros(0), shape=(5, 6, 7))
    for m in range(3):
        got = sp.cp_completion_mode(empty, U, m, 0.5)
        assert got.shape == (U[m].shape[0], 4) and not got.any() and not np.signbit(got).any()
        assert np.isnan(sp.cp_completion_mode(empty, U, m, 0)).all()
    X = rand_tensor(sp, rng, (5, 6, 7), 60, "float64")
    assert sp.cp_completion_mode(X, [np.zeros((s, 0)) for s in X.shape], 1, 1.0).shape == (6, 0)
    zero_ext = sp.COO(np.zeros((3, 0), np.int64), np.zeros(0), shape=(5, 0, 7))
    got = sp.cp_completion_mode(zero_ext, [np.ones((5, 2)), np.ones((0, 2)), np.ones((7, 2))], 1, 1.0)
    assert got.shape == (0, 2)
    got = sp.cp_completion_mode(X, [U[0], None, U[2]], 1, np.float32(0.5))
    assert same_bits(got, sp.cp_completion_mode(X, U, -2, 0.5))


def test_errors(sp, monkeypatch):
    rng = np.random.default_rng(11)
    X = rand_tensor(sp, rng, (5, 6, 7), 40, "float64")
    U = [rng.random((s, 3)) for s in X.shape]
    for bad in (np.nan, np.inf, -np.inf, -1e-3):
        with pytest.raises(ValueError, match="reg"):
            sp.cp_completion_mode(X, U, 0, bad)
    with pytest.raises(ValueError, match="reg"):  # finite in float64, inf once cast to float32
        sp.cp_completion_mode(X.astype(np.float32), [u.astype(np.float32) for u in U], 0, 1e39)
    for bad in (None, "1", 1j, True):
        with pytest.raises(TypeError):
            sp.cp_completion_mode(X, U, 0, bad)

    # R above the limit: refused before the mode stream or the result is allocated
    def no_alloc(*a, **k):
        raise AssertionError("allocated before the rank check")

    limit = sp._kernels.cp_completion_max_rank()
    assert limit == 64
    monkeypatch.setattr(sp._fused, "_mode_stream", no_alloc)
    monkeypatch.setattr(sp._kernels, "full", no_alloc)
    with pytest.raises(ValueError, match="exceeds the limit"):
        sp.cp_completion_mode(X, [rng.random((s, limit + 1)) for s in X.shape], 0, 1.0)


def als(sp, X, U, reg, sweeps):
    """ALS sweeps; yields the regularised training objective after each sweep (tttp for the fit term)."""
    P = sp.COO(X.coords, np.ones(X.nnz, X.dtype), shape=X.shape, has_duplicates=False, sorted=True)
    for _ in range(sweeps):
        for n in range(X.ndim):
            U[n] = sp.cp_completion_mode(X, U, n, reg)
        resid = sp.tttp(P, U) - X
        r = np.asarray(resid.data, np.float64)
        yield 0.5 * float(r @ r) + 0.5 * reg * sum(float((np.asarray(host(u), np.float64) ** 2).sum()) for u in U)


def model_at(U, coords):
    return np.prod([np.asarray(host(u), np.float64)[c] for u, c in zip(U, coords)], axis=0).sum(1)


def test_als_completion_converges(sp):
    """A rank-4 (60, 50, 40) tensor from 30 % of its entries: held-out relative RMSE below 1e-6 within 30 sweeps, and
    the regularised objective never increases beyond rounding."""
    rng = np.random.default_rng(12)
    shape, R, reg = (60, 50, 40), 4, 1e-12
    truth = [rng.standard_normal((s, R)) for s in shape]
    lin = rng.permutation(int(np.prod(shape)))
    n_obs = int(0.3 * lin.size)
    obs, held = np.sort(lin[:n_obs]), lin[n_obs:n_obs + 5000]
    oc = np.stack(np.unravel_index(obs, shape))
    X = sp.COO(oc, model_at(truth, oc), shape=shape, has_duplicates=False, sorted=True)
    U = [rng.standard_normal((s, R)) for s in shape]
    hc = np.stack(np.unravel_index(held, shape))
    want = model_at(truth, hc)
    losses = []
    for loss in als(sp, X, U, reg, 30):
        losses.append(loss)
        err = np.sqrt(np.mean((model_at(U, hc) - want) ** 2) / np.mean(want ** 2))
        if err < 1e-6:
            break
    assert err < 1e-6, (len(losses), err)
    for a, b in zip(losses, losses[1:]):
        assert b <= a * (1 + 1e-9) + 1e-18


@pytest.mark.gpu
def test_als_completion_large_f32():
    """About 1e7 observed entries of a rank-4 (2000, 1500, 1000) float32 tensor: ALS reaches a held-out relative RMSE
    below 2e-2 within 25 sweeps, and sampled rows of a call match a float64 solve and the CPU restatement bit for bit."""
    import torch

    import sparse_b200 as spm

    devc = torch.device("cuda")
    shape, R, reg, nnz = (2000, 1500, 1000), 4, 1e-6, 10_000_000
    g = torch.Generator(device=devc).manual_seed(5)
    truth = [torch.randn((s, R), generator=g, device=devc) for s in shape]
    lin = torch.unique(torch.randint(0, shape[0] * shape[1] * shape[2], (nnz,), generator=g, device=devc))
    coords = torch.stack(torch.unravel_index(lin, shape))
    vals = (truth[0][coords[0]] * truth[1][coords[1]] * truth[2][coords[2]]).sum(1)
    X = spm.COO(coords, vals, shape=shape, has_duplicates=False, sorted=True)
    U = [torch.randn((s, R), generator=g, device=devc) for s in shape]
    hc = torch.stack([torch.randint(0, s, (20000,), generator=g, device=devc) for s in shape])

    def model(F):
        return (F[0][hc[0]].double() * F[1][hc[1]].double() * F[2][hc[2]].double()).sum(1)

    want = model(truth)
    for _ in range(25):
        for n in range(3):
            U[n] = spm.cp_completion_mode(X, U, n, reg)
        err = float(((model(U) - want) ** 2).mean().sqrt() / (want ** 2).mean().sqrt())
        if err < 2e-2:
            break
    assert err < 2e-2, err
    # one more call at mode 1: sampled rows against a float64 solve and the restatement
    got = spm.cp_completion_mode(X, U, 1, reg)
    (sc, sv) = X._mode_streams[(1, True)]  # the cached mode-1 stream the call read
    rows = np.random.default_rng(3).choice(shape[1], 16, replace=False)
    ends = torch.from_numpy(np.stack([rows, rows + 1])).to(devc).to(sc[1].dtype)
    bounds = torch.searchsorted(sc[1], ends).cpu().numpy()
    Uh = [u.cpu().numpy() for u in U]
    Gu, b = [], []
    for lo, hi in zip(bounds[0], bounds[1]):
        c = [x[lo:hi].long().cpu().numpy() for x in sc]
        v = sv[lo:hi].cpu().numpy()
        gathered = [Uh[0][c[0]], Uh[2][c[2]]]
        h, p = TO.products(None, gathered, np.float32), TO.products(v, gathered, np.float32)
        gu, bb = TO.row_system(h, p, int(lo), 512, np.float32)
        Gu.append(gu)
        b.append(bb)
        H = Uh[0][c[0]].astype(np.float64) * Uh[2][c[2]].astype(np.float64)
        ref = np.linalg.solve(H.T @ H + np.float64(np.float32(reg)) * np.eye(R), H.T @ v.astype(np.float64))
        np.testing.assert_allclose(got[int(c[1][0])].cpu().numpy(), ref, rtol=1e-2, atol=1e-2 * np.abs(ref).max())
    want_rows = TO.solve(np.array(Gu), np.array(b), np.float32(reg), np.float32)
    assert same_bits(got[torch.from_numpy(rows).to(devc)].cpu().numpy(), want_rows)

