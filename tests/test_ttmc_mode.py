"""ttmc_mode(X, factors, mode): mode-n TTMc (tensor times matrix chain) of sparse tensors of order 2..8.

Parity with float64 dense einsum and with the reference's unfused broadcast expression (golden fixture), bit equality
with a CPU restatement of the fixed order of operations (tests/_tensor_order.py) on both column paths, the diagonal
identity with mttkrp_mode, edge cases, the width limit, and a small HOOI that reconstructs a tensor of exact multilinear
rank.  Determinism, the mode-stream cache shared with mttkrp_mode, the int64 index path, factor layouts and the shared
argument errors are in tests/test_tensor_ops_contract.py.  Every body runs on the NumPy mock without a GPU and on the
CUDA kernels with `-m gpu`."""
import numpy as np
import pytest

import _tensor_order as TO
from _api import dec, sp  # noqa: F401
from _golden import load
from _tensor_cases import (LAYOUTS, SHAPES, chunk, chunk_structured, dev, full_size_tensor, host, layout_id,
                           plant_specials, rand_tensor, ttmc_einsum as einsum_ref)

TOL = {"float32": 2e-5, "float64": 1e-12}
same_bits = TO.same_bits


def factors(rng, shape, ranks, dtype, signed=False):
    if signed:
        return [rng.standard_normal((s, r)).astype(dtype) for s, r in zip(shape, ranks)]
    return [rng.random((s, r)).astype(dtype) + np.asarray(0.05, dtype) for s, r in zip(shape, ranks)]


def order_ref(sp, X, U, mode, dtype):
    c = X.tocoo() if X.format == "gcxs" else X
    return TO.ttmc_mode(c.coords, c.data, U, mode, X.shape[mode], chunk(sp), dtype)


def width(U, mode):
    return int(np.prod([u.shape[1] for m, u in enumerate(U) if m != mode]))


# per order: unequal ranks (R_last often not a multiple of 16 B / itemsize), and a set whose W spans several column
# tiles of both paths
RANKS = {2: [(3, 5), (70, 150)], 3: [(3, 4, 2), (12, 16, 9)], 4: [(2, 3, 5, 4), (4, 6, 8, 5)],
         5: [(2, 3, 1, 4, 2), (3, 4, 2, 5, 4)], 6: [(2, 1, 3, 2, 2, 3), (3, 2, 4, 2, 3, 4)],
         8: [(2, 1, 2, 3, 1, 2, 2, 1), (2, 3, 2, 2, 3, 2, 2, 4)]}


@pytest.mark.parametrize("rset", [0, 1], ids=["small", "wide"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("order", [2, 3, 4, 5, 6, 8])
@pytest.mark.parametrize("layout", range(len(LAYOUTS)), ids=layout_id)
def test_fp64_parity_every_mode(sp, order, dtype, rset, layout):
    shape, ranks = SHAPES[order], RANKS[order][rset]
    fmt, ca = LAYOUTS[layout]
    if ca == "last":
        ca = (order - 1,)
    if ca == (0, 1) and order == 2:
        pytest.skip("an order-2 tensor cannot compress two axes")
    rng = np.random.default_rng(100 * order + rset)
    X = rand_tensor(sp, rng, shape, max(int(np.prod(shape)) // 4, 5), dtype, fmt, ca)
    U = factors(rng, shape, ranks, dtype)
    for mode in range(order):
        got = sp.ttmc_mode(X, U, mode)
        assert isinstance(got, np.ndarray) and got.dtype == np.dtype(dtype)
        assert got.shape == (shape[mode], width(U, mode))
        np.testing.assert_allclose(got, einsum_ref(X, U, mode), rtol=TOL[dtype], atol=0)


GOLDEN = [c for c in load("ttmc_mode_api") if c["op"] == "ttmc_mode"]


@pytest.mark.parametrize("c", GOLDEN, ids=lambda c: f"{c['dtype']}-order{c['order']}-mode{c['mode']}")
@pytest.mark.parametrize("fmt", ["coo", "gcxs"])
def test_golden_parity(sp, c, fmt):
    X = dec(sp, c, "X_", fmt)
    U = [np.array(c.arr[f"U{m}"]) for m in range(int(c["order"]))]
    mode = int(c["mode"])
    U[mode] = None
    got = sp.ttmc_mode(X, U, mode)
    w = c.sub("out_")
    want = sp.COO(np.array(w["coords"]), np.array(w["data"]), shape=tuple(int(s) for s in w["shape"])).todense()
    assert want.ndim == X.ndim  # (I_mode, R_a, R_b, ...)
    tol = TOL[c["dtype"]]
    assert got.dtype == want.dtype
    np.testing.assert_allclose(got, want.reshape(X.shape[mode], -1), rtol=tol, atol=tol)


def special_factors(rng, shape, ranks, dtype):
    """Signed normal factors with +-inf, NaN and -0.0 planted in each."""
    return plant_specials(rng, factors(rng, shape, ranks, dtype, signed=True))


# (ranks, what they exercise): f32 vector packs hold 4 columns and f64 ones 2, so R_last = 8 takes the vector path in
# both dtypes, R_last = 5 or 3 the scalar path; W = 96..160 spans several tiles of either
@pytest.mark.parametrize("ranks", [(3, 5, 8), (6, 8, 3), (4, 4, 4), (1, 7, 2)])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_exact_order(sp, dtype, ranks):
    rng = np.random.default_rng(sum(ranks))
    X, _ = chunk_structured(sp, rng, dtype, 1)
    U = special_factors(rng, X.shape, ranks, dtype)
    for mode in range(3):
        got = sp.ttmc_mode(X, U, mode)
        assert same_bits(got, order_ref(sp, X, U, mode, dtype)), mode


def test_exact_order_skewed_mode_order4(sp):
    """A mode with 3 slices of thousands of entries each (every slice spans many chunks), order 4."""
    rng = np.random.default_rng(7)
    X = rand_tensor(sp, rng, (20, 15, 3, 14), 6000, "float32", signed=True)
    U = factors(rng, X.shape, (3, 2, 5, 4), "float32", signed=True)
    for mode in (2, -1, 0):
        assert same_bits(sp.ttmc_mode(X, U, mode), order_ref(sp, X, U, mode % 4, "float32"))


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_vector_and_scalar_paths_agree(sp, dtype):
    """The restatement's bits through aligned contiguous factors (vector path where R_last fills whole 16-byte packs)
    and through device views one column into a wider buffer (unaligned rows: scalar path); a float64 factor promotes
    the result.  Fortran-ordered, transposed and mixed host / device factors are in test_tensor_ops_contract.py."""
    rng = np.random.default_rng(31)
    X = rand_tensor(sp, rng, (40, 30, 20), 2500, dtype, signed=True)
    U = special_factors(rng, X.shape, (5, 6, 8), dtype)
    wide = [dev(sp, np.concatenate([np.zeros((u.shape[0], 1), dtype), u], axis=1))[:, 1:] for u in U]
    for m in range(3):
        want = order_ref(sp, X, U, m, dtype)
        assert same_bits(sp.ttmc_mode(X, U, m), want), m
        assert same_bits(host(sp.ttmc_mode(X, wide, m)), want), m
    U64 = [U[0].astype(np.float64), U[1], U[2]]
    got = sp.ttmc_mode(X, U64, 1)
    assert got.dtype == np.float64
    assert same_bits(got, order_ref(sp, X, U64, 1, "float64"))


def diagonal(out, I_, R, n_other):
    return out.reshape((I_,) + (R,) * n_other)[(slice(None),) + (np.arange(R),) * n_other]


@pytest.mark.parametrize("R", [3, 8])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("order", [2, 3, 4, 5])
def test_diagonal_equals_mttkrp_mode(sp, order, dtype, R):
    shape = SHAPES[order]
    rng = np.random.default_rng(40 + order + R)
    X = rand_tensor(sp, rng, shape, max(int(np.prod(shape)) // 3, 5), dtype, signed=True)
    U = factors(rng, shape, (R,) * order, dtype, signed=True)
    for mode in range(order):
        t = sp.ttmc_mode(X, U, mode)
        k = sp.mttkrp_mode(X, U, mode)
        assert same_bits(diagonal(t, shape[mode], R, order - 1), k), mode
        if order == 2:
            assert same_bits(t, k)


def test_edge_cases(sp):
    rng = np.random.default_rng(17)
    U = [rng.random((s, r)) for s, r in ((5, 2), (6, 3), (7, 4))]
    empty = sp.COO(np.zeros((3, 0), np.int64), np.zeros(0), shape=(5, 6, 7))
    for m in range(3):
        got = sp.ttmc_mode(empty, U, m)
        assert got.shape == (U[m].shape[0], width(U, m)) and not got.any() and not np.signbit(got).any()
    X = rand_tensor(sp, rng, (5, 6, 7), 60, "float64")
    U0 = [U[0], np.zeros((6, 0)), U[2]]
    assert sp.ttmc_mode(X, U0, 0).shape == (5, 0)
    assert sp.ttmc_mode(X, U0, 2).shape == (7, 0)
    assert sp.ttmc_mode(X, U0, 1).shape == (6, 8)  # the zero-rank factor is the one not read
    sparse_rows = rand_tensor(sp, rng, (500, 4, 3), 20, "float64")  # most rows empty
    Us = [None, rng.random((4, 2)), rng.random((3, 3))]
    got = sp.ttmc_mode(sparse_rows, Us, 0)
    np.testing.assert_allclose(got, einsum_ref(sparse_rows, [np.zeros((500, 1))] + Us[1:], 0), rtol=1e-12)
    assert (got == 0).sum() >= 480 * 6 and not np.signbit(got[got == 0]).any()
    assert same_bits(sp.ttmc_mode(X, U, -1), sp.ttmc_mode(X, U, 2))
    G = X.asformat("gcxs", compressed_axes=(2,))
    assert same_bits(sp.ttmc_mode(G, U, 1), sp.ttmc_mode(X, U, 1))


def test_errors(sp):
    rng = np.random.default_rng(23)
    X = rand_tensor(sp, rng, (5, 6, 7), 40, "float64")
    limit = sp._kernels.ttmc_mode_max_width()
    assert limit == 65535 * 32
    big = [None, np.ones((6, 1449)), np.ones((7, 1448))]  # W = 2,098,152
    assert 1449 * 1448 > limit
    with pytest.raises(ValueError, match="exceed the limit"):
        sp.ttmc_mode(X, big, 0)


def test_small_hooi_reconstructs_exact_multilinear_rank(sp):
    """A float64 tensor of multilinear rank (2, 3, 2), every entry stored: two HOOI sweeps (ttmc_mode + SVD) from random
    orthonormal factors recover it to 1e-10.  Uses the documented unfolding: Y_n = ttmc_mode(X, U, n) is (I_n, W), its
    leading left singular vectors are U_n, and U_n^T Y_n is the core unfolded in C order over the other modes."""
    rng = np.random.default_rng(2024)
    shape, ranks = (8, 9, 7), (2, 3, 2)
    core = rng.standard_normal(ranks)
    A = [np.linalg.qr(rng.standard_normal((s, r)))[0] for s, r in zip(shape, ranks)]
    dense = np.einsum("abc,ia,jb,kc->ijk", core, *A)
    coords = np.stack(np.unravel_index(np.arange(dense.size), shape)).astype(np.int64)
    X = sp.COO(coords, dense.reshape(-1), shape=shape, has_duplicates=False, sorted=True)
    assert X.nnz == dense.size
    U = [np.linalg.qr(rng.standard_normal((s, r)))[0] for s, r in zip(shape, ranks)]
    for _ in range(2):
        for n in range(3):
            Y = sp.ttmc_mode(X, U, n)
            U[n] = np.linalg.svd(Y, full_matrices=False)[0][:, : ranks[n]]
    G = (U[2].T @ sp.ttmc_mode(X, U, 2)).reshape(ranks[2], ranks[0], ranks[1])  # (r_c, r_a, r_b)
    rec = np.einsum("cab,ia,jb,kc->ijk", G, *U)
    assert np.linalg.norm(rec - dense) <= 1e-10 * np.linalg.norm(dense)


@pytest.mark.gpu
def test_full_size_each_mode():
    """(1e6, 1e6, 100) with 1e8 uniform entries, R_m = 16 (W = 256), f32: every row within 2e-5 of a float64
    restatement on the device, computed in blocks of 16 columns; 4 sampled rows per mode bit-equal to the CPU
    restatement of the order."""
    import torch

    import sparse_b200 as spm

    X, coords, vals, g = full_size_tensor(78)
    shape, R = X.shape, 16
    U = [torch.rand((s, R), generator=g, device=coords.device) + 0.05 for s in shape]
    ch = spm._kernels.mttkrp_mode_chunk()
    rng = np.random.default_rng(6)
    for mode in range(3):
        a, b = [m for m in range(3) if m != mode]
        got = spm.ttmc_mode(X, U, mode)
        assert got.shape == (shape[mode], R * R)
        step = 10_000_000
        for ra in range(R):  # columns ra * R .. ra * R + R - 1
            want = torch.zeros((shape[mode], R), dtype=torch.float64, device=coords.device)
            for s in range(0, coords.shape[1], step):
                c = coords[:, s:s + step]
                p = vals[s:s + step].double() * U[a][c[a], ra].double()
                want.index_add_(0, c[mode], p[:, None] * U[b][c[b]].double())
            assert torch.allclose(got[:, ra * R:(ra + 1) * R].double(), want, rtol=2e-5, atol=0), (mode, ra)
        del want
        rows = rng.choice(shape[mode], 4, replace=False)
        assert TO.sampled_rows_exact(got, coords, vals, U, mode, rows, ch, kron=True), mode
        del got
