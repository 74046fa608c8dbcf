"""mttkrp_mode(X, factors, mode): mode-n MTTKRP of sparse tensors of order 2..8.

Parity with float64 dense einsum and with the reference's unfused broadcast expression (golden fixtures), bit
equality with a CPU restatement of the fixed order of operations (tests/_tensor_order.py), edge cases, and the full-size
workload on the GPU.  Determinism, the mode-stream cache, factor layouts and errors are shared with the other
sparse-tensor ops (tests/test_tensor_ops_contract.py).  Every body runs on the NumPy mock without a GPU and on the CUDA
kernels with `-m gpu`."""
import numpy as np
import pytest

import _tensor_order as TO
from _api import dec, sp  # noqa: F401
from _golden import load
from _tensor_cases import (LAYOUTS, SHAPES, chunk, chunk_structured, full_size_tensor, layout_id, rand_tensor,
                           mttkrp_einsum as einsum_ref)

TOL = {"float32": 2e-5, "float64": 1e-12}
same_bits = TO.same_bits


def order_ref(sp, X, factors, mode, dtype):
    c = X.tocoo() if X.format == "gcxs" else X
    return TO.mttkrp_mode(c.coords, c.data, factors, mode, X.shape[mode], chunk(sp), dtype)


@pytest.mark.parametrize("R", [1, 3, 8, 32, 33, 100, 256])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("order", [2, 3, 4, 5, 8])
@pytest.mark.parametrize("layout", range(len(LAYOUTS)), ids=layout_id)
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


@pytest.mark.parametrize("R", [1, 5, 8, 32])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_exact_order(sp, dtype, R):
    X, U = chunk_structured(sp, np.random.default_rng(R), dtype, R)
    for mode in range(3):
        got = sp.mttkrp_mode(X, U, mode)
        assert same_bits(got, order_ref(sp, X, U, mode, dtype)), mode


def test_exact_order_skewed_mode(sp):
    """A mode with 3 slices of thousands of entries each: every slice spans many chunks."""
    rng = np.random.default_rng(7)
    X = rand_tensor(sp, rng, (60, 50, 3), 6000, "float32", signed=True)
    U = [rng.standard_normal((s, 8)).astype(np.float32) for s in X.shape]
    for mode in (2, -1, 0):
        assert same_bits(sp.mttkrp_mode(X, U, mode), order_ref(sp, X, U, mode % 3, "float32"))


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
    assert same_bits(sp.mttkrp_mode(X, U, -1), sp.mttkrp_mode(X, U, 2))


@pytest.mark.gpu
def test_full_size_each_mode():
    """(1e6, 1e6, 100) with 1e8 uniform entries, R = 32, f32: every row within 2e-5 of a float64 restatement on the
    device; 16 sampled rows per mode (two of the 100 slices of mode 2) bit-equal to the CPU order restatement."""
    import torch

    import sparse_b200 as spm

    X, coords, vals, g = full_size_tensor(77)
    shape, R = X.shape, 32
    U = [torch.rand((s, R), generator=g, device=coords.device) + 0.05 for s in shape]
    ch = spm._kernels.mttkrp_mode_chunk()
    rng = np.random.default_rng(5)
    for mode in range(3):
        got = spm.mttkrp_mode(X, U, mode)
        want = torch.zeros((shape[mode], R), dtype=torch.float64, device=coords.device)
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
        assert TO.sampled_rows_exact(got, coords, vals, U, mode, rows, ch, kron=False), mode
