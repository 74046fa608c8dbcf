"""K1p tiled passes (column tile x K panel, spmm_panel.cu): bit-identical to the one-pass kernel and the oracle.

Small shapes are pushed through many panels (explicit n_panels) and every tile width (spmm_set_tiling), so that rows
split into many runs, tiles end inside N, and partial sums go through C many times."""
import numpy as np
import pytest

import oracle
from _util import bits_equal, rand_csr, rand_dense

pytestmark = pytest.mark.gpu


@pytest.fixture
def tiling():
    from sparse_b200 import _kernels as Kn

    yield Kn.spmm_set_tiling
    Kn.spmm_set_tiling(0, 0)


def _csr_with_edge_rows(rng, M, K, dtype):
    """Sorted rows: random rows plus empty rows, rows inside one narrow column range, duplicate columns, -0.0 values."""
    rows = []
    for r in range(M):
        kind = r % 7
        if kind == 0:
            cols = np.zeros(0, np.int64)
        elif kind == 1:  # wholly inside one panel
            lo = rng.integers(0, K - 8)
            cols = np.sort(rng.integers(lo, lo + 8, rng.integers(1, 12)))
        elif kind == 2:  # duplicates, some straddling panel boundaries
            cols = np.sort(np.repeat(rng.integers(0, K, 6), rng.integers(1, 4, 6)))
        elif kind == 3:  # long row across every panel
            cols = np.sort(rng.choice(K, min(K, 300), replace=False))
        else:
            cols = np.sort(rng.choice(K, rng.integers(1, 40), replace=False))
        rows.append(cols)
    indptr = np.zeros(M + 1, np.int64)
    np.cumsum([len(c) for c in rows], out=indptr[1:])
    indices = np.concatenate(rows).astype(np.int64)
    data = (rng.random(len(indices)) * 2 - 1).astype(dtype)
    data[::5] = -0.0
    return data, indices, indptr


def _run(data, indices, indptr, b, K, N, idt, n_panels, bt=None, out=None):
    from sparse_b200 import _device as D
    from sparse_b200 import _kernels as Kn

    M = len(indptr) - 1
    bd = D.upload(b) if bt is None else bt
    got = Kn.spmm_csr_dense(D.upload(data), D.upload(indices.astype(idt)), D.upload(indptr.astype(idt)), bd, M, K, N,
                            out=out, n_panels=n_panels)
    return D.download(got)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("idt", [np.int32, np.int64])
@pytest.mark.parametrize("N", [128, 256, 64, 36, 8])
@pytest.mark.parametrize("tile_bytes,n_panels", [(64, 13), (128, 2), (128, 31), (256, 5)])
def test_tiled_passes_match_oracle(tiling, dtype, idt, N, tile_bytes, n_panels):
    rng = np.random.default_rng(N * 1000 + n_panels)
    M, K = 700, 2000
    data, indices, indptr = _csr_with_edge_rows(rng, M, K, dtype)
    b = rand_dense(rng, (K, N), dtype)
    want = oracle.dot_csr_ndarray((M, N), data, indices, indptr, b)
    tiling(0, tile_bytes)
    got = _run(data, indices, indptr, b, K, N, idt, n_panels)
    assert bits_equal(got, want)


@pytest.mark.parametrize("dtype,N", [(np.float32, 128), (np.float64, 36)])
def test_tiled_passes_strided_b_and_c(tiling, dtype, N):
    """ldb, ldc > N: B is a column slice of a wider array, C a column slice of a wider output."""
    from sparse_b200 import _device as D

    rng = np.random.default_rng(3)
    M, K = 500, 1500
    data, indices, indptr = _csr_with_edge_rows(rng, M, K, dtype)
    bfull = rand_dense(rng, (K, N + 12), dtype)
    b = np.ascontiguousarray(bfull[:, :N])
    want = oracle.dot_csr_ndarray((M, N), data, indices, indptr, b)
    t = D.torch()
    cfull = t.full((M, N + 20), 7.0, dtype=D.upload(b).dtype, device="cuda")
    tiling(0, 64)
    _run(data, indices, indptr, b, K, N, np.int32, 9, bt=D.upload(bfull)[:, :N], out=cfull[:, :N])
    got = D.download(cfull)
    assert bits_equal(np.ascontiguousarray(got[:, :N]), want)
    assert (got[:, N:] == 7.0).all()  # the padding columns of C are not written


def test_tiled_passes_inf_nan_in_b(tiling):
    """inf / NaN rows of B: same bits as the one-pass kernel; the oracle agrees up to NaN payloads."""
    rng = np.random.default_rng(4)
    M, K, N = 600, 1000, 128
    data, indices, indptr = _csr_with_edge_rows(rng, M, K, np.float32)
    b = rand_dense(rng, (K, N), np.float32)
    b[5, :7] = np.inf
    b[17, 3:40] = -np.inf
    b[300, ::3] = np.nan
    want = oracle.dot_csr_ndarray((M, N), data, indices, indptr, b)
    tiling(0, 128)
    one = _run(data, indices, indptr, b, K, N, np.int32, 1)
    got = _run(data, indices, indptr, b, K, N, np.int32, 11)
    assert bits_equal(got, one)
    assert np.isnan(got).any() and np.isinf(got).any()
    assert np.array_equal(got, want, equal_nan=True)
    fin = np.isfinite(want)
    assert bits_equal(got[fin], want[fin])


@pytest.mark.parametrize("idt", [np.int32, np.int64])
def test_one_reversed_row_takes_the_guarded_fallback(tiling, idt):
    """One unsorted row in an otherwise sorted matrix: the passes stand down and the one-pass kernel computes the
    whole product in the stored order (which the passes could not reproduce for that row)."""
    rng = np.random.default_rng(5)
    M, K, N = 800, 1200, 128
    data, indices, indptr = rand_csr(rng, M, K, 0.03, np.float32)
    r = int(np.argmax(np.diff(indptr)))
    s, e = indptr[r], indptr[r + 1]
    indices[s:e] = indices[s:e][::-1].copy()
    data[s:e] = data[s:e][::-1].copy()
    b = rand_dense(rng, (K, N), np.float32)
    want = oracle.dot_csr_ndarray((M, N), data, indices, indptr, b)
    tiling(0, 128)
    for n_panels in (6, 0):
        assert bits_equal(_run(data, indices, indptr, b, K, N, idt, n_panels), want)


def test_automatic_choice_with_a_small_panel_budget(tiling):
    """B larger than twice the L2 and nnz >= 64 K: the automatic choice takes the passes; a 1 MB budget gives many
    panels.  Compared with the one-pass kernel on the whole output."""
    from sparse_b200 import _device as D
    from sparse_b200 import _kernels as Kn

    t = D.torch()
    g = t.Generator(device="cuda").manual_seed(2)
    M, K, N = 200_000, 250_000, 128  # B = 128 MB fp32
    nnz = 18_000_000
    lin = t.unique(t.randint(0, M * K, (nnz,), generator=g, device="cuda", dtype=t.int64))
    rows, cols = lin // K, (lin % K).to(t.int32)
    indptr = t.zeros(M + 1, dtype=t.int64, device="cuda")
    indptr[1:] = t.cumsum(t.bincount(rows, minlength=M), 0)
    indptr = indptr.to(t.int32)
    vals = t.rand(len(lin), generator=g, device="cuda", dtype=t.float32)
    B = t.rand((K, N), generator=g, device="cuda", dtype=t.float32)
    from sparse_b200 import _lib

    ref = Kn.spmm_csr_dense(vals, cols, indptr, B, M, K, N, n_panels=1)
    for panel_bytes, min_launches in ((1 << 20, 4 * 30), (0, 4 * 2)):
        tiling(panel_bytes, 0)
        n0 = _lib.launch_count()
        got = Kn.spmm_csr_dense(vals, cols, indptr, B, M, K, N)
        assert _lib.launch_count() - n0 >= min_launches  # 4 column tiles x P panels
        assert t.equal(got.view(t.int32), ref.view(t.int32))


def test_c2_automatic_path_equals_one_pass_kernel():
    """Full C2 (1e6 x 1e6, nnz 1e8, N = 128 fp32): the automatic (tiled) path against the one-pass kernel, whole output."""
    import torch

    import bench
    from sparse_b200 import _kernels as Kn

    M = K = 1_000_000
    vals, cols, indptr, B = bench.make_workload(torch, M, K, 100_000_000, 128, 1234, torch.device("cuda", 0))
    auto = Kn.spmm_csr_dense(vals, cols, indptr, B, M, K, 128)
    one = Kn.spmm_csr_dense(vals, cols, indptr, B, M, K, 128, n_panels=1)
    assert torch.equal(auto.view(torch.int32), one.view(torch.int32))
