"""CSR x dense kernels on matrices where every warp walks many rows, bit for bit against the oracle.

The persistent kernels only exercise their cross-row code once a warp (or a group of L lanes in the tiled passes)
takes more than one row: the tiled passes carry a two-chunk register ring, A entries two chunks ahead and offsets two
rows ahead across row boundaries, and the one-pass kernel draws 2-row tickets from a global counter.  The rows here
come from tests/_spmm_rows.py, whose runs per K panel have known lengths (0, 1, L-1, L, L+1, 2L, 2L+1, long; blocks of
empty rows; rows in the first or last panel only).  Every product goes into an output pre-filled with a NaN pattern,
is computed twice, and is compared bit for bit with the oracle; padding columns of a wider output must keep the
pattern.  The CPU tests at the top check the generator's promises on any machine."""
import os

import numpy as np
import pytest

import oracle
from _spmm_rows import (BLOCK, measured_runs, panel_of, panel_ranges, panel_rows, pass_grid, run_cycle, run_lengths,
                        walk)
from _util import bits_equal, rand_dense

gpu = pytest.mark.gpu

M_ROWS = 100_003          # odd: never a multiple of a grid's row stride, so the last warp has groups past M
H100_SMS = 132            # the CPU tests replay the walk for an H100 SXM ...
MAX_PASS_CTAS = 2         # ... at the most CTAs per SM the tiled passes reach
ONE_PASS_MAX_CTAS = 5     # the most CTAs per SM of any form of the one-pass kernel (form 12)
SENTINEL = {np.dtype(np.float32): np.uint32(0x7FC05A5A), np.dtype(np.float64): np.uint64(0x7FF85A5A5A5A5A5A)}


def tile_lanes(N, dtype, tile_bytes):
    """Lanes per row group of the tiled passes: the tile width, halved while N needs no more than half the lanes."""
    lanes = {64: 4, 128: 8, 256: 16}[tile_bytes]
    packs = -(-N * np.dtype(dtype).itemsize // 16)
    while lanes > 4 and packs <= lanes // 2:
        lanes //= 2
    return lanes


# dtype, index dtype, N, tile bytes, K, P, extra output columns (ldc - N).  L = 4, 8, 16; L = 4 from N = 8 fp32 with
# idle lanes; N ending inside a tile (36 fp32, 72 fp64); P = 2, odd P not dividing K, P > K (width 1, empty panels).
K1P_CASES = [
    (np.float32, np.int32, 128, 128, 5000, 2, 0),
    (np.float32, np.int64, 64, 64, 5000, 7, 12),
    (np.float32, np.int32, 256, 256, 4999, 5, 0),
    (np.float32, np.int32, 8, 128, 5000, 3, 4),
    (np.float32, np.int32, 36, 128, 5000, 9, 0),
    (np.float32, np.int64, 128, 128, 11, 16, 4),
    (np.float64, np.int64, 72, 128, 13, 16, 2),
    (np.float64, np.int32, 64, 256, 4999, 3, 0),
    (np.float64, np.int64, 32, 64, 5000, 2, 2),
]


def _k1p_id(c):
    dt, it, N, tb, K, P, pad = c
    return f"{np.dtype(dt).name}-{np.dtype(it).name}-N{N}-L{tile_lanes(N, dt, tb)}-K{K}-P{P}-pad{pad}"


# ---------------------------------------------------------------------------------------------------------------------
# the generator (CPU)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", K1P_CASES, ids=_k1p_id)
def test_generator_delivers_its_runs(case):
    dt, _, N, tb, K, P, _ = case
    L = tile_lanes(N, dt, tb)
    data, indices, indptr = panel_rows(np.random.default_rng(1), M_ROWS, K, P, L, dt)
    R = run_lengths(M_ROWS, K, P, L)
    assert np.array_equal(measured_runs(indices, indptr, K, P), R)
    assert indptr[-1] == len(indices) and (np.diff(indptr) >= 0).all()
    row = np.repeat(np.arange(M_ROWS), np.diff(indptr))
    same_row = row[1:] == row[:-1]
    assert (indices[1:][same_row] >= indices[:-1][same_row]).all()  # rows sorted (repeats allowed)
    assert indices.min() >= 0 and indices.max() == K - 1
    lo, hi = panel_ranges(K, P)
    live = np.flatnonzero(hi > lo)
    want = set(run_cycle(L).tolist())
    for p in live:
        assert want <= set(R[:, p].tolist()), p  # every run length of the cycle, in every panel with columns
        e = np.concatenate([[0], (R[:, p] == 0).astype(np.int8), [0]])
        d = np.flatnonzero(np.diff(e))
        assert (d[1::2] - d[::2]).max() >= BLOCK  # a block of >= 64 consecutive rows empty in this panel
    if P > K:
        assert (R[:, K:] == 0).all() and len(live) == K
    nz = R > 0
    assert (nz[:, 0] & ~nz[:, 1:].any(axis=1)).any()  # rows with entries in the first panel only
    assert (nz[:, live[-1]] & ~nz[:, :live[-1]].any(axis=1)).any()  # ... and in the last panel only
    present = set(np.unique(indices).tolist())
    for p in live[1:]:
        assert {lo[p] - 1, lo[p]} <= present
    # repeated columns on both sides of a panel boundary within one row
    q = panel_of(indices, K, P)
    dup = same_row & (indices[1:] == indices[:-1])
    at_end = np.zeros(len(indices), bool)
    at_end[:-1] = dup & (indices[:-1] == hi[q[:-1]] - 1)
    at_start = np.zeros(len(indices), bool)
    at_start[:-1] = dup & (indices[:-1] == lo[q[:-1]])
    if len(live) > 1:
        assert (at_end[:-2] & at_start[2:] & (row[:-2] == row[2:])).any()
    neg0 = (data == 0) & np.signbit(data)
    assert neg0.any()


@pytest.mark.parametrize("case", K1P_CASES, ids=_k1p_id)
def test_every_group_walks_many_rows(case):
    """Replay of every pass's walk on an H100 SXM grid: each group walks at least 4 rows, the groups of one warp
    walk different numbers of chunks, and some warp steps find every chunk empty (the skipped step)."""
    dt, _, N, tb, K, P, _ = case
    L = tile_lanes(N, dt, tb)
    R = run_lengths(M_ROWS, K, P, L)
    stride = pass_grid(M_ROWS, L, H100_SMS, MAX_PASS_CTAS)
    lo, hi = panel_ranges(K, P)
    assert M_ROWS % (32 // L), "the last warp must have groups past M"
    for p in range(P):
        rows, skips, uneven = walk(R[:, p], L, stride)
        assert rows >= 4
        assert skips > 0
        if hi[p] > lo[p]:
            assert uneven > stride // (32 // L) // 2  # most warps


def test_walk_replay_on_a_hand_made_stream():
    # L = 16: 2 groups per warp, stride 4 -> warps (0, 1) and (2, 3); rows 0..9
    runs = np.array([0, 17, 0, 0, 0, 1, 0, 40, 3, 0])
    rows, skips, uneven = walk(runs, 16, 4)
    # group chunk streams: g0: rows 0,4,8 -> [e][e][1]; g1: rows 1,5,9 -> [2 chunks][1][e]; g2: rows 2,6 -> [e][e];
    # g3: rows 3,7 -> [e][3 chunks].  Warp 0: steps 0..3 = (e,x) (e,x) (x,x) (past,e) -> step 3 skipped.
    # Warp 1: (e,e) (e,x) (past,x) (past,x) -> step 0 skipped.  Both warps' groups walk 3 / 4 and 2 / 4 chunks.
    assert (rows, skips, uneven) == (2, 2, 2)


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def orc():
    oracle.set_threads(min(16, os.cpu_count() or 1))
    return oracle


@pytest.fixture
def tiling():
    from sparse_b200 import _kernels as Kn

    yield Kn.spmm_set_tiling
    Kn.spmm_set_tiling(0, 0)


@pytest.fixture
def variant():
    from sparse_b200 import _kernels as Kn

    yield Kn.spmm_set_variant
    Kn.spmm_set_variant(1, 8)


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _sentinel_out(M, N, dtype, pad):
    """(M, N + pad) output filled with a NaN bit pattern; returns (whole tensor, the (M, N) column slice)."""
    import torch

    from sparse_b200 import _device as D

    s = SENTINEL[np.dtype(dtype)]
    it = torch.int32 if s.dtype.itemsize == 4 else torch.int64
    whole = torch.full((M, N + pad), int(s.view(np.int32 if it == torch.int32 else np.int64)), dtype=it,
                       device="cuda").view(D.torch_dtype(dtype))
    return whole, whole[:, :N]


def _check(whole, N, want):
    """The (M, N) slice equals `want` bit for bit and every padding column still holds the sentinel."""
    from sparse_b200 import _device as D

    got = D.download(whole)
    assert bits_equal(np.ascontiguousarray(got[:, :N]), want), _first_diff(got[:, :N], want)
    pad = np.ascontiguousarray(got[:, N:])
    assert (pad.view(SENTINEL[got.dtype].dtype) == SENTINEL[got.dtype]).all(), "padding columns were written"


def _first_diff(got, want):
    u = {4: np.uint32, 8: np.uint64}[want.dtype.itemsize]
    bad = np.argwhere(np.ascontiguousarray(got).view(u) != np.ascontiguousarray(want).view(u))
    if len(bad) == 0:
        return "shapes or dtypes differ"
    r, c = bad[0]
    return f"{len(bad)} elements differ, first at row {r} col {c}: got {got[r, c]!r}, want {want[r, c]!r}"


def _upload(data, indices, indptr, b, idt):
    from sparse_b200 import _device as D

    return D.upload(data), D.upload(indices.astype(idt)), D.upload(indptr.astype(idt)), D.upload(b)


def _run_twice(args, M, K, N, dtype, pad, want, **kw):
    """Two calls, each into a fresh sentinel-filled output; both must equal `want` (and so each other)."""
    from sparse_b200 import _kernels as Kn

    for _ in range(2):
        whole, out = _sentinel_out(M, N, dtype, pad)
        Kn.spmm_csr_dense(*args, M, K, N, out=out, **kw)
        _check(whole, N, want)


# ---------------------------------------------------------------------------------------------------------------------
# K1p: the tiled passes, forced
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("case", K1P_CASES, ids=_k1p_id)
def test_tiled_passes_walk_many_rows(orc, tiling, case):
    from sparse_b200 import _kernels as Kn
    from sparse_b200 import _lib

    dt, idt, N, tb, K, P, pad = case
    L = tile_lanes(N, dt, tb)
    stride = pass_grid(M_ROWS, L, _sms(), MAX_PASS_CTAS)
    assert M_ROWS // stride >= 4, "every group must walk at least 4 rows"
    data, indices, indptr = panel_rows(np.random.default_rng(hash(case[2:]) % 2**32), M_ROWS, K, P, L, dt)
    b = rand_dense(np.random.default_rng(7), (K, N), dt)
    want = orc.dot_csr_ndarray((M_ROWS, N), data, indices, indptr, b)
    args = _upload(data, indices, indptr, b, idt)
    assert Kn.csr_rows_sorted(args[1], args[2], M_ROWS)  # else the passes would stand down for the one-pass kernel
    tiling(0, tb)
    tiles = -(-N // (L * (16 // np.dtype(dt).itemsize)))
    for _ in range(2):
        whole, out = _sentinel_out(M_ROWS, N, dt, pad)
        n0 = _lib.launch_count()
        Kn.spmm_csr_dense(*args, M_ROWS, K, N, out=out, n_panels=P)
        assert _lib.launch_count() - n0 >= tiles * P  # the passes ran: one launch per (tile, panel)
        _check(whole, N, want)
    _run_twice(args, M_ROWS, K, N, dt, pad, want, n_panels=1)


@gpu
def test_automatic_choice_takes_the_passes_on_generated_rows(orc, tiling):
    """B = 128 MB fp32 (> 2 L2) and nnz >= 48 K: the library picks the passes; a 1 MB budget gives 31 panels, which
    is the P the rows were generated for.  Whole output against the one-pass kernel and the oracle."""
    import torch

    from sparse_b200 import _kernels as Kn
    from sparse_b200 import _lib

    M, K, N, L = 60_001, 250_000, 128, 8
    P = -(-K * L * 16 // (1 << 20))
    assert P == 31
    assert M // pass_grid(M, L, _sms(), MAX_PASS_CTAS) >= 4
    data, indices, indptr = panel_rows(np.random.default_rng(31), M, K, P, L, np.float32)
    assert len(data) >= 48 * K
    b = rand_dense(np.random.default_rng(8), (K, N), np.float32)
    want = orc.dot_csr_ndarray((M, N), data, indices, indptr, b)
    args = _upload(data, indices, indptr, b, np.int32)
    one = Kn.spmm_csr_dense(*args, M, K, N, n_panels=1)
    tiling(1 << 20, 0)
    for _ in range(2):
        whole, out = _sentinel_out(M, N, np.float32, 0)
        n0 = _lib.launch_count()
        Kn.spmm_csr_dense(*args, M, K, N, out=out)
        assert _lib.launch_count() - n0 >= 4 * P
        assert torch.equal(whole.view(torch.int32), one.view(torch.int32))
        _check(whole, N, want)


# ---------------------------------------------------------------------------------------------------------------------
# K1: the one-pass kernels with many rows per warp
# ---------------------------------------------------------------------------------------------------------------------
_ONE_PASS_K = 5000
_one_pass_cache = {}


def _one_pass_case(orc, dtype, N):
    """Rows of 0, 1, 31, 32, 33, 64, 65 and 163 entries (runs of the L = 32 cycle, one panel) and the oracle's
    product, shared by the variants."""
    key = (np.dtype(dtype), N)
    if key not in _one_pass_cache:
        data, indices, indptr = panel_rows(np.random.default_rng(N), M_ROWS, _ONE_PASS_K, 1, 32, dtype)
        b = rand_dense(np.random.default_rng(N + 1), (_ONE_PASS_K, N), dtype)
        _one_pass_cache[key] = (data, indices, indptr, b, orc.dot_csr_ndarray((M_ROWS, N), data, indices, indptr, b))
    return _one_pass_cache[key]


# variant, unroll, dtype, N, index dtype, extra output columns
ONE_PASS_CASES = [
    (1, 8, np.float32, 128, np.int32, 0),    # default: dynamic rows, 8 gathers in flight
    (1, 8, np.float32, 128, np.int64, 12),
    (1, 8, np.float32, 256, np.int32, 4),    # two column tiles
    (1, 8, np.float32, 129, np.int32, 3),    # VEC = 1
    (1, 8, np.float64, 64, np.int64, 2),
    (10, 8, np.float32, 128, np.int32, 0),   # forms of the dynamic-row kernel
    (11, 8, np.float32, 128, np.int32, 4),
    (12, 8, np.float32, 128, np.int64, 0),
    (13, 8, np.float32, 128, np.int32, 0),
    (13, 8, np.float32, 129, np.int32, 0),
    (3, 8, np.float32, 128, np.int32, 4),    # static one-row-per-warp grid
    (1, 4, np.float32, 128, np.int32, 0),    # static grid, U = 4 / 16 / 32
    (1, 16, np.float32, 128, np.int64, 0),
    (1, 32, np.float32, 128, np.int32, 12),
    (2, 8, np.float32, 128, np.int32, 0),    # bulk-copy ring (N * 4 = 512 bytes); wraps past 1,584 rows
    (2, 8, np.float64, 64, np.int64, 2),
]


@gpu
@pytest.mark.parametrize("v,u,dt,N,idt,pad", ONE_PASS_CASES,
                         ids=lambda x: np.dtype(x).name if isinstance(x, type) else str(x))
def test_one_pass_kernels_walk_many_rows(orc, variant, v, u, dt, N, idt, pad):
    assert M_ROWS >= 4 * 2 * _sms() * ONE_PASS_MAX_CTAS * 8, "every warp must draw several 2-row tickets"
    data, indices, indptr, b, want = _one_pass_case(orc, dt, N)
    args = _upload(data, indices, indptr, b, idt)
    variant(v, u)
    _run_twice(args, M_ROWS, _ONE_PASS_K, N, dt, pad, want, n_panels=1)


@gpu
@pytest.mark.parametrize("dt,N,pad", [(np.float32, 8320, 4), (np.float64, 4160, 0)])
def test_static_fallback_for_more_than_64_column_tiles(orc, dt, N, pad):
    """N = 8320 fp32 / 4160 fp64 is 65 tiles of 32 packs: past the dynamic kernel's 64 counters, the static grid runs
    (also when long rows are asked for)."""
    M, K = 2001, 300
    data, indices, indptr = panel_rows(np.random.default_rng(N), M, K, 1, 32, dt)
    b = rand_dense(np.random.default_rng(66), (K, N), dt)
    want = orc.dot_csr_ndarray((M, N), data, indices, indptr, b)
    args = _upload(data, indices, indptr, b, np.int32)
    _run_twice(args, M, K, N, dt, pad, want)
    _run_twice(args, M, K, N, dt, pad, want, long_rows=True)


# ---------------------------------------------------------------------------------------------------------------------
# long rows (column-split kernels) at scale
# ---------------------------------------------------------------------------------------------------------------------
def _long_row_csr(rng, M, K, dtype):
    """Rows of the L = 32 cycle (mean about 32 entries, so the long-row threshold is 512) with every 997th row
    replaced by 512 (not long), 513, 600, 2049 or 4100 entries."""
    lens = run_lengths(M, K, 1, 32)[:, 0]
    longs = np.arange(5, M, 997)
    lens[longs] = np.resize([512, 513, 600, 2049, 4100], len(longs))
    indptr = np.zeros(M + 1, np.int64)
    np.cumsum(lens, out=indptr[1:])
    row = np.repeat(np.arange(M, dtype=np.int64), lens)
    indices = np.sort(row * K + rng.integers(0, K, len(row))) - row * K
    data = (rng.random(len(row)) * 2 - 1).astype(dtype)
    data[::7] = -0.0
    return data, indices, indptr


@gpu
@pytest.mark.parametrize("dt,N,pad", [(np.float32, 128, 4), (np.float32, 129, 0), (np.float64, 64, 0)])
def test_long_rows_scattered_through_many_tickets(orc, dt, N, pad):
    """~100 long rows among 100k: the shared-memory ring (aligned rows) or the register-staged kernel (N = 129)
    computes them on the side stream while the dynamic-row kernel reads its skip flags across many tickets."""
    K = 5000
    data, indices, indptr = _long_row_csr(np.random.default_rng(N), M_ROWS, K, dt)
    assert (np.diff(indptr) > 512).sum() >= 80
    b = rand_dense(np.random.default_rng(5), (K, N), dt)
    want = orc.dot_csr_ndarray((M_ROWS, N), data, indices, indptr, b)
    args = _upload(data, indices, indptr, b, np.int32)
    _run_twice(args, M_ROWS, K, N, dt, pad, want, long_rows=True)
    _run_twice(args, M_ROWS, K, N, dt, pad, want, long_rows=False)


@gpu
def test_long_rows_past_the_column_split_cap(orc):
    """2^18 + 100 rows of 600 entries among 1.2M rows of 10 (4 x mean = 463 < 600, so all of them are long): the
    column-split kernels take the first 2^18 in their list and the row kernel must still compute the other 100.
    Whole output against long_rows=False; sampled rows, long ones included, against the oracle."""
    import torch

    from sparse_b200 import _device as D
    from sparse_b200 import _kernels as Kn

    n_long, n_short, K, N = (1 << 18) + 100, 1_200_001, 1000, 128
    M = n_long + n_short
    g = torch.Generator(device="cuda").manual_seed(18)
    lens = torch.full((M,), 10, dtype=torch.int64, device="cuda")
    long_rows = torch.randperm(M, generator=g, device="cuda")[:n_long].sort().values
    lens[long_rows] = 600
    indptr = torch.zeros(M + 1, dtype=torch.int64, device="cuda")
    indptr[1:] = torch.cumsum(lens, 0)
    nnz = int(indptr[-1])
    threshold = max(512, 4 * (nnz // M))  # spmm_skew.cu: rows longer than this are long
    assert threshold < 600 and n_long > 1 << 18 and nnz < 2**31
    cols = torch.randint(0, K, (nnz,), generator=g, device="cuda", dtype=torch.int32)
    vals = torch.rand(nnz, generator=g, device="cuda", dtype=torch.float32) * 2 - 1
    B = torch.rand((K, N), generator=g, device="cuda", dtype=torch.float32) * 2 - 1
    ip32 = indptr.to(torch.int32)
    outs = []
    for long_mode in (True, True, False):
        whole, out = _sentinel_out(M, N, np.float32, 0)
        Kn.spmm_csr_dense(vals, cols, ip32, B, M, K, N, out=out, long_rows=long_mode)
        outs.append(whole)
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
    assert torch.equal(outs[0].view(torch.int32), outs[2].view(torch.int32))
    del outs[1:]
    # sampled rows: the first and last 64 long rows, 64 long rows in between, 128 short rows
    lr = long_rows.cpu().numpy()
    short = np.setdiff1d(np.arange(M), lr)
    rng = np.random.default_rng(19)
    sel = np.unique(np.concatenate([lr[:64], lr[-64:], rng.choice(lr, 64), rng.choice(short, 128)]))
    ip = D.download(indptr)
    take = np.concatenate([np.arange(ip[r], ip[r + 1]) for r in sel])
    tk = torch.from_numpy(take).cuda()
    sub_ptr = np.zeros(len(sel) + 1, np.int64)
    np.cumsum(ip[sel + 1] - ip[sel], out=sub_ptr[1:])
    want = orc.dot_csr_ndarray((len(sel), N), D.download(vals[tk]), D.download(cols[tk]).astype(np.int64), sub_ptr,
                               D.download(B))
    got = D.download(outs[0][torch.from_numpy(sel).cuda()])
    assert bits_equal(got, want), _first_diff(got, want)
