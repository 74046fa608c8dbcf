"""CSR x CSR kernels (spgemm.cu) on rows that reach every path, bit for bit against the reference.

The rows come from tests/_spgemm_rows.py: A rows of 0, 1, 31, 32, 33, 64, 65 and more than 256 entries whose product
counts P sit on every table edge of the warp kernel (16/17, 32/33, 64/65, 256) and past it (257 and up, the CTA
kernel); empty B rows at lane 0, lane 31, in runs and as a chunk's last entry; columns that collide in one bucket of
either kernel's hash table (probes wrapping past the last slot) or that one CTA-kernel warp owns alone; products that
cancel to +0; -0.0, NaN and Inf; sums that differ between float32 / int64 and the float64 accumulator.  Every call
goes through the C ABI in REF order (reverse first touch) and SORTED order, with and without pruning, runs twice and
must give the same bits both times; indptr, column order, value bits (NaN positions for NaN) and the structural count
are compared with the oracle, or with the CPU restatement in tests/_spgemm_order.py where the oracle cannot serve
(wrapping integers, the float64 accumulator, columns of 2^32 and more).  The CPU tests at the top check the generator's
promises and pin the restatement against the oracle on any machine."""
import os

import numpy as np
import pytest

import _spgemm_order as R
import _spgemm_rows as G
import oracle

gpu = pytest.mark.gpu

H100_SMS = 132            # the CPU tests count for an H100 SXM
ROWS_KERNEL_REGS = 64     # spgemm_rows_kernel<float, float, int, 512, 4, *> (tools/res_usage.py): 8 CTAs per SM
M_KINDS = 6_007           # the row-kind matrix: ~460 long rows, every kind at every ticket position
M_SCALE = 200_003         # every warp of the row kernel draws several tickets; ~1,000 long rows
KINDS_LONG_EVERY, KINDS_SPECIAL_EVERY = 13, 17
SCALE_LONG_EVERY, SCALE_SPECIAL_EVERY = 199, 97
EDGES = (0, 1, 16, 17, 32, 33, 64, 65, 255, 256, 257)


def _kinds_pair(dtype, mode, M=M_KINDS, seed=0):
    kinds = G.row_kinds(M, KINDS_LONG_EVERY, KINDS_SPECIAL_EVERY)
    return G.make_pair(np.random.default_rng(seed), kinds, dtype, mode)


def _scale_pair():
    kinds = G.row_kinds(M_SCALE, SCALE_LONG_EVERY, SCALE_SPECIAL_EVERY)
    return G.make_pair(np.random.default_rng(1), kinds, np.float32, "special")


def _oracle(a, b, M, n_col):
    """REF-order (indptr, indices, data, nnz_struct) from the oracle."""
    d, i, p = oracle.dot_csr_csr((M, n_col), a[0], b[0], a[1], b[1], a[2], b[2])
    return p, i, d, len(i)


def _expect(ref, sorted_order, prune):
    """The wanted result in either order, pruned or not, from a REF-order result."""
    ip, ix, d, n = ref
    if sorted_order:
        ip, ix, d = R.sort_rows(ip, ix, d)
    if prune:
        ip, ix, d = R.prune(ip, ix, d)
    return ip, ix, d, n


# ---------------------------------------------------------------------------------------------------------------------
# the generator (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def test_product_counts_hit_every_edge():
    a, b, _ = _kinds_pair(np.float32, "plain")
    P = G.products(a, b)
    n = np.diff(a[2])
    assert set(EDGES) <= set(P.tolist())
    assert {0, 1, 31, 32, 33, 64, 65} <= set(n.tolist()) and (n > 256).any()
    for lo, hi in ((1, 16), (17, 32), (33, 64), (65, 256)):  # every table size of the warp kernel, both shapes
        band = (P >= lo) & (P <= hi)
        assert {G.warp_table(lo), G.warp_table(hi)} == {G.warp_table(lo)}
        assert (band & (n <= 32)).any() and (band & (n > 32)).any()
    assert ((P == 0) & (n > 32)).any() and ((P == 0) & (n == 0)).any()
    # every kind meets every position of a 4-row ticket; every short kind follows a row of each kernel
    kinds = G.row_kinds(M_KINDS, KINDS_LONG_EVERY, KINDS_SPECIAL_EVERY)
    nk = len(G.KINDS)
    seen = np.zeros((nk, 4), bool)
    seen[kinds, np.arange(M_KINDS) % 4] = True
    assert seen.all()
    follows = np.zeros((nk, 3), bool)  # (kind, previous row: P = 0 / warp kernel / CTA kernel)
    cls = np.where(P == 0, 0, np.where(P <= G.WARP_PMAX, 1, 2))
    follows[kinds[1:], cls[:-1]] = True
    assert follows[:len(G.SHORT_KINDS), 1:].all()


def test_multi_chunk_rows_stay_in_the_warp_kernel():
    a, b, _ = _kinds_pair(np.float32, "plain")
    P = G.products(a, b)
    n = np.diff(a[2])
    multi = (n > 32) & (P > 0) & (P <= G.WARP_PMAX)
    assert multi.sum() >= 1000
    assert set(P[multi].tolist()) >= {16, 17, 32, 33, 64, 65, 255, 256}
    assert (multi & (n > 256)).any()


def test_empty_b_rows_at_lane_0_lane_31_in_runs_and_at_chunk_ends():
    a, b, _ = _kinds_pair(np.float32, "plain")
    _, ai, ap = a
    empty = (b[2][ai + 1] == b[2][ai])
    P = G.products(a, b)
    n = np.diff(ap)
    for r in np.flatnonzero((n > 32) & (P > 0) & (P <= G.WARP_PMAX))[:200]:
        e = empty[ap[r]:ap[r + 1]]
        if not e[0]:
            continue
        assert e[0] and e[31] and e[-1] and e[8:16].all()
        assert all(e[c] for c in range(31, n[r], 32))
        break
    else:
        pytest.fail("no multi-chunk row with the hole pattern")
    # one-chunk rows too: lane 0 and lane 31 (the chunk's last entry) empty in a row with products
    one = np.flatnonzero((n == 32) & (P > 0))
    assert any(empty[ap[r]] and empty[ap[r] + 31] for r in one)


def test_hash_restatement_and_collision_sets():
    # the NumPy hashes against plain integer arithmetic
    ks = [0, 1, 5003, 2**31 - 1, 2**31, 2**32 - 1, 2**32, 2**32 + 12345, 2**39 + 7, 2**40 - 1]
    for k in ks:
        x = ((k & 0xFFFFFFFF) ^ (((k >> 32) * 0x85EBCA6B) & 0xFFFFFFFF))
        assert int(G.hash_small(np.array([k]))[0]) == ((x * 0x9E3779B1) & 0xFFFFFFFF) >> 20
        assert int(G.hash_col(np.array([k]))[0]) == ((k * 0x9E3779B97F4A7C15) & (2**64 - 1)) >> 32
    sp = G.special_rows()
    n_col = max(int(c.max()) for c in sp.values()) + 1
    for H in (64, 128, 256, 512):
        c = sp[f"c{H}"]
        P = len(c) * (2 if H == 512 else 1)  # the kinds that reference them alone (c512: with its reverse)
        assert G.warp_table(P) == H and P <= G.WARP_PMAX
        buckets = G.hash_small(c) & np.uint32(H - 1)
        assert len(set(buckets.tolist())) == 1 and len(set(c.tolist())) == len(c)
        assert int(buckets[0]) + len(c) > H  # the probe chain wraps past slot H - 1
    c = sp["cc"]
    H = G.cta_table(2 * len(c), n_col)
    assert 2 * len(c) > G.WARP_PMAX and H == 1024
    assert len(set((G.hash_col(c) & np.uint32(H - 1)).tolist())) == 1
    assert int(G.hash_col(c[:1])[0] & np.uint32(H - 1)) + len(c) > H
    assert set(G.cta_owner(c).tolist()) == {5} and set(G.cta_owner(sp["co"]).tolist()) == {2}


def test_long_rows_outnumber_the_cta_grid():
    for M, le, se in ((M_KINDS, KINDS_LONG_EVERY, KINDS_SPECIAL_EVERY), (M_SCALE, SCALE_LONG_EVERY,
                                                                          SCALE_SPECIAL_EVERY)):
        a, b, n_col = G.make_pair(np.random.default_rng(0), G.row_kinds(M, le, se), np.float32)
        P = G.products(a, b)
        long_rows = np.flatnonzero(P > G.WARP_PMAX)
        assert len(long_rows) > 2 * H100_SMS
        assert len({G.cta_table(int(p), n_col) for p in P[long_rows]}) >= 4
        n = np.diff(a[2])
        assert (n[long_rows] > G.CTA_THREADS).any()
        totals = np.concatenate([G.chunk_totals(a, b, r) for r in long_rows[:60]])
        assert (totals == G.CTA_TILE).any() and (totals == 2 * G.CTA_TILE).any()


def test_every_warp_draws_several_tickets():
    assert G.rows_kernel_ctas_per_sm(4, 4, False, 0) == 11  # shared memory alone
    ctas = G.rows_kernel_ctas_per_sm(4, 4, False, ROWS_KERNEL_REGS)
    assert G.tickets_per_warp(M_SCALE, H100_SMS, ctas) >= 8


# ---------------------------------------------------------------------------------------------------------------------
# the restatement against the oracle (CPU)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64])
def test_restatement_matches_the_oracle(dtype):
    a, b, n_col = _kinds_pair(dtype, "special" if np.dtype(dtype).kind == "f" else "plain", M=1201, seed=4)
    ref = _oracle(a, b, 1201, n_col)
    for s in (False, True):
        got = R.spgemm(a, b, 1201, n_col, sorted_order=s)
        want = _expect(ref, s, False)
        assert got[3] == want[3]
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert _same_values(got[2], want[2])


def test_restatement_reverses_completely_dense_rows():
    a, b, n_col = _dense_pair(np.float64)
    ref = _oracle(a, b, len(a[2]) - 1, n_col)
    assert ref[3] == (len(a[2]) - 1) * n_col
    got = R.spgemm(a, b, len(a[2]) - 1, n_col)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]) and _same_values(got[2], ref[2])


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64])
def test_wide_restatement_matches_the_csc_oracle(dtype):
    """wide=True is _dot_csc_ndarray_sparse: out^T = sparsify(b^T) @ A^T.  Here S = sparsify(b^T) (N x C, no stored
    zeros, ascending columns) and B = the CSC arrays of A; the written prefix of the oracle must equal the
    restatement's pruned result."""
    a, b, R_rows = _kinds_pair(dtype, "plain", M=601, seed=2)
    ad, ai, ap = a
    N, C = len(ap) - 1, len(b[2]) - 1
    # S: A's structure with its columns sorted per row, explicit zeros and -0.0 removed
    row = np.repeat(np.arange(N), np.diff(ap))
    ad = ad.copy()
    ad[ad == 0] = 1
    o = np.lexsort((ai, row))
    key = row[o] * C + ai[o]
    u = np.ones(len(key), bool)
    u[1:] = key[1:] != key[:-1]
    sd, si = ad[o][u], ai[o][u]
    sp = np.zeros(N + 1, np.int64)
    np.cumsum(np.bincount(row[o][u], minlength=N), out=sp[1:])
    dense_b = np.zeros((C, N), np.dtype(dtype))
    dense_b[si, np.repeat(np.arange(N), np.diff(sp))] = sd
    # the oracle's `prod = u * a_data` is the restatement's S value times B value
    wd, wi, wptr, written = oracle.dot_csc_ndarray_sparse((R_rows, C), (C, N), b[0], b[1], b[2], dense_b)
    ip, ix, d, n_struct = R.spgemm((sd, si, sp), b, N, R_rows, wide=True)
    assert n_struct == wptr[-1]
    ip, ix, d = R.prune(ip, ix, d)
    assert len(ix) == written
    assert np.array_equal(ix, wi[:written]) and _same_values(d, wd[:written])


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def _same_values(got, want):
    """Equal bits, except that a NaN only has to meet a NaN (payloads differ between the CPU and the GPU)."""
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    if got.shape != want.shape or got.dtype != want.dtype:
        return False
    u = R._UNSIGNED[got.dtype.itemsize]
    same = got.view(u) == want.view(u)
    if got.dtype.kind == "f":
        same |= np.isnan(got) & np.isnan(want)
    return bool(same.all())


def _dense_pair(dtype, M=300, n_col=40, K=64, seed=6):
    """Every row reaches every one of n_col columns: even rows through the warp kernel (P < 256), odd rows through the
    CTA kernel (seven complete B rows, P >= 280).  B rows 0..15 hold all columns (in random orders), the others random
    subsets."""
    rng = np.random.default_rng(seed)
    rows = [rng.permutation(n_col) for _ in range(16)]
    rows += [rng.choice(n_col, int(rng.integers(1, n_col)), replace=False) for _ in range(K - 16)]
    bp = np.zeros(K + 1, np.int64)
    np.cumsum([len(r) for r in rows], out=bp[1:])
    bi = np.concatenate(rows).astype(np.int64)
    a_rows = []
    for r in range(M):
        full = rng.choice(16, 7 if r % 2 else 1, replace=False)
        part = rng.choice(np.arange(16, K), 2, replace=False)
        a_rows.append(np.concatenate([part[:1], full, part[1:]]))
    ap = np.zeros(M + 1, np.int64)
    np.cumsum([len(r) for r in a_rows], out=ap[1:])
    ai = np.concatenate(a_rows).astype(np.int64)
    return (G.values(rng, len(ai), dtype, "plain"), ai, ap), (G.values(rng, len(bi), dtype, "plain"), bi, bp), n_col


class _Dev:
    """The operands on the device, in one index type."""

    def __init__(self, a, b, M, n_col, idt):
        from sparse_b200 import _device as D

        up = lambda x: D.upload(np.ascontiguousarray(x))
        self.args = (up(a[2].astype(idt)), up(a[1].astype(idt)), up(a[0]), up(b[2].astype(idt)),
                     up(b[1].astype(idt)), up(b[0]))
        self.M, self.K, self.n_col = M, len(b[2]) - 1, n_col


def _check(dev, want, *, sorted_order, prune, wide=False):
    """Two calls (with the COO row ids, then without) must both equal `want` and each other bit for bit."""
    from sparse_b200 import _device as D
    from sparse_b200 import _kernels as Kn

    wip, wix, wd, wn = want
    outs = []
    for want_rows in (True, False):
        ip, ix, rows, d, n = Kn.spgemm(*dev.args, dev.M, dev.K, dev.n_col, sorted_order=sorted_order, wide=wide,
                                       prune=prune, want_indptr=True, want_rows=want_rows)
        ip, ix, d = D.download(ip), D.download(ix), D.download(d)
        assert n == wn, "structural count"
        assert np.array_equal(ip, wip), "indptr"
        assert np.array_equal(ix, wix), _first_diff(ix, wix, ip, "column")
        assert _same_values(d, wd), _first_diff(d, wd, ip, "value")
        if want_rows:
            assert np.array_equal(D.download(rows), np.repeat(np.arange(dev.M), np.diff(wip)))
        outs.append(d)
    assert np.array_equal(outs[0].view(np.uint8), outs[1].view(np.uint8)), "two calls gave different bits"


def _first_diff(got, want, indptr, what):
    if got.shape != want.shape:
        return f"{what}s: {got.shape} vs {want.shape}"
    u = R._UNSIGNED[got.dtype.itemsize]
    bad = np.flatnonzero(np.ascontiguousarray(got).view(u) != np.ascontiguousarray(want).view(u))
    if not len(bad):
        return ""
    r = int(np.searchsorted(indptr, bad[0], side="right") - 1)
    return f"{len(bad)} {what}s differ, first at entry {bad[0]} (row {r}): got {got[bad[0]]!r}, want {want[bad[0]]!r}"


@pytest.fixture(scope="module")
def orc():
    oracle.set_threads(min(16, os.cpu_count() or 1))
    return oracle


@pytest.fixture
def thresholds():
    from sparse_b200 import _kernels as Kn

    yield Kn.spgemm_set_thresholds
    Kn.spgemm_set_thresholds(64, 256)


_cache = {}


def _kinds_case(dtype, mode):
    """The row-kind matrix and its REF result (oracle, or the restatement for wrapping integers), shared by tests."""
    key = (np.dtype(dtype), mode)
    if key not in _cache:
        a, b, n_col = _kinds_pair(dtype, mode)
        ref = R.spgemm(a, b, M_KINDS, n_col) if mode == "wrap" else _oracle(a, b, M_KINDS, n_col)
        _cache[key] = (a, b, n_col, ref)
    return _cache[key]


def _mode(dtype):
    return "special" if np.dtype(dtype).kind == "f" else "wrap"


# ---------------------------------------------------------------------------------------------------------------------
# GPU: row kinds, bin edges, collisions, special values
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("idt", [np.int32, np.int64], ids=["i32idx", "i64idx"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32, np.int64], ids=lambda d: np.dtype(d).name)
def test_row_kinds(orc, dtype, idt):
    a, b, n_col, ref = _kinds_case(dtype, _mode(dtype))
    dev = _Dev(a, b, M_KINDS, n_col, idt)
    for s in (False, True):
        for p in (False, True):
            _check(dev, _expect(ref, s, p), sorted_order=s, prune=p)


@gpu
@pytest.mark.parametrize("t1", [1, 33, 200])
@pytest.mark.parametrize("dtype,idt", [(np.float32, np.int32), (np.int64, np.int64)], ids=["f32", "i64"])
def test_rows_move_between_kernels(orc, thresholds, dtype, idt, t1):
    """Rows above t1 products go to the CTA kernel instead of the warp kernel; the result must not change."""
    a, b, n_col, ref = _kinds_case(dtype, _mode(dtype))
    dev = _Dev(a, b, M_KINDS, n_col, idt)
    thresholds(64, t1)
    _check(dev, _expect(ref, False, False), sorted_order=False, prune=False)
    _check(dev, _expect(ref, True, True), sorted_order=True, prune=True)


@gpu
@pytest.mark.parametrize("t1", [256, 1])
def test_collision_rows(orc, thresholds, t1):
    """Only the special kinds: one-bucket columns of every warp table and of the CTA table, one owner warp, twins."""
    nk = len(G.SHORT_KINDS) + len(G.LONG_KINDS)
    kinds = nk + np.arange(997) % len(G.SPECIAL_KINDS)
    a, b, n_col = G.make_pair(np.random.default_rng(12), kinds, np.float64, "plain")
    ref = _oracle(a, b, len(kinds), n_col)
    thresholds(64, t1)
    for idt in (np.int32, np.int64):
        dev = _Dev(a, b, len(kinds), n_col, idt)
        for s in (False, True):
            _check(dev, _expect(ref, s, True), sorted_order=s, prune=True)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: scale (every warp takes several tickets; ~1,000 long rows share 264 CTAs' scratch)
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_every_warp_walks_many_tickets(orc):
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = G.rows_kernel_ctas_per_sm(4, 4, False, ROWS_KERNEL_REGS)
    assert G.tickets_per_warp(M_SCALE, sms, ctas) >= 4
    a, b, n_col = _scale_pair()
    assert (G.products(a, b) > G.WARP_PMAX).sum() > 2 * sms
    ref = _oracle(a, b, M_SCALE, n_col)
    dev = _Dev(a, b, M_SCALE, n_col, np.int32)
    _check(dev, _expect(ref, False, False), sorted_order=False, prune=False)
    _check(dev, _expect(ref, True, True), sorted_order=True, prune=True)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: 64-bit columns
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", [np.float64, np.int64], ids=lambda d: np.dtype(d).name)
def test_columns_past_2_to_the_32(orc, dtype):
    """A strictly increasing relabel of B's columns into [2^32, 2^40) keeps the first-touch and ascending orders, so
    the result is the relabelled reference result.  Random gaps on the row-kind matrix; on a matrix of 40 columns
    (completely dense rows from both kernels), new labels that all share their low 32 bits."""
    rng = np.random.default_rng(40)
    a, b, n_col, ref = _kinds_case(dtype, _mode(dtype))
    new = 2**32 + np.cumsum(rng.integers(1, 2**17, n_col))
    da, db, dn = _dense_pair(dtype)
    dref = _oracle(da, db, len(da[2]) - 1, dn + 1)  # not completely dense once the columns are relabelled
    low = (np.arange(1, dn + 1, dtype=np.int64) << 32) | 0x5A5A5A5A
    for (a, b, ref, new) in ((a, b, ref, new), (da, db, dref, low)):
        assert new[0] >= 2**32 and new[-1] < 2**40 and (np.diff(new) > 0).all()
        M = len(a[2]) - 1
        b2 = (b[0], new[b[1]], b[2])
        dev = _Dev(a, b2, M, 2**40, np.int64)
        ip, ix, d, n = ref
        for s in (False, True):
            for p in (False, True):
                w = _expect((ip, ix, d, n), s, p)
                _check(dev, (w[0], new[w[1]], w[2], w[3]), sorted_order=s, prune=p)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the float64 accumulator
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", [np.float32, np.int64], ids=lambda d: np.dtype(d).name)
def test_wide_accumulator(orc, dtype):
    """wide=True: products in T, sums in float64, zero sums stored as +0 (dropped by prune).  The w1 / w2 / w3 rows
    sum to values that float32 and int64 accumulators get wrong."""
    a, b, n_col = _kinds_pair(dtype, "special" if np.dtype(dtype).kind == "f" else "plain", seed=5)
    ref = R.spgemm(a, b, M_KINDS, n_col, wide=True)
    narrow = R.spgemm(a, b, M_KINDS, n_col)
    assert not _same_values(ref[2], narrow[2])  # the matrix tells the two accumulators apart
    dev = _Dev(a, b, M_KINDS, n_col, np.int64)
    _check(dev, _expect(ref, False, True), sorted_order=False, prune=True, wide=True)
    _check(dev, _expect(ref, True, False), sorted_order=True, prune=False, wide=True)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: completely dense results, degenerate shapes
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", [np.float32, np.int64], ids=lambda d: np.dtype(d).name)
def test_completely_dense_rows_from_both_kernels(orc, dtype):
    a, b, n_col = _dense_pair(dtype)
    M = len(a[2]) - 1
    P = G.products(a, b)
    assert (P > G.WARP_PMAX).any() and (P <= G.WARP_PMAX).any()
    ref = _oracle(a, b, M, n_col)
    assert ref[3] == M * n_col
    dev = _Dev(a, b, M, n_col, np.int32)
    for s in (False, True):
        _check(dev, _expect(ref, s, False), sorted_order=s, prune=False)


def _small(M, K, n_col, a_lens, b_lens, seed=0):
    rng = np.random.default_rng(seed)
    ap = np.concatenate([[0], np.cumsum(a_lens)]).astype(np.int64)
    bp = np.concatenate([[0], np.cumsum(b_lens)]).astype(np.int64)
    ai = rng.integers(0, max(K, 1), ap[-1]).astype(np.int64)
    bi = np.concatenate([rng.choice(n_col, n, replace=False) for n in b_lens] or [[]]).astype(np.int64)
    return ((rng.random(ap[-1]) * 2 - 1), ai, ap), ((rng.random(bp[-1]) * 2 - 1), bi, bp)


@gpu
@pytest.mark.parametrize("M,K,n_col,a_lens,b_lens", [
    (0, 5, 7, [], [1, 0, 3, 2, 7]),             # no rows
    (4, 0, 7, [0, 0, 0, 0], []),                # no inner dimension
    (5, 4, 0, [2, 0, 3, 1, 4], [0, 0, 0, 0]),   # no columns
    (6, 4, 1, [2, 0, 3, 1, 4, 40], [1, 0, 1, 1]),  # one column: every row with products is completely dense
    (5, 6, 9, [0, 0, 0, 0, 0], [3, 2, 0, 1, 4, 9]),  # nnz(A) = 0
    (7, 5, 9, [3, 0, 40, 1, 300, 2, 1], [0, 0, 0, 0, 0]),  # every B row empty: no products at all
], ids=["M0", "K0", "ncol0", "ncol1", "nnzA0", "Bempty"])
def test_degenerate_shapes(orc, M, K, n_col, a_lens, b_lens):
    a, b = _small(M, K, n_col, a_lens, b_lens)
    ref = _oracle(a, b, M, n_col)
    for idt in (np.int32, np.int64):
        dev = _Dev(a, b, M, n_col, idt)
        for s in (False, True):
            _check(dev, _expect(ref, s, True), sorted_order=s, prune=True)
