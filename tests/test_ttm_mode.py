"""ttm_mode(X, U, mode): mode-n tensor times matrix (TTM) and vector (TTV) of a sparse tensor of order 2..8, with a sparse
COO result.

Bit identity with ``moveaxis(tensordot(X, U, axes=([mode], [0]), return_type=COO), -1, mode)`` and with the dense
tensordot at the stored positions, golden parity with the reference's own tensordot (tests/golden/ttm_mode_api.npz),
shapes far beyond tensordot's size limit against a CPU restatement of the order (tests/_tensor_order.py), the kernel's
layouts (fiber lengths, group sizes, both end modes, the scalar column path, GCXS layouts), the cached fiber stream,
edge cases and errors of U.  Determinism across calls, U's location and layout, both index widths and the argument
errors shared with the other sparse-tensor ops are in tests/test_tensor_ops_contract.py.  Every body runs on the NumPy
mock without a GPU and on the CUDA kernels with `-m gpu`."""
import itertools

import numpy as np
import pytest

import _tensor_order as TO
from _api import dec, sp  # noqa: F401
from _golden import load
from _tensor_cases import SHAPES, dev, rand_tensor

same_bits = TO.same_bits


def unfused(sp, X, U, mode, **kw):
    """tensordot's answer, with the R axis moved to `mode` for a 2-D U."""
    r = sp.tensordot(X, U, axes=([mode], [0]), **kw)
    if np.ndim(U) == 2:
        r = sp.moveaxis(r, -1, mode) if isinstance(r, sp.COO) else np.moveaxis(r, -1, mode)
    return r


def assert_same(got, want):
    """Same canonical COO: shape, dtype, fill value, coordinates and values bit for bit."""
    assert got.format == "coo" and want.format == "coo"
    assert got.shape == want.shape and got.dtype == want.dtype
    assert same_bits(np.asarray(got.fill_value), np.asarray(want.fill_value))
    assert np.array_equal(np.asarray(got.coords, np.int64), np.asarray(want.coords, np.int64))
    assert same_bits(got.data, want.data)


def assert_order(got, X, U, mode):
    """got equals the CPU restatement of the order on X's entries."""
    coords, vals = TO.result(np.asarray(X.coords), np.asarray(X.data), X.shape, U, mode, got.dtype)
    assert got.format == "coo" and got.dtype == vals.dtype
    assert same_bits(np.asarray(got.fill_value), np.asarray(got.dtype.type(0)))
    assert np.array_equal(np.asarray(got.coords, np.int64), coords)
    assert same_bits(got.data, vals)


def factor(rng, n, R, dtype):
    return rng.standard_normal(n).astype(dtype) if R is None else rng.standard_normal((n, R)).astype(dtype)


# R = None is the 1-D (TTV) form; 4 and 128 take the vector path in both dtypes, 1, 3 and 37 the scalar path
@pytest.mark.parametrize("R", [0, 1, 3, 4, 37, 128, None])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("order", sorted(SHAPES))
def test_tensordot_bit_identity(sp, order, dtype, R):
    shape = SHAPES[order]
    rng = np.random.default_rng(10 * order + (R or 0))
    X = rand_tensor(sp, rng, shape, max(int(np.prod(shape)) // 3, 5), dtype, signed=True)
    for mode in range(order):
        U = factor(rng, shape[mode], R, dtype)
        got = sp.ttm_mode(X, U, mode)
        assert_same(got, unfused(sp, X, U, mode, return_type=sp.COO))
        dense = unfused(sp, X, U, mode)
        assert same_bits(dense[tuple(np.asarray(got.coords))], got.data)
        assert np.count_nonzero(dense != 0) == got.nnz
        assert same_bits(got.data, sp.ttm_mode(X, U, mode - order).data)  # negative modes count from the end


def special_inputs(sp, rng, shape, mode, dtype):
    """Signed values; fibers whose two entries cancel exactly (U's rows 0 and 1 equal, values +v at i_mode = 0 and -v at
    i_mode = 1); U rows holding +-inf (inf - inf and 0 * inf give NaN, which is stored)."""
    X = rand_tensor(sp, rng, shape, int(np.prod(shape)) // 3, dtype, signed=True)
    c, v = np.asarray(X.coords), np.asarray(X.data)
    lead = c[mode] == 0
    twin = c[:, lead].copy()
    twin[mode] = 1
    keep = ~np.isin(np.ravel_multi_index(c, shape), np.ravel_multi_index(twin, shape))
    c = np.concatenate([c[:, keep], twin], axis=1)
    v = np.concatenate([v[keep], -v[lead]]).astype(dtype)
    v[rng.choice(len(v), 3, replace=False)] = 0.0  # stored zeros: 0 * inf is NaN, 0 * finite adds a zero
    X = sp.COO(c, v, shape=shape)
    U = rng.standard_normal((shape[mode], 5)).astype(dtype)
    U[1] = U[0]
    U[2, 1], U[3, 1], U[4, 2] = np.inf, -np.inf, np.nan
    return X, U


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_cancellation_inf_nan(sp, dtype):
    rng = np.random.default_rng(3)
    shape = (9, 8, 7)
    for mode in range(3):
        X, U = special_inputs(sp, rng, shape, mode, dtype)
        got = sp.ttm_mode(X, U, mode)
        assert_same(got, unfused(sp, X, U, mode, return_type=sp.COO))
        assert_order(got, X, U, mode)
        assert np.isnan(got.data).any() and np.isinf(got.data).any()
        assert got.nnz < len(np.unique(np.delete(np.asarray(X.coords), mode, 0), axis=1).T) * U.shape[1]  # pruned
        dense = unfused(sp, X, U, mode)
        assert same_bits(dense[tuple(np.asarray(got.coords))], got.data)
        assert np.count_nonzero(dense != 0) == got.nnz
        u = U[:, 1].copy()
        assert_same(sp.ttm_mode(X, u, mode), unfused(sp, X, u, mode, return_type=sp.COO))


GOLDEN = [c for c in load("ttm_mode_api")]


@pytest.mark.parametrize("c", GOLDEN, ids=lambda c: f"{c['op']}-{c['dtype']}-order{c['order']}-mode{c['mode']}")
def test_golden_parity(sp, c):
    X = dec(sp, c, "X_")
    got = sp.ttm_mode(X, np.array(c.arr["U"]), int(c["mode"]))
    w = c.sub("out_")
    assert got.shape == tuple(int(s) for s in w["shape"]) and got.dtype == w["data"].dtype
    assert same_bits(np.asarray(got.fill_value), np.asarray(w["fill"]))
    assert np.array_equal(np.asarray(got.coords, np.int64), np.asarray(w["coords"], np.int64))
    assert same_bits(got.data, w["data"])


def huge_tensor(sp, rng, shape, nnz, dtype):
    """Random entries, plus for every axis copies of a tenth of them moved along that axis (fibers of length > 1)."""
    c = np.stack([rng.integers(0, s, nnz) for s in shape])
    extra = []
    for a, s in enumerate(shape):
        d = c[:, : nnz // 10].copy()
        d[a] = rng.integers(0, s, d.shape[1])
        extra.append(d)
    c = np.concatenate([c] + extra, axis=1)
    v = (rng.random(c.shape[1]) + 0.1) * rng.choice([-1.0, 1.0], c.shape[1])
    return sp.COO(c, v.astype(dtype), shape=shape)  # duplicates summed, sorted


@pytest.mark.parametrize("nnz", [1_000, 100_000])
def test_beyond_tensordot_size_limit(sp, nnz):
    """(2e5, 2e5, 2e5): tensordot would build an indptr of 4e10 entries; ttm_mode needs O(nnz + result)."""
    rng = np.random.default_rng(nnz)
    shape = (200_000,) * 3
    X = huge_tensor(sp, rng, shape, nnz, "float32")
    for mode in range(3):
        for R in (4, None):
            U = factor(rng, shape[mode], R, "float32")
            got = sp.ttm_mode(X, U, mode)
            assert got.shape == shape[:mode] + ((4,) if R else ()) + shape[mode + 1:]
            assert_order(got, X, U, mode)


def long_and_short_fibers(sp, rng, dtype):
    """(3, 2000, 4): along axis 1, fibers (i0, i2) of up to 1500 entries next to fibers of one entry."""
    shape = (3, 2000, 4)
    c = []
    for i0, i2 in itertools.product(range(3), range(4)):
        n = 1500 if (i0 + i2) % 2 == 0 else 1
        ks = np.sort(rng.choice(shape[1], n, replace=False))
        c.append(np.stack([np.full(n, i0), ks, np.full(n, i2)]))
    c = np.concatenate(c, axis=1)
    v = (rng.random(c.shape[1]) + 0.1) * rng.choice([-1.0, 1.0], c.shape[1])
    return sp.COO(c, v.astype(dtype), shape=shape)


# 8 is the vector path in both dtypes, 5 the scalar path, 200 more column tiles than one lane group covers
@pytest.mark.parametrize("R", [5, 8, 200])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_long_fibers_and_groups(sp, dtype, R):
    """Mode 1: fibers longer than any tile or warp, groups of four fibers.  Mode 0: one group spanning every fiber.
    Mode 2 (the last): groups of one fiber."""
    rng = np.random.default_rng(R)
    X = long_and_short_fibers(sp, rng, dtype)
    for mode in range(3):
        U = rng.standard_normal((X.shape[mode], R)).astype(dtype)
        got = sp.ttm_mode(X, U, mode)
        assert_same(got, unfused(sp, X, U, mode, return_type=sp.COO))
    U = rng.standard_normal((X.shape[1], R)).astype(dtype)
    assert_order(sp.ttm_mode(X, U, 1), X, U, 1)


# 8 and 128 (f32) / 64 (f64) fill one column tile of the long-fiber CTAs on the vector path, 200 takes several; 5 and
# 37 the scalar path
@pytest.mark.parametrize("R", [5, 8, 37, 64, 128, 200])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_long_fiber_role_same_bits(sp, dtype, R, monkeypatch):
    """Every fiber in the short-fiber lanes, every fiber in whole thread blocks, and the default split at 512 entries
    (fibers of 1 to 1500 entries, chunk boundaries of the staged products crossed): the same bits, equal to tensordot."""
    X = long_and_short_fibers(sp, np.random.default_rng(31 + R), dtype)
    results = {}
    for long_min in (10**12, 0, 1, 512):
        monkeypatch.setattr(sp._fused, "_TTM_LONG_FIBER", long_min)
        for mode in range(3):
            U = np.random.default_rng(mode + R).standard_normal((X.shape[mode], R)).astype(dtype)
            got = sp.ttm_mode(X, U, mode)
            if mode in results:
                assert_same(got, results[mode])
            else:
                results[mode] = got
                assert_same(got, unfused(sp, X, U, mode, return_type=sp.COO))
            if mode == 1 and long_min == 512:
                assert X._mode_streams[("fiber-long", 1, True, 512)].shape[0] == 6  # the 1500-entry fibers
    u = np.random.default_rng(2).standard_normal(X.shape[1]).astype(dtype)
    monkeypatch.setattr(sp._fused, "_TTM_LONG_FIBER", 0)
    assert_same(sp.ttm_mode(X, u, 1), unfused(sp, X, u, 1, return_type=sp.COO))


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_unaligned_u_scalar_path(sp, dtype):
    """A column slice of a wider device tensor is not 16-byte aligned: the scalar path, the same bits."""
    rng = np.random.default_rng(21)
    X = rand_tensor(sp, rng, (20, 30, 12), 2000, dtype, signed=True)
    for mode, R in itertools.product(range(3), (8, 16)):
        U = rng.standard_normal((X.shape[mode], R)).astype(dtype)
        wide = dev(sp, np.concatenate([np.zeros((U.shape[0], 1), dtype), U], axis=1))[:, 1:]
        want = sp.ttm_mode(X, U, mode)
        got = sp.ttm_mode(X, wide, mode)
        assert_same(got, want)
        strided = dev(sp, np.repeat(U[:, :1], 2, axis=1))[:, 0]  # a 1-D view with stride 2
        assert_same(sp.ttm_mode(X, strided, mode), sp.ttm_mode(X, U[:, 0], mode))


def test_gcxs_layouts(sp):
    rng = np.random.default_rng(22)
    X = rand_tensor(sp, rng, (11, 9, 7), 300, "float64", signed=True)
    for k in (1, 2):
        for ca in itertools.combinations(range(3), k):
            G = X.asformat("gcxs", compressed_axes=ca)
            for mode in range(3):
                U = rng.standard_normal((X.shape[mode], 6))
                assert_same(sp.ttm_mode(G, U, mode), sp.ttm_mode(X, U, mode))
                assert_same(sp.ttm_mode(G, U[:, 0], mode), sp.ttm_mode(X, U[:, 0], mode))


def test_second_call_does_not_sort(sp, monkeypatch):
    rng = np.random.default_rng(24)
    X = rand_tensor(sp, rng, (25, 18, 9), 1200, "float64", signed=True)
    sorts = []
    real = sp._kernels.sort_keys

    def counting(*a, **k):
        sorts.append(1)
        return real(*a, **k)

    monkeypatch.setattr(sp._kernels, "sort_keys", counting)
    U = [rng.standard_normal((s, 7)) for s in X.shape]
    sp.ttm_mode(X, U[2], 2)
    assert len(sorts) == 0  # the last mode reads X's canonical order
    for mode in (0, 1):
        launches = [sp._lib.launch_count()] if not sp._device._TEST_CPU else None
        first = sp.ttm_mode(X, U[mode], mode)
        n = len(sorts)
        assert n == 1 + mode
        if launches:
            launches.append(sp._lib.launch_count())
        again = sp.ttm_mode(X, U[mode], mode)
        assert len(sorts) == n
        if launches:  # the second call launches the kernel and the pruning only
            assert sp._lib.launch_count() - launches[1] < launches[1] - launches[0]
        assert_same(again, first)
    # replacing X's contents in place drops its cached fiber streams: the next call sorts again, on the new values
    before = sp.ttm_mode(X, U[0], 0)
    np.multiply(X, 2, out=X)
    assert not any(str(k[0]).startswith("fiber") for k in (X._mode_streams or {}))
    after = sp.ttm_mode(X, U[0], 0)
    assert len(sorts) == 3
    assert np.array_equal(after.coords, before.coords) and same_bits(after.data, 2 * before.data)


def test_edge_cases(sp):
    rng = np.random.default_rng(25)
    shape = (5, 6, 7)
    empty = sp.COO(np.zeros((3, 0), np.int64), np.zeros(0, np.float32), shape=shape)
    X = rand_tensor(sp, rng, shape, 60, "float64", signed=True)
    for mode in range(3):
        for src, U, want_shape in ((empty, np.ones((shape[mode], 3)), shape[:mode] + (3,) + shape[mode + 1:]),
                                   (X, np.ones((shape[mode], 0)), shape[:mode] + (0,) + shape[mode + 1:]),
                                   (empty, np.ones(shape[mode], np.float32), shape[:mode] + shape[mode + 1:])):
            got = sp.ttm_mode(src, U, mode)
            assert got.format == "coo" and got.nnz == 0 and got.shape == want_shape
            assert got.dtype == np.result_type(src.dtype, U.dtype)
            if src.nnz:
                assert_same(got, unfused(sp, src, U, mode, return_type=sp.COO))
    zero_ext = sp.COO(np.zeros((3, 0), np.int64), np.zeros(0), shape=(5, 0, 7))
    for mode, U, want_shape in ((1, np.ones((0, 2)), (5, 2, 7)), (0, np.ones((5, 2)), (2, 0, 7)),
                                (2, np.ones(7), (5, 0))):
        got = sp.ttm_mode(zero_ext, U, mode)
        assert got.shape == want_shape and got.nnz == 0 and got.dtype == np.float64
    one = sp.COO(np.array([[4], [5], [6]]), np.array([2.0]), shape=shape)
    U = rng.standard_normal((6, 3))
    got = sp.ttm_mode(one, U, 1)
    assert np.array_equal(got.coords, [[4, 4, 4], [0, 1, 2], [6, 6, 6]]) and same_bits(got.data, 2.0 * U[5])
    # order 2: TTV gives a 1-D result
    M = rand_tensor(sp, rng, (30, 20), 100, "float32", signed=True)
    for mode in range(2):
        u = rng.standard_normal(M.shape[mode]).astype(np.float32)
        got = sp.ttm_mode(M, u, mode)
        assert got.ndim == 1
        assert_same(got, unfused(sp, M, u, mode, return_type=sp.COO))


def test_errors(sp):
    rng = np.random.default_rng(26)
    X = rand_tensor(sp, rng, (5, 6, 7), 40, "float64")
    with pytest.raises(ValueError, match="shape mismatch"):
        sp.ttm_mode(X, rng.random((5, 3)), 1)
    with pytest.raises(ValueError, match="shape mismatch"):
        sp.ttm_mode(X, rng.random(7), 1)
    with pytest.raises(ValueError, match="shape mismatch"):
        sp.ttm_mode(X, rng.random((6, 3, 2)), 1)
    with pytest.raises(TypeError, match="outside the CUDA dtype matrix"):
        sp.ttm_mode(X, np.ones((6, 3), np.complex128), 1)
    big = sp.COO(np.zeros((3, 1), np.int64), np.ones(1), shape=(2**31, 2**31, 1))
    with pytest.raises(ValueError, match="2\\*\\*63"):
        sp.ttm_mode(big, np.ones((1, 2)), 2)
    sp.ttm_mode(big, np.ones(1), 2)  # the TTV result, (2**31, 2**31), fits


@pytest.mark.gpu
def test_beyond_tensordot_full_size():
    """(1e6, 2e6, 1.5e6) with 1.2e7 entries, every mode, R = 16 and TTV, f32: every value within 2e-5 of a float64
    restatement on the device, and 2,000 sampled fibers bit-equal to the CPU restatement of the order."""
    import torch

    import sparse_b200 as spm

    devc = torch.device("cuda")
    shape, nnz = (1_000_000, 2_000_000, 1_500_000), 10_000_000
    g = torch.Generator(device=devc).manual_seed(5)
    c = torch.stack([torch.randint(0, s, (nnz,), generator=g, device=devc) for s in shape])
    extra = []
    for a, s in enumerate(shape):  # fibers of length > 1 along every axis
        d = c[:, : nnz // 15].clone()
        d[a] = torch.randint(0, s, (d.shape[1],), generator=g, device=devc)
        extra.append(d)
    c = torch.cat([c] + extra, dim=1)
    v = (torch.rand(c.shape[1], generator=g, device=devc) + 0.1) * (
        torch.randint(0, 2, (c.shape[1],), generator=g, device=devc) * 2 - 1)
    X = spm.COO(c, v.float(), shape=shape)
    del c, v, extra
    assert X.nnz > 10_000_000
    Xc, Xv = X.coords, X.data
    rng = np.random.default_rng(7)
    for mode in range(3):
        for R in (16, None):
            U = torch.rand((shape[mode], R) if R else (shape[mode],), generator=g, device=devc) - 0.5
            got = spm.ttm_mode(X, U, mode)
            gc = got._dev()[0]
            gv = got._data_dev()
            # float64 restatement on the device: scatter-add of v * U[k] over the fibers' linear keys
            others = [m for m in range(3) if m != mode]
            cd = torch.from_numpy(Xc).to(devc)
            fk = cd[others[0]] * shape[others[1]] + cd[others[1]]
            Ud = (U if R else U[:, None]).double()
            prod = torch.from_numpy(Xv).to(devc).double()[:, None] * Ud[cd[mode]]
            uk, inv = torch.unique(fk, return_inverse=True)
            want = torch.zeros((len(uk), Ud.shape[1]), dtype=torch.float64, device=devc).index_add_(0, inv, prod)
            rest = [gc[m] for m in (others if R else (0, 1))]
            gk = rest[0] * shape[others[1]] + rest[1]
            gr = gc[mode] if R else torch.zeros_like(gk)
            w = want[torch.searchsorted(uk, gk), gr]
            assert torch.allclose(gv.double(), w, rtol=2e-5, atol=2e-5 * float(w.abs().max()))
            # sampled fibers against the CPU restatement, bit for bit
            pick = np.unique(rng.choice(len(uk), 2_000, replace=False))
            keys = uk[torch.from_numpy(pick).to(devc)].cpu().numpy()
            hk = Xc[others[0]] * shape[others[1]] + Xc[others[1]]
            sel = np.isin(hk, keys)
            rc, rv = TO.result(Xc[:, sel], Xv[sel], shape, U.cpu().numpy(), mode, np.float32)
            gsel = torch.isin(gk, torch.from_numpy(keys).to(devc))
            assert np.array_equal(gc[:, gsel].cpu().numpy(), rc)
            assert same_bits(gv[gsel].cpu().numpy(), rv)
            del got, gc, gv, prod, want
