"""What the sparse-tensor ops share: mttkrp_mode, ttmc_mode, tttp, cp_completion_mode and, where its single U fits,
ttm_mode.

The argument checks of the tensor and its factors, bit-identical results across repeated calls, copies of X, factor
locations and layouts, storage layouts and both index widths (with the cached streams' widths), and the mode-stream
cache that mttkrp_mode, ttmc_mode and cp_completion_mode share.  Each test is parametrised over the ops it applies to;
what only one op does is tested in that op's file.  Every body runs on the NumPy mock without a GPU and on the CUDA
kernels with `-m gpu`."""
import pickle

import numpy as np
import pytest

from _api import sp  # noqa: F401
from _tensor_cases import LAYOUTS, dev, entries, host, layout, layout_id, plant_specials, rand_tensor
from _tensor_order import same_bits


def _ttm(sp, X, U, mode):
    return sp.ttm_mode(X, U[mode % len(U)], mode)  # the factor of `mode` (any one for an out-of-range mode)


# (name, call(sp, X, factors, mode)); tttp reads every factor and has no mode
OPS = {"mttkrp_mode": lambda sp, X, U, mode: sp.mttkrp_mode(X, U, mode),
       "ttmc_mode": lambda sp, X, U, mode: sp.ttmc_mode(X, U, mode),
       "tttp": lambda sp, X, U, mode: sp.tttp(X, U),
       "cp_completion_mode": lambda sp, X, U, mode: sp.cp_completion_mode(X, U, mode, 0.5),
       "ttm_mode": _ttm}
FACTOR_LIST_OPS = ["mttkrp_mode", "ttmc_mode", "tttp", "cp_completion_mode"]  # one factor per mode
STREAM_OPS = ["mttkrp_mode", "ttmc_mode", "cp_completion_mode"]  # the cached, sorted mode stream
# unequal ranks for ttmc_mode: R_last = 8 fills whole 16-byte packs in both dtypes, 6 and 5 do not in float32
RANKS = {"ttmc_mode": (5, 6, 8)}


def factors(op, rng, shape, dtype):
    """Signed normal factors (ranks 12, or RANKS[op]) with +-inf, NaN and -0.0 planted in each; cp_completion_mode's
    stay finite, since one non-finite value turns every row whose entries reach it into NaN."""
    U = [rng.standard_normal((s, r)).astype(dtype) for s, r in zip(shape, RANKS.get(op, (12,) * len(shape)))]
    return U if op == "cp_completion_mode" else plant_specials(rng, U)


def same(a, b):
    """Bit-identical results: dense ones (host arrays or device tensors) by their values, sparse ones by format, shape,
    fill value and their entries in stored order."""
    if not hasattr(a, "nnz"):
        return same_bits(host(a), host(b))
    (ca, va), (cb, vb) = entries(a), entries(b)
    return (a.format == b.format and a.shape == b.shape and np.array_equal(ca, cb) and same_bits(va, vb)
            and same_bits(np.asarray(a.fill_value), np.asarray(b.fill_value)))


def coo(r):
    return r.tocoo() if getattr(r, "format", None) == "gcxs" else r


def index_arrays(op, X, mode, narrow):
    """The index arrays of the stream `op` cached on X for `mode`, with int32 (`narrow`) or int64 indices."""
    if op == "ttm_mode":
        s = X._mode_streams[("fiber", mode, narrow)]
        return [s[0], *s[2:5]]
    return X._mode_streams[(0 if op == "tttp" else mode, narrow)][0]


@pytest.mark.parametrize("op", OPS)
def test_argument_errors(sp, op):
    call = OPS[op]
    rng = np.random.default_rng(23)
    X = rand_tensor(sp, rng, (5, 6, 7), 40, "float64")
    U = [rng.random((s, 3)) for s in X.shape]
    with pytest.raises(TypeError):
        call(sp, X.todense(), U, 0)
    with pytest.raises(ValueError):
        call(sp, rand_tensor(sp, rng, (9,), 4, "float64"), [rng.random((9, 2))], 0)
    nine = sp.COO(np.zeros((9, 1), np.int64), np.ones(1), shape=(2,) * 9)
    with pytest.raises(ValueError):
        call(sp, nine, [np.ones((2, 2))] * 9, 0)
    with pytest.raises(ValueError, match="zero fill"):
        call(sp, sp.COO(X.coords, X.data, shape=X.shape, fill_value=1.0), U, 0)
    if op != "tttp":
        for bad in (3, -4):
            with pytest.raises(np.exceptions.AxisError):
                call(sp, X, U, bad)
    with pytest.raises(TypeError, match="outside the CUDA dtype matrix"):
        Xi = sp.COO(X.coords, np.arange(1, X.nnz + 1), shape=X.shape)
        call(sp, Xi, [np.ones((s, 3), np.int64) for s in X.shape], 1)
    if op not in FACTOR_LIST_OPS:
        return
    with pytest.raises(ValueError):
        call(sp, X, U[:2], 0)
    with pytest.raises(ValueError):
        call(sp, X, U + [U[0]], 0)
    with pytest.raises(ValueError):
        call(sp, X, [U[0], rng.random((5, 3)), U[2]], 0)
    with pytest.raises(ValueError):
        call(sp, X, [U[0], rng.random(6), U[2]], 0)
    if op != "ttmc_mode":  # ttmc_mode takes a rank per mode
        with pytest.raises(ValueError):
            call(sp, X, [U[0], rng.random((6, 4)), U[2]], 0)


@pytest.mark.parametrize("lay", range(len(LAYOUTS)), ids=layout_id)
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("op", OPS)
def test_bit_identical_across_calls_copies_locations_and_index_widths(sp, op, dtype, lay, monkeypatch):
    """Repeated calls, a copy of X (which builds its streams again), device and mixed host / device factors and int64
    indices give the first call's bits, in every storage layout, and the same bits as the COO tensor (a sparse result
    converted to COO); the cached streams hold int32 and int64 indices as asked."""
    call = OPS[op]
    rng = np.random.default_rng(11)
    X = rand_tensor(sp, rng, (70, 60, 8), 9000, dtype, signed=True)
    U = factors(op, rng, X.shape, dtype)
    Ud = [dev(sp, u) for u in U]
    Y = layout(X, *LAYOUTS[lay])
    for mode in range(3):
        first = call(sp, Y, U, mode)
        if lay:
            assert same(coo(first), call(sp, X, U, mode)), mode
        for other in [call(sp, Y, U, mode) for _ in range(3)] + [call(sp, Y.copy(), U, mode), call(sp, Y, Ud, mode),
                                                                 call(sp, Y, [U[0], Ud[1], U[2]], mode)]:
            assert same(other, first), mode
        monkeypatch.setattr(sp._fused, "_FORCE_WIDE_INDEX", True)
        wide = call(sp, Y, U, mode)
        monkeypatch.setattr(sp._fused, "_FORCE_WIDE_INDEX", False)
        assert same(wide, first), mode
        if op == "tttp" and Y.format == "gcxs":
            continue  # tttp reads a GCXS tensor's own arrays, without a stream
        assert all(c.element_size() == 4 for c in index_arrays(op, Y, mode, True)), mode
        assert all(c.element_size() == 8 for c in index_arrays(op, Y, mode, False)), mode


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("op", OPS)
def test_factor_layouts_and_output_kind(sp, op, dtype):
    """Fortran-ordered host factors, transposed (column-major) device factors and device views one column into a wider
    buffer (unaligned rows) give the bits of C-contiguous host factors; a device factor makes a dense result a device
    tensor; a float64 factor promotes the result to the float64 call's bits."""
    import torch

    call = OPS[op]
    rng = np.random.default_rng(13)
    X = rand_tensor(sp, rng, (40, 30, 20), 2500, dtype, signed=True)
    U = factors(op, rng, X.shape, dtype)
    fortran = [np.asfortranarray(u) for u in U]
    transposed = [dev(sp, u.T.copy()).T for u in U]
    offset = [dev(sp, np.concatenate([np.zeros((u.shape[0], 1), dtype), u], axis=1))[:, 1:] for u in U]
    mixed = [U[0], dev(sp, U[1]), U[2]]
    for m in range(3):
        want = call(sp, X, U, m)
        assert same(call(sp, X, fortran, m), want), m
        for variant in (transposed, offset, mixed):
            got = call(sp, X, variant, m)
            if not hasattr(got, "nnz"):
                assert isinstance(got, torch.Tensor)
            assert same(got, want), m
    if op in FACTOR_LIST_OPS:
        U64 = [U[0], U[1].astype(np.float64), U[2]]
        got = call(sp, X, U64, 0)
        assert got.dtype == np.float64
        assert same(got, call(sp, X.astype(np.float64), [u.astype(np.float64) for u in U], 0))


@pytest.mark.parametrize("op", STREAM_OPS)
def test_mode_stream_cache(sp, op, monkeypatch):
    """One sort per mode other than 0 (mode 0 reads X's C order), whichever of the ops builds the stream; none in the
    others' calls afterwards; a copy or an unpickled X starts without streams; a GCXS tensor caches its own; new
    contents (np.multiply(..., out=X)) drop the cache."""
    calls = []
    real = sp._kernels.sort_keys

    def counting(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(sp._kernels, "sort_keys", counting)
    call = OPS[op]
    rng = np.random.default_rng(3)
    X = rand_tensor(sp, rng, (30, 20, 10), 1500, "float64", signed=True)
    U = [rng.standard_normal((s, 6)) for s in X.shape]
    before = {}
    for mode in (0, 1, 2):
        calls.clear()
        for _ in range(3):
            before[mode] = call(sp, X, U, mode)
        assert len(calls) == (0 if mode == 0 else 1), mode
        for other in STREAM_OPS:
            OPS[other](sp, X, U, mode)
        assert len(calls) == (0 if mode == 0 else 1), mode
    assert X.copy()._mode_streams is None
    assert pickle.loads(pickle.dumps(X))._mode_streams is None
    np.multiply(X, 2, out=X)
    for mode in (0, 1, 2):
        assert same(call(sp, X, U, mode), 2 * host(before[mode])), mode

    G = X.asformat("gcxs", compressed_axes=(1,))
    calls.clear()
    for _ in range(2):
        g1 = call(sp, G, U, 1)
    assert same(g1, call(sp, X, U, 1))
    n_first = len(calls)
    call(sp, G, U, 1)
    assert len(calls) == n_first
