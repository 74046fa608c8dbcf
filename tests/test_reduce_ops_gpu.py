"""The grouped reduction (K7, csrc/reduce_fused.cu, `b2s_reduce_single`), op by op, dtype by dtype and form by form.

Every (op, work dtype) pair the host can send runs through both kernel forms (count / scan / emit, and the single-pass
look-back kernel) on key streams whose runs start and end at every offset relative to a thread, a warp and a tile,
span the look-back windows and cover tile counts 1 .. ~5000, at group widths on both sides of the form threshold and on
every FastDiv path.  Group ids, values and the count of results equal to the result fill are compared with the
restatement in tests/_red_ops.py: bit for bit on exactly representable values and for the order-sensitive extrema,
within a rounding-error bound on random floats.  Then the fill-value step (every fill, complete and incomplete groups,
n_fill past 2^24), the prune, and the public API (axes, COO / GCXS, narrow and unsigned integers).

The CPU tests at the top pin the kernel geometry, the case list, the streams and the restatement itself (against the
reference's golden outputs)."""
import math
import os
import zlib

import numpy as np
import pytest

import _red_ops as R
from _api import sp  # noqa: F401  (fixture: the mock kernels on a CPU box, the CUDA kernels on a GPU box)
from _golden import load

gpu = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
KERNEL = os.path.join(HERE, "..", "sparse_b200", "csrc", "reduce_fused.cu")


def _host_pairs():
    """(op code, work dtype) for every reduction the host sends to the kernel: _reduce.py's op table and dtype matrix
    under NumPy's result-type rules (int32 sums in int64, narrow and unsigned integers through int64, logical ops on
    bool)."""
    from sparse_b200 import _reduce

    inputs = [np.dtype(t) for t in (np.float32, np.float64, np.int8, np.uint8, np.int16, np.int32, np.int64,
                                    np.uint32, np.uint64, np.bool_)]
    pairs = set()
    for method, op in _reduce._RED.items():
        for dt in inputs:
            try:
                with np.errstate(all="ignore"):
                    res = method.reduce(np.zeros(1, dt)).dtype
            except TypeError:
                continue
            if res not in _reduce._RED_DTYPES and res.kind in "iu":
                res = np.dtype(np.int64)
            if res not in _reduce._RED_DTYPES:
                continue
            pairs.add((op, np.dtype(np.bool_) if op in (4, 5) else res))
    return sorted(pairs, key=lambda p: (p[0], p[1].name))


PAIRS = _host_pairs()
CASES = [pytest.param(op, T, id=f"{R.OPS[op].__name__}-{T.name}") for op, T in PAIRS]
FLOAT_CASES = [p for p in CASES if p.values[1].kind == "f"]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: geometry, case list, streams, restatement
# ---------------------------------------------------------------------------------------------------------------------
def test_geometry_matches_the_kernel():
    with open(KERNEL) as f:
        g = R.parse_geometry(f.read())
    assert (g["threads"], g["items"], g["tile"]) == (R.THREADS, R.ITEMS, R.TILE)
    assert g["carry"] == [R.CARRY_WINDOW] and g["heads"] == [R.HEADS_WINDOW]
    assert g["form_max"] == R.TWO_PASS_MAX_NCOLS
    assert max(R.NCOLS_TWO_PASS) == R.TWO_PASS_MAX_NCOLS < min(R.NCOLS_SINGLE)


def test_every_op_code_has_a_case():
    assert {op for op, _ in PAIRS} == set(range(11))
    assert (4, np.dtype(np.bool_)) in PAIRS and (0, np.dtype(np.bool_)) not in PAIRS
    assert (0, np.dtype(np.int32)) not in PAIRS and (2, np.dtype(np.int32)) in PAIRS
    assert not any(op in (4, 5) and T != np.bool_ for op, T in PAIRS)
    assert not any(op in (6, 7, 8) and T.kind == "f" for op, T in PAIRS)


def test_streams_cover_the_tile_geometry():
    S = R.streams()
    starts = []
    for name in ("lengths", "tile_fill", "span", "whole"):
        s = np.cumsum([0] + S[name][:-1])
        starts.append(s)
        ends = s + np.asarray(S[name]) - 1
        if name == "lengths":
            assert set(np.asarray(S[name])) == set(R.LENGTHS) | {3}
            assert len(set(s % R.ITEMS)) == R.ITEMS and len(set(ends % R.ITEMS)) == R.ITEMS
            assert len(set(s % (32 * R.ITEMS))) > 40 and len(set(s % R.TILE)) > 40
        if name == "tile_fill":
            assert ((s % R.TILE == 0) & (np.asarray(S[name]) == R.TILE)).sum() >= 3
            assert ((ends % R.TILE) == R.TILE - 1).sum() >= 6
    spans = np.asarray(S["span"]) // R.TILE
    for t in (31, 32, 33, 63, 64, 65, 300):
        assert t in spans
    for tiles in (1, 2, 31, 32, 33, 64, 65, 5000):
        assert -(-sum(S[f"tiles{tiles}"]) // R.TILE) == tiles
    for n in (1, 7, 8, 2047, 2048, 2049):
        assert sum(S[f"n{n}"]) == n


@pytest.mark.parametrize("ncols", R.NCOLS)
def test_layout(ncols):
    runs = R.streams()["lengths"]
    keys = R.layout(runs, ncols)
    assert len(keys) == sum(runs) and (np.diff(keys) > 0).all() and keys[-1] < 2**63 - 1
    g, starts = R.heads(keys, ncols)
    counts = np.diff(np.r_[starts, len(keys)])
    assert counts.max() <= ncols
    if ncols >= max(runs):  # every run is one group
        assert np.array_equal(counts, runs)
    if 1 < ncols <= max(runs):
        assert (counts == ncols).any() and (counts < ncols).any()


def test_ordered_fold_is_a_left_fold():
    rng = np.random.default_rng(0)
    for T in (np.float32, np.float64):
        keys = R.layout([1, 2, 3, 5, 8, 13, 40] * 30, 64)
        v = R.extrema_values(np.dtype(T), keys, 64, rng)
        _, starts = R.heads(keys, 64)
        for method in (np.maximum, np.minimum, np.fmax, np.fmin):
            got = R.ordered_reduceat(method, v, starts)
            want = []
            for a, b in zip(starts, np.r_[starts[1:], len(v)]):
                acc = v[a:a + 1]
                for x in v[a + 1:b]:
                    acc = R.first_wins(method, acc, np.array([x]))
                want.append(acc[0])
            assert np.array_equal(R.bits(got), R.bits(np.array(want, T))), method.__name__
    # the rule itself: the earlier zero, the earlier NaN
    nan = R.qnans(np.float64)
    z = np.array([0.0]), np.array([-0.0])
    assert not np.signbit(R.first_wins(np.maximum, *z))[0] and np.signbit(R.first_wins(np.minimum, z[1], z[0]))[0]
    assert R.bits(R.first_wins(np.maximum, nan[1:2], nan[0:1]))[0] == R.bits(nan[1:2])[0]
    assert R.bits(R.first_wins(np.fmax, nan[1:2], np.array([1.0])))[0] == R.bits(np.array([1.0]))[0]


def _golden_cases():
    out = []
    plain = {"sum": (np.add, None), "prod": (np.multiply, None), "max": (np.maximum, None), "min": (np.minimum, None),
             "any": (np.logical_or, None), "all": (np.logical_and, None), "nansum": (np.add, 0),
             "nanprod": (np.multiply, 1), "nanmax": (np.fmax, None), "nanmin": (np.fmin, None)}
    for name in ("reduce_api", "nanreduce_api"):
        for i, c in enumerate(load(name)):
            if c["op"] in plain and c["fmt"] == "coo":
                out.append(pytest.param(c, plain[c["op"]], id=f"{name}-{i}-{c['op']}-{c['dtype']}-ax{c['axis']}"))
    return out


@pytest.mark.parametrize("c,rule", _golden_cases())
def test_restatement_matches_the_reference_goldens(c, rule):
    method, nan_to = rule
    a, w = c.sub("a_"), c.sub("out_")
    data, fill = np.array(a["data"]), np.asarray(a["fill"])[()]
    if nan_to is not None and data.dtype.kind == "f":  # _replace_nan: stored values and the fill value
        data = np.where(np.isnan(data), data.dtype.type(nan_to), data)
        fill = fill.dtype.type(nan_to) if np.isnan(fill) else fill
    axis = c["axis"]
    axis = tuple(axis) if isinstance(axis, list) else axis
    shape = tuple(int(s) for s in a["shape"])
    if method in (np.logical_or, np.logical_and):
        data = data.astype(bool)  # any / all reduce truth values
        fill = np.bool_(fill)
    coords, vals, rf, kshape = R.restate_api(a["coords"], data, shape, fill, method, axis)
    assert w["fill"].dtype == vals.dtype, (w["fill"].dtype, vals.dtype)
    # float sums and products: NumPy's reduceat order is its own, so rounding may differ (by at most a few ulps here)
    rounding = method in (np.add, np.multiply) and vals.dtype.kind == "f"

    def same(got, want):
        got, want = np.asarray(got), np.asarray(want)
        if rounding:
            return np.allclose(got, want, rtol=16 * np.finfo(got.dtype).eps, atol=0, equal_nan=True)
        return np.array_equal(R.bits(got), R.bits(want))

    if not kshape:  # 0-d: one stored value, or none and the fill value
        v = vals[:1] if len(vals) else np.array([rf])
        assert same(v, w["data"][:1] if len(w["data"]) else np.array([w["fill"][()]]))
        return
    assert R.bits(np.array([rf]))[0] == R.bits(np.array([w["fill"][()]]))[0]
    if c["keepdims"]:
        red = set(range(len(shape))) - set(d for d in range(len(shape)) if d not in
                                          (tuple(range(len(shape))) if axis is None else
                                           tuple(x % len(shape) for x in (axis if isinstance(axis, tuple) else (axis,)))))
        full = np.zeros((len(shape), coords.shape[1]), np.int64)
        full[[d for d in range(len(shape)) if d not in red]] = coords
        coords = full
    assert np.array_equal(coords, w["coords"])
    assert same(vals, w["data"])


def test_error_bound_sees_one_entry():
    """For a group of 64 entries of similar magnitude the bound is far below any entry, for sums and products: a
    dropped or duplicated entry cannot hide in it (the fixed rtol of the golden tests is above one entry at these
    sizes)."""
    rng = np.random.default_rng(1)
    starts = np.array([0])
    for T in (np.dtype(np.float32), np.dtype(np.float64)):
        v = (rng.uniform(1, 2, size=64) * rng.choice([-1, 1], size=64)).astype(T)
        for method in (np.add, np.multiply):
            want = method.reduce(v.astype(np.float64))
            _, err, bound = R.group_errors(method, np.array([want], T), v, starts, 64, T.type(1), T)
            assert err[0] <= bound[0] < 1e-3 * np.abs(v).min() * (abs(want) if method is np.multiply else 1)
            _, err, _ = R.group_errors(method, np.array([want * (1 + 1e-3)], T), v, starts, 64, T.type(1), T)
            assert err[0] > bound[0]


@pytest.mark.parametrize("method", [np.add, np.multiply], ids=lambda m: m.__name__)
def test_fraction_fallback_agrees_with_long_double(method):
    """The exact rational reference used for float64 where long double is short gives the errors of the long double
    one, on short groups and with fills."""
    if not R.long_double_ok():
        pytest.skip("needs a long double with at least 63 mantissa bits to compare with")
    rng = np.random.default_rng(5)
    T = np.dtype(np.float64)
    keys = R.layout(R._random_runs(20_000, rng), 4096)
    _, starts = R.heads(keys, 4096)
    vals = R.random_floats(T, len(keys), rng) if method is np.add else R.random_factors(T, len(keys), rng)
    fill = T.type(1.25 if method is np.add else -1.0)
    _, got, _, _ = R.restate(method, keys, vals, 4096, fill)
    ok_l, err_l, bound_l = R.group_errors(method, got, vals, starts, 4096, fill, T)
    ok_f, err_f, bound_f = R.group_errors(method, got, vals, starts, 4096, fill, T, fraction=True)
    assert ok_f.sum() > 50 and ok_l.all()
    assert (err_f[ok_f] <= bound_f[ok_f]).all()
    # the long double reference is itself within ~2^-64 of the sum: far below the bound
    assert (np.abs(err_f - err_l)[ok_f] <= 1e-2 * bound_f[ok_f]).all()
    assert np.allclose(bound_f[ok_f], bound_l[ok_f], rtol=1e-9)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: kernel level
# ---------------------------------------------------------------------------------------------------------------------
def _kn():
    import _mock_kernels

    _mock_kernels.uninstall()
    from sparse_b200 import _device as D
    from sparse_b200 import _kernels as Kn
    from sparse_b200 import _lib

    _lib.load()
    return Kn, D


def _run(Kn, D, op, keys_d, vals, ncols, fill, rfill, form):
    Kn.reduce_set_form(form)
    try:
        _, gids, out, neq = Kn.reduce_fused(op, keys_d, D.upload(vals), ncols, fill, rfill, (1,), want_coords=False)
    finally:
        Kn.reduce_set_form(0)
    return D.download(gids), D.download(out), neq


def _fills(op, T):
    if T == np.bool_:
        return [np.False_, np.True_]
    if T.kind in "iu":
        ii = np.iinfo(T)
        return [T.type(v) for v in (0, -1, 7, ii.min, ii.max)]
    if op == 0:
        return [T.type(v) for v in (0.0, 0.25, -1.5, -0.0)]
    if op == 1:
        return [T.type(v) for v in (1.0, -1.0, 2.0, 0.5)]
    return [T.type(v) for v in (0.0, -0.0, np.inf, -np.inf, 1.0)] + list(R.qnans(T)[:1])


def _values(op, T, keys, ncols, rng):
    if T == np.bool_:
        return R.bool_values(keys, ncols, rng)
    if T.kind in "iu":
        return R.int_values(T, len(keys), rng)
    if op == 0:
        return R.exact_sum_values(T, len(keys), rng)
    if op == 1:
        return R.exact_prod_values(T, len(keys), rng)
    return R.extrema_values(T, keys, ncols, rng)


def _pow_ulps(op, T):
    """float64 fill ** n_fill is CUDA's pow (2 ulps), so a float64 product with the fill step may be that far off
    NumPy's; float32's goes through double and rounds once, add is exact."""
    return 4 if op == 1 and T == np.float64 else 0


BIG = "tiles5000"
BIG_NCOLS = (1, 2048, 2049, 2**40 + 1)  # the ~5000-tile stream: both sides of the form threshold and the extremes
RANDOM_MAX = 300_000  # random-float streams (bound check) up to this length


def _describe(stream, ncols, form, fill):
    return f"stream {stream}, ncols {ncols}, form {form}, fill {fill!r}"


def _check_exact(got, want, what, computed_nan=False, ulps=0):
    """Group ids, value bits and n_equal_fill equal.  With `computed_nan` (float add / multiply) a NaN the arithmetic
    made only has to be a NaN: its bits are unspecified, so a NaN result fill is not counted either.  `ulps` allows
    that many ulps on finite values (float64 fill ** n_fill comes from the device's pow)."""
    gg, gv, neq = got
    wg, wv, wneq = want
    assert np.array_equal(gg, wg), f"{what}: group ids ({len(gg)} vs {len(wg)})"
    bad = R.bits(gv) != R.bits(wv)
    if computed_nan:
        bad &= ~(np.isnan(gv) & np.isnan(wv))
    if ulps:
        with np.errstate(all="ignore"):
            bad &= ~(np.isfinite(wv) & (np.abs(gv - wv) <= ulps * np.spacing(np.abs(wv))))
    bad = np.flatnonzero(bad)
    assert len(bad) == 0, (f"{what}: {len(bad)} values differ, first at group {wg[bad[0]]}: got {gv[bad[0]]!r} "
                           f"want {wv[bad[0]]!r}")
    if computed_nan and np.isnan(wv).any():
        assert neq <= wneq + int(np.isnan(wv).sum()), f"{what}: n_equal_fill {neq}"
    else:
        assert neq == wneq, f"{what}: n_equal_fill {neq} != {wneq}"


@gpu
@pytest.mark.parametrize("op,T", CASES)
def test_kernel_streams(op, T):
    """Every stream x ncols x form: group ids exact, values bit for bit, n_equal_fill exact."""
    Kn, D = _kn()
    method = R.OPS[op]
    fills = _fills(op, T)
    rng = np.random.default_rng(zlib.crc32(f"{op}-{T.name}".encode()))
    for si, stream in enumerate(R.streams()):
        for ci, ncols in enumerate(R.NCOLS):
            if stream == BIG and ncols not in BIG_NCOLS:
                continue
            keys = R.stream_keys(stream, ncols)
            kd = D.upload(keys)
            vals = _values(op, T, keys, ncols, rng)
            fill = fills[(si + ci) % len(fills)]
            wg, wv, _, rfill = R.restate(method, keys, vals, ncols, fill)
            want = (wg, wv, R.n_equal(wv, rfill))
            for form in (1, 2):
                _check_exact(_run(Kn, D, op, kd, vals, ncols, fill, rfill, form), want,
                             _describe(stream, ncols, form, fill), computed_nan=op in (0, 1) and T.kind == "f", ulps=_pow_ulps(op, T))


@gpu
@pytest.mark.parametrize("op,T", [p for p in FLOAT_CASES if p.values[0] in (0, 1)])
def test_kernel_random_arithmetic(op, T):
    """Random floats: every group sum (with cancellation) within gamma_{n+1} (sum |x| + |fill| n_fill) of the exact one,
    every group product within gamma_{n+1} |exact|; exact in float64 for float32 data, in long double for float64 data
    (or as fractions on short groups without a long double of 63 mantissa bits)."""
    Kn, D = _kn()
    method = R.OPS[op]
    rng = np.random.default_rng(7 + T.itemsize + op)
    for si, (stream, runs) in enumerate(R.streams().items()):
        if sum(runs) > RANDOM_MAX:
            continue
        for ncols in R.NCOLS:
            keys = R.stream_keys(stream, ncols)
            if op == 0:
                vals = R.random_floats(T, len(keys), rng)
                fill = T.type(0.0 if si % 2 else 1.25)
            else:
                vals = R.random_factors(T, len(keys), rng)
                fill = T.type(1.0 if si % 2 else -1.0)
            g, starts = R.heads(keys, ncols)
            rfill = R.result_fill(method, fill, ncols, T)
            for form in (1, 2):
                gg, gv, neq = _run(Kn, D, op, D.upload(keys), vals, ncols, fill, rfill, form)
                what = _describe(stream, ncols, form, fill)
                assert np.array_equal(gg, g[starts]), f"{what}: group ids"
                checked, err, bound = R.group_errors(method, gv, vals, starts, ncols, fill, T)
                bad = np.flatnonzero(checked & ~(err <= bound))
                assert checked.any() and len(bad) == 0, \
                    f"{what}: {len(bad)} results outside the bound, e.g. group {g[starts][bad[0]]}: {gv[bad[0]]!r}"
                assert neq == R.n_equal(gv, rfill), what


def _fill_matrix_fills(op, T):
    if T == np.bool_:
        return [np.False_, np.True_]
    if T.kind in "iu":
        ii = np.iinfo(T)
        return [T.type(v) for v in (0, 1, -1, 3, ii.min, ii.max)]
    huge = T.type(3e38 if T == np.float32 else 1.5e308)
    return [T.type(v) for v in (0.0, -0.0, 1.5, -3.0, np.inf, -np.inf)] + [R.qnans(T)[1], huge, -huge,
                                                                           T.type(0.5), T.type(2.0**-70)]


@gpu
@pytest.mark.parametrize("op,T", CASES)
def test_fill_matrix(op, T):
    """Every fill (0, -0.0, non-zero, NaN, +-inf, huge, a tiny product base) on groups that are complete, miss one
    entry, or miss more than 2^24 (float32's (T) n_fill would round), under both forms: bit for bit, add included."""
    Kn, D = _kn()
    method = R.OPS[op]
    rng = np.random.default_rng(zlib.crc32(f"fill-{op}-{T.name}".encode()))
    for ncols in (1, 3, 2048, 2**24 + 3, 2**40 + 1):
        # per group: complete (when ncols is small), one entry missing, most missing; 1..3 entries otherwise
        lens = [min(ncols, k) for k in (1, 2, 3, ncols, max(ncols - 1, 1), 2, 1)] * 40
        lens = [L for L in lens if L <= 3000]
        keys = R.layout(lens, ncols, seed=ncols % 97)
        for fill in _fill_matrix_fills(op, T):
            if T.kind == "f" and op == 0:
                vals = np.concatenate([R.exact_sum_values(T, len(keys) - 3, rng),
                                       np.array([T.type(-3e38 if T == np.float32 else -1.5e308), 1, 0], T)])
            elif T.kind == "f" and op == 1:
                vals = R.exact_prod_values(T, len(keys), rng)
                vals[::7] = T.type(2.0**100)
            else:
                vals = _values(op, T, keys, ncols, rng)
            wg, wv, _, rfill = R.restate(method, keys, vals, ncols, fill)
            for form in (1, 2):
                _check_exact(_run(Kn, D, op, D.upload(keys), vals, ncols, fill, rfill, form),
                             (wg, wv, R.n_equal(wv, rfill)), f"ncols {ncols}, form {form}, fill {fill!r}",
                             computed_nan=op in (0, 1) and T.kind == "f", ulps=_pow_ulps(op, T))


@gpu
@pytest.mark.parametrize("form", [1, 2])
def test_fill_power_of_two_past_2_53_fills(form):
    """A product whose groups miss about 2^62 entries, with power-of-two fills far from 1: fill ** n_fill saturates to
    inf or 0 (with the sign of an odd count), exactly as NumPy's pow does."""
    Kn, D = _kn()
    T = np.dtype(np.float64)
    ncols = 2**62
    keys = np.array([0, 1, 7, ncols + 5], np.int64)
    vals = np.array([0.75, -2.0, 3.0, 1.5], T)
    for fill in (2.0**1000, 2.0**-1000, -(2.0**-1000), -(2.0**1000), 2.0**-1074, 1.0, -1.0):
        fill = T.type(fill)
        wg, wv, _, rfill = R.restate(np.multiply, keys, vals, ncols, fill)
        _check_exact(_run(Kn, D, 1, D.upload(keys), vals, ncols, fill, rfill, form), (wg, wv, R.n_equal(wv, rfill)),
                     f"fill {fill!r}")


@gpu
@pytest.mark.parametrize("T", [np.dtype(np.float32), np.dtype(np.float64)], ids=lambda t: t.name)
def test_prune_at_tile_edges(T):
    """Results equal to the result fill at tile starts, at tile ends and in a run the two-pass form finishes by reading
    ahead; a -0.0 result beside a +0.0 fill stays stored.  Kernel counts and API output."""
    Kn, D = _kn()
    ncols = 4096
    # runs: 2047 singles | a run over the tile boundary (read-ahead) | runs ending on the last entry of tile 1 | ...
    runs = [1] * 2047 + [60] + [2] * 994 + [1] + [2048] + [1] * 100
    keys = R.layout(runs, ncols)
    g, starts = R.heads(keys, ncols)
    vals = R.exact_sum_values(T, len(keys), np.random.default_rng(3))
    ends = np.r_[starts[1:], len(keys)] - 1
    # groups cancelling to exactly 0 at tile starts and tile ends, and the read-ahead run
    zero_groups = [i for i in range(len(starts)) if starts[i] % R.TILE == 0 or ends[i] % R.TILE == R.TILE - 1
                   or (starts[i] // R.TILE) != (ends[i] // R.TILE)]
    assert len(zero_groups) >= 4
    for i in zero_groups:
        seg = vals[starts[i]:ends[i] + 1]
        seg[-1] = -(seg[:-1].sum()) if len(seg) > 1 else 0.0
    neg = [i for i in range(len(starts)) if i % 5 == 3 and i not in zero_groups][:20]
    for form in (1, 2):
        for op, fill in ((0, 0.0), (1, 1.0)):
            v = vals.copy()
            if op == 1:
                v = np.where(v == 0, T.type(1), v)
                for i in zero_groups:
                    v[starts[i]] = 0.0
                for i in neg:
                    v[starts[i]] = -0.0
                    v[starts[i] + 1:ends[i] + 1] = np.abs(v[starts[i] + 1:ends[i] + 1])
            fill = T.type(fill)
            wg, wv, _, rfill = R.restate(R.OPS[op], keys, v, ncols, fill)
            got = _run(Kn, D, op, D.upload(keys), v, ncols, fill, rfill, form)
            _check_exact(got, (wg, wv, R.n_equal(wv, rfill)), f"op {op} form {form}")
            assert R.n_equal(wv, rfill) >= len(zero_groups) - 1
    # through the API: prod of complete groups (n_fill 0) keeps a -0.0 result, fill +0.0
    import sparse_b200 as sb

    d = np.array([[-0.0, 1.0], [0.0, 2.0], [3.0, -0.0]], T)
    x = sb.COO(np.array([[0, 0, 1, 1, 2, 2], [0, 1, 0, 1, 0, 1]]), d.reshape(-1), shape=(3, 2),
               has_duplicates=False, sorted=True, fill_value=T.type(0))
    r = x.prod(axis=1)
    assert r.coords.tolist() == [[0, 2]] and np.signbit(np.asarray(r.data)).all()


# ---------------------------------------------------------------------------------------------------------------------
# public API (mock kernels on a CPU box, CUDA kernels on an H100)
# ---------------------------------------------------------------------------------------------------------------------
AXES = [("trailing", 2), ("leading", 0), ("middle", 1), ("last-two", (1, 2)), ("all", None)]
API_OPS = [("sum", np.add), ("prod", np.multiply), ("max", np.maximum), ("min", np.minimum),
           ("any", np.logical_or), ("all", np.logical_and), ("nansum", np.add), ("nanmax", np.fmax),
           ("nanmin", np.fmin), ("bitwise_and", np.bitwise_and), ("bitwise_or", np.bitwise_or),
           ("bitwise_xor", np.bitwise_xor)]
API_DTYPES = ["float32", "int8", "uint8", "int16", "uint64"]


def _api_array(T, rng):
    """A (23, 37, 41) array, ~15% stored.  float32: quarters, some NaN, fill 0.5 (sums and products stay exact);
    integers: the whole range, fill 0; uint64 values above 2^63 included."""
    shape = (23, 37, 41)
    size = int(np.prod(shape))
    lin = np.sort(rng.choice(size, size=size * 15 // 100, replace=False))
    coords = np.stack(np.unravel_index(lin, shape))
    n = len(lin)
    if T == np.float32:
        data = (rng.integers(1, 9, size=n) / 4.0 * rng.choice([-1, 1], size=n)).astype(T)
        data[rng.random(n) < 0.02] = np.nan
        return coords, data, shape, T.type(0.5)
    ii = np.iinfo(T)
    data = rng.integers(ii.min, ii.max, size=n, dtype=T, endpoint=True)
    data[data == 0] = 1
    return coords, data, shape, T.type(0)


def _api_call(sp, x, name, axis):  # noqa: F811
    if name.startswith("bitwise"):
        return x.reduce(getattr(np, name), axis=axis)
    if name.startswith("nan"):
        return getattr(sp, name)(x, axis=axis)
    return getattr(x, name)(axis=axis)


def _api_case_ok(name, T):
    if name.startswith("bitwise") and T.kind == "f":
        return False
    if name in ("any", "all") and T.kind == "f":  # a non-zero fill: the result would be dense
        return False
    return T != np.uint64 or name in ("max", "min", "bitwise_and", "bitwise_or", "bitwise_xor")


@pytest.mark.parametrize("fmt", ["coo", "gcxs"])
@pytest.mark.parametrize("dt", API_DTYPES)
def test_api_reductions(sp, dt, fmt):  # noqa: F811
    """sum / prod / max / min / any / all / nansum / nanmax / nanmin / reduce(bitwise_*) over trailing, leading, middle
    and all axes: coordinates, fill value and dtype exact, values bit for bit (extrema by value: the stored data hold
    no signed zeros, and a NaN only has to be a NaN)."""
    import warnings

    T = np.dtype(dt)
    rng = np.random.default_rng(zlib.crc32(dt.encode()))
    coords, data, shape, fill = _api_array(T, rng)
    x = sp.COO(coords, data, shape=shape, has_duplicates=False, sorted=True, fill_value=fill)
    if fmt == "gcxs":
        x = x.asformat("gcxs", compressed_axes=(1,))
    for name, method in API_OPS:
        if not _api_case_ok(name, T):
            continue
        for label, axis in AXES:
            what = f"{name} {dt} {fmt} axis {label}"
            d, f = data, fill
            if name in ("nansum",) and T.kind == "f":
                d = np.where(np.isnan(d), T.type(0), d)
            if name in ("any", "all"):
                d, f = d.astype(bool), np.bool_(f)
            with np.errstate(all="ignore"), warnings.catch_warnings():
                warnings.simplefilter("ignore")
                got = _api_call(sp, x, name, axis)
            wc, wv, wf, kshape = R.restate_api(coords, d, shape, f, method, axis)
            got_c = got.asformat("coo") if hasattr(got, "asformat") else got
            assert got_c.dtype == wv.dtype, f"{what}: dtype {got_c.dtype} != {wv.dtype}"
            if not kshape:
                v = wv[0] if len(wv) else wf
                gv = np.asarray(got_c.todense()).reshape(())
                assert (np.isnan(v) and np.isnan(gv)) if T.kind == "f" and np.isnan(v) else gv == v, what
                continue
            assert tuple(got_c.shape) == kshape, what
            assert R.bits(np.array([got_c.fill_value], wv.dtype))[0] == R.bits(np.array([wf], wv.dtype))[0], what
            assert np.array_equal(np.asarray(got_c.coords), wc), f"{what}: coordinates"
            gd = np.asarray(got_c.data)
            if method in R.EXTREMA and T.kind == "f":
                assert np.array_equal(gd, wv, equal_nan=True), f"{what}: values"
            else:  # a NaN that arithmetic made (a sum or product over a stored NaN) only has to be a NaN
                nan = np.isnan(gd) & np.isnan(wv) if T.kind == "f" else np.zeros(len(gd), bool)
                assert np.array_equal(np.where(nan, 0, R.bits(gd)), np.where(nan, 0, R.bits(wv))), f"{what}: values"


def test_api_f32_sum_fill_overflow_regression(sp):  # noqa: F811
    """fill * n_fill overflows float32 on its own (3e38 * 2) but not the result: the fill step runs in float64, as in
    NumPy, and row 0 is 3e38, stored; row 1 is inf, the result fill, and pruned."""
    x = sp.COO(np.array([[0, 1], [0, 0]]), np.array([-3e38, 1], np.float32), shape=(2, 3), has_duplicates=False,
               sorted=True, fill_value=np.float32(3e38))
    r = x.sum(axis=1)
    assert r.dtype == np.float32 and np.isposinf(r.fill_value)
    assert np.asarray(r.coords).tolist() == [[0]]
    assert np.asarray(r.data).tolist() == [np.float32(3e38)]


def test_api_f32_prod_fill_underflow_regression(sp):  # noqa: F811
    """fill ** n_fill underflows float32 on its own (0.5 ** 150) but not the result: 2^100 * 0.5^150 = 2^-50 and
    3 * 0.5^150 rounds to the subnormal 2^-148, both stored; the result fill 0.5^151 is 0."""
    x = sp.COO(np.array([[0, 1], [0, 0]]), np.array([2.0**100, 3], np.float32), shape=(2, 151), has_duplicates=False,
               sorted=True, fill_value=np.float32(0.5))
    r = x.prod(axis=1)
    assert r.dtype == np.float32 and r.fill_value == 0
    assert np.asarray(r.coords).tolist() == [[0, 1]]
    assert R.bits(np.asarray(r.data)).tolist() == R.bits(np.array([2.0**-50, 2.0**-148], np.float32)).tolist()
    assert math.isclose(float(r.data[1]), 2.8e-45, rel_tol=0.01)


def test_api_f32_prod_fill_steps_match_the_reference(sp):  # noqa: F811
    """float32 1.3 over 151 columns, as the reference computes it: the result fill 1.3 ** 151 in float32 arithmetic
    (its n_cols is a Python int) is 1.6048846e17, while each row's fill step 1.3 ** 150 goes through float64 (n_fill is
    an int64 array) and rounds once: row 0 is 1.6048845e17, one ulp below the result fill, so both rows stay stored."""
    x = sp.COO(np.array([[0, 1], [0, 0]]), np.array([1.3, 3.0], np.float32), shape=(2, 151), has_duplicates=False,
               sorted=True, fill_value=np.float32(1.3))
    r = x.prod(axis=1)
    rfill = np.float32(1.6048846e17)
    assert R.bits(np.array([np.power(np.float32(1.3), 151)]))[0] == R.bits(np.array([rfill]))[0]
    assert R.bits(np.array([r.fill_value], np.float32))[0] == R.bits(np.array([rfill]))[0]
    assert np.asarray(r.coords).tolist() == [[0, 1]]
    f = np.power(np.float64(np.float32(1.3)), 150)
    want = np.array([np.float64(np.float32(1.3)) * f, 3 * f]).astype(np.float32)
    assert want[0] == np.float32(1.6048845e17) and want[0] != rfill
    assert R.bits(np.asarray(r.data)).tolist() == R.bits(want).tolist()


def test_api_f64_prod_power_of_two_fill_regression(sp):  # noqa: F811
    """fill ** n_fill for a power-of-two fill is exact (CUDA's pow was an ulp off for 0.5 ** 6): 0.5 * 0.5 ** 6 equals
    the result fill 0.5 ** 7 and is pruned; 0.25 * 0.5 ** 6 = 2^-8 and -4 * 0.5 ** 6 = -2^-4 are stored exactly."""
    x = sp.COO(np.array([[0, 1, 2], [3, 0, 6]]), np.array([0.5, 0.25, -4.0]), shape=(4, 7), has_duplicates=False,
               sorted=True, fill_value=0.5)
    r = x.prod(axis=1)
    assert r.fill_value == 0.5**7
    assert np.asarray(r.coords).tolist() == [[1, 2]]
    assert R.bits(np.asarray(r.data)).tolist() == R.bits(np.array([2.0**-8, -(2.0**-4)])).tolist()
