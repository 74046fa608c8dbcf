"""The element-wise op table (K5, csrc/elemwise.cu), op by op, dtype by dtype and kernel form by kernel form.

Every binary and unary op code runs on the map kernel (scalar on the right, on the left, unary), the dense gather
(both operand orders) and the fused merge, for every compute dtype in which NumPy keeps the op's result type, on the
special values and ~10^5 random values of tests/_ew_ops.py.  Exact ops are compared bit for bit with NumPy,
transcendental ones with a higher-precision reference within the CUDA math library's ulp budgets; the rules are in
_ew_ops.py.  Then the merge's tile structure (pairs split at tile boundaries, tile counts around the look-back window,
runs of fully pruned tiles, virtual trailing broadcasts, tiny operands), the dense gather's index arithmetic, the
broadcast expansion, and the integer ops fixed alongside these tests through the public API.

The CPU tests at the top check the generators, the ulp measure and the references on any machine."""
import zlib

import numpy as np
import pytest

import _ew_ops as E
from _api import sp  # noqa: F401  (fixture: the mock kernels on a CPU box, the CUDA kernels on a GPU box)

gpu = pytest.mark.gpu


def _tables():
    from sparse_b200 import _elemwise

    return _elemwise


def _op_cases(binary):
    """(name, dtype) for every op code and compute dtype where NumPy keeps the result in that dtype (bool for
    predicates)."""
    ew = _tables()
    table = ew._BINARY if binary else ew._UNARY
    cases = []
    for func in table:
        name = func.__name__
        for T in E.DTYPES:
            z = np.empty(0, T)
            try:
                out_dt, ct = ew._resolve(func, z, z) if binary else ew._resolve(func, z)
            except TypeError:
                continue
            pred = name in (E.PREDICATES_BIN if binary else E.PREDICATES_UN)
            if ct == T and (out_dt == (np.bool_ if pred else T)):
                cases.append(pytest.param(name, T, id=f"{name}-{T.name}"))
    return cases


BIN_CASES = _op_cases(True)
UN_CASES = _op_cases(False)


def _func(name, binary):
    table = _tables()._BINARY if binary else _tables()._UNARY
    return next(f for f in table if f.__name__ == name)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: generators, ulp measure, references
# ---------------------------------------------------------------------------------------------------------------------
def test_every_op_code_has_a_case():
    ew = _tables()
    assert {f.__name__ for f in ew._BINARY} == {p.values[0] for p in BIN_CASES}
    assert {f.__name__ for f in ew._UNARY} == {p.values[0] for p in UN_CASES}
    assert {n for n, _ in STRUCT_OPS} <= {p.values[0] for p in BIN_CASES}


@pytest.mark.parametrize("s", range(7))
def test_split_pairs_fall_across_tile_boundaries(s):
    """Replay of the merge path (ties to A): with s odd every tile boundary has A's copy of a key as the tile's last
    position and B's copy as the next tile's first; with s even the boundaries fall between keys."""
    ka, kb = E.split_pair_streams(s, 3 * E.TILE + 5)
    from_a, keys = E.merged_sources(ka, kb)
    total = len(ka) + len(kb)
    bounds = range(E.TILE, total, E.TILE)
    assert len(bounds) >= 3
    for d in bounds:
        split = bool(from_a[d - 1] and not from_a[d] and keys[d - 1] == keys[d])
        assert split == (s % 2 == 1), (s, d)
    # for every s, some thread boundary (multiple of 7) splits a pair
    tb = np.arange(E.ITEMS, total, E.ITEMS)
    assert (from_a[tb - 1] & ~from_a[tb] & (keys[tb - 1] == keys[tb])).any()


@pytest.mark.parametrize("tiles", [1, 2, 63, 64, 65, 129, 5003])
def test_tile_count_streams(tiles):
    ka, kb = E.tile_count_streams(tiles, np.random.default_rng(tiles))
    assert E.tiles_of(len(ka) + len(kb)) == tiles
    assert (np.diff(ka) > 0).all() and (np.diff(kb) > 0).all()
    assert len(np.intersect1d(ka, kb)) > 0 and len(np.setdiff1d(ka, kb)) > 0 and len(np.setdiff1d(kb, ka)) > 0


PRUNED_PATTERN = "PP" + "K" + "P" * 70 + "KK" + "P" + "K" + "PPP"


def test_pruned_tile_streams():
    ka, kb, cancel = E.pruned_tile_streams(PRUNED_PATTERN, np.random.default_rng(0))
    from_a, keys = E.merged_sources(ka, kb)
    assert E.tiles_of(len(ka) + len(kb)) == len(PRUNED_PATTERN)
    a_pos = np.cumsum(from_a) - 1                   # index into A of each merged A item
    kept = np.zeros(len(keys), bool)
    kept[from_a] = ~cancel[a_pos[from_a]]
    per_tile = np.add.reduceat(kept.astype(np.int64), np.arange(0, len(keys), E.TILE))
    assert ((per_tile == 0) == np.array([c == "P" for c in PRUNED_PATTERN])).all()
    assert per_tile[0] == 0 and per_tile[-1] == 0
    best = run = 0
    for empty in per_tile == 0:
        run = run + 1 if empty else 0
        best = max(best, run)
    assert best > E.LOOKBACK
    # a cancelled A entry always has its B twin
    assert np.isin(ka[cancel], kb).all() and not np.isin(ka[~cancel], kb).any()


@pytest.mark.parametrize("R", [2, 3, 7, 64, 1000, 65537])
@pytest.mark.parametrize("both", [False, True])
def test_broadcast_streams(R, both):
    rng = np.random.default_rng(R)
    n = max(2, 200_000 // R)
    pa, Ra, kb, Rb = E.broadcast_streams(R, both, n, rng, top=True)
    ea, eb = E.expand(pa, Ra), E.expand(kb, Rb)
    assert (np.diff(ea) > 0).all() and (np.diff(eb) > 0).all()
    top = max(ea[-1], eb[-1])
    assert np.iinfo(np.int64).max - top < 8 * n * R
    assert len(np.intersect1d(ea, eb)) > 0


def test_ulp_error_on_hand_picked_pairs():
    f32 = np.dtype(np.float32)
    e = lambda got, ref, T=f32: float(E.ulp_error(np.array([got], T), np.array([ref], E.hp_dtype(T)), T)[0])  # noqa
    assert e(1.0, 1.0) == 0
    assert e(np.nextafter(np.float32(1), np.float32(2)), 1.0) == 1
    assert e(np.nextafter(np.float32(1), np.float32(0)), 1.0) == 0.5          # below 2^0 the spacing halves
    assert e(np.float32(1), 1.0 - 2.0 ** -24) == 1                           # ulp at the reference, not at got
    sub = np.finfo(f32).smallest_subnormal
    assert e(sub, 0.0) == 1 and e(3 * sub, float(sub)) == 2
    assert e(0.0, float(sub) / 4) == 0.25
    assert e(-0.0, 0.0) == 0 and e(0.0, -0.0) == 0
    assert e(np.inf, float(np.finfo(f32).max)) == 1                           # +inf counts as 2^128
    f64 = np.dtype(np.float64)
    if np.finfo(np.longdouble).nmant >= 63:
        one = np.longdouble(1)
        assert e(np.nextafter(1.0, 2.0), one, f64) == 1
        assert e(1.0, one + np.ldexp(one, -54), f64) == 0.25


def test_pinned_literals_and_rules_agree_with_numpy_here():
    with np.errstate(all="ignore"):
        for T in E.INTS:
            lo = np.iinfo(T).min
            a = np.array([lo, 5, -5, 0, lo, 7], T)
            b = np.array([-1, 0, 0, 0, 0, -1], T)
            for name in ("floor_divide", "remainder"):
                m, v = E.int_literals(name, a, b)
                assert m[:5].all() and np.array_equal(v[m], getattr(np, name)(a, b)[m]), name
            x = np.array([0, 1, -1, 2, -2, lo, np.iinfo(T).max], T)
            _, v = E.int_literals("reciprocal", x)
            assert np.array_equal(v, np.reciprocal(x))
        # rules of maximum / minimum (NaN first, +-0 tie -> second) and fmax / fmin (NaN loses, both NaN -> first)
        for T in E.FLOATS:
            a, b = E.pair_set(T, np.random.default_rng(1), 1000)
            for name in ("maximum", "minimum", "fmax", "fmin"):
                got = getattr(np, name)(a, b)
                bad = E.mismatches(name, T, got, a, b)
                assert not bad.any(), E.worst(name, T, got, a, b)
            assert E.exact_reference("maximum", np.array([0.0, -0.0]), np.array([-0.0, 0.0])).tolist() == [-0.0, 0.0]
            assert np.signbit(E.exact_reference("maximum", np.array([0.0]), np.array([-0.0])))[0]


@pytest.mark.parametrize("T", E.DTYPES, ids=lambda t: t.name)
def test_references_agree_with_numpy_here(T):
    """The exact references are NumPy's own results on the value sets; the transcendental references pass their own
    check; float32 rad2deg is x * (f32(180) / f32(pi)) bit for bit."""
    rng = np.random.default_rng(7)
    a, b = E.pair_set(T, rng, 20_000)
    x = E.unary_set(T, rng, 20_000)
    with np.errstate(all="ignore"):
        for p in BIN_CASES:
            name, t = p.values
            if t != T or E.is_transcendental(name, T) or name in E.PREDICATES_BIN:
                continue
            bb = E.nonneg_exponent(b) if name == "power" else b
            if name in ("nan_replace", "_sel_x", "_sel_y", "_bitor_raw"):
                got = getattr(_tables(), name)(a, bb)
            else:
                got = getattr(np, name)(a, bb)
            assert not E.mismatches(name, T, got, a, bb).any(), E.worst(name, T, got, a, bb)
        for p in UN_CASES:
            name, t = p.values
            if t != T or name in E.PREDICATES_UN:
                continue
            if E.is_transcendental(name, T):
                got = E.hp_reference(name, x).astype(T)  # the correctly rounded value is within every budget
            else:
                got = getattr(np, name)(x)
            assert not E.mismatches(name, T, got, x).any(), E.worst(name, T, got, x)
        if T == np.float32:
            k = np.float32(180) / np.float32(np.pi)
            assert k == np.float32(57.295776) and k != np.float32(57.29577951308232)
            assert np.array_equal(E.bits(np.rad2deg(x)), E.bits(x * k))


def test_mismatches_catch_one_ulp_and_fma_variants():
    """The comparison would see a kernel that is off by one ulp in an exact op, or contracts a * b + c."""
    rng = np.random.default_rng(3)
    for T in E.FLOATS:
        a, b = E.pair_set(T, rng, 5000)
        with np.errstate(all="ignore"):
            good = a * b
            off = np.nextafter(good, np.array(np.inf, T))
            assert E.mismatches("multiply", T, off, a, b).any()
            # rad2deg with the float64 constant rounded to T: the old kernel
            x = E.unary_set(T, rng, 5000)
            old = x * T.type(57.29577951308232)
            if T == np.float32:
                assert E.mismatches("rad2deg", T, old, x).any()
            # a transcendental two ulps past its budget (which is stated against the correctly rounded result; one ulp
            # past it can sit exactly on the allowed B + 1/2 within the long double reference's resolution)
            ref = E.hp_reference("exp", x)
            rT = ref.astype(T)
            fin = np.isfinite(rT) & (rT != 0) & ~E.special_input(x)
            budget = E.ULP_BUDGET["exp"][0 if T == np.float32 else 1]
            worse = rT.copy()
            for _ in range(budget + 2):
                worse = np.where(fin, np.nextafter(worse, np.array(np.inf, T)), worse)
            assert E.mismatches("exp", T, worse, x)[fin].all()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: op table x dtype x form
# ---------------------------------------------------------------------------------------------------------------------
def _kn():
    import _mock_kernels

    _mock_kernels.uninstall()
    from sparse_b200 import _device as D
    from sparse_b200 import _kernels as Kn
    from sparse_b200 import _lib

    _lib.load()
    return Kn, D


def _rng(name, T):
    return np.random.default_rng(zlib.crc32(f"{name}-{T.name}".encode()))


def _needs_long_double(name, T):
    if E.is_transcendental(name, T) and T == np.float64 and np.finfo(np.longdouble).nmant < 63:
        pytest.skip("the float64 reference needs a long double with at least 63 mantissa bits")


def _out_fill(func, out_dt, *fills):
    return np.asarray(_tables()._fill_of(func, *fills)).astype(out_dt)[()]


def _check_flags(vals, flags, out_fill, what):
    fb = E.bits(np.array([out_fill], dtype=vals.dtype))[0]
    want = E.bits(vals) != fb
    assert np.array_equal(flags.astype(bool), want), f"{what}: flags != bits(value) != bits(out_fill)"


def _check(name, T, got, a, b, what):
    bad = E.mismatches(name, T, got, a, b)
    assert not bad.any(), f"{what}: " + E.worst(name, T, got, a, b)


def _merge_check(Kn, D, name, T, out_dt, code, ka, da, Ra, kb, db, Rb, fa, fb, out_fill, what):
    """Run the fused merge and check: keys strictly increasing, a subset of the union; every union position absent
    from the output has a value whose bits equal out_fill, every one present has other bits; all values meet the op's
    contract against the restated union."""
    _, vals, keys = Kn.ew_merge_fused(code, D.upload(ka), D.upload(da), Ra, D.upload(kb), D.upload(db), Rb,
                                      T.type(fa), T.type(fb), out_fill, out_dt, (1,), want_coords=False)
    keys, vals = D.download(keys), D.download(vals)
    _, _, union, va, vb = E.union_oracle(name, ka, da, Ra, kb, db, Rb, fa, fb, out_fill)
    assert len(keys) == len(vals)
    assert (np.diff(keys) > 0).all(), f"{what}: output keys not in order"
    pos = np.searchsorted(union, keys)
    assert (pos < len(union)).all() and np.array_equal(union[np.minimum(pos, len(union) - 1)], keys), \
        f"{what}: output keys outside the union"
    fbits = E.bits(np.array([out_fill], dtype=out_dt))[0]
    assert (E.bits(vals) != fbits).all(), f"{what}: an output value equals the fill value"
    full = np.full(len(union), out_fill, dtype=out_dt)
    full[pos] = vals
    _check(name, T, full, va, vb, what)
    return keys, vals


@gpu
@pytest.mark.parametrize("name,T", BIN_CASES)
def test_binary_op_table(name, T):
    Kn, D = _kn()
    func = _func(name, True)
    code = _tables()._BINARY[func]
    pred = name in E.PREDICATES_BIN
    out_dt = np.dtype(np.bool_) if pred else T
    int_pow = name == "power" and T.kind == "i"
    _needs_long_double(name, T)
    rng = _rng(name, T)
    a, b = E.pair_set(T, rng)
    if int_pow:
        b = E.nonneg_exponent(b)
    fills = E.fill_values(T)
    # map: f(x, s) and f(s, x)
    x = E.unary_set(T, rng)
    xd = D.upload(x)
    for i, s in enumerate(E.scalar_set(T)):
        for mode in (0, 1):
            if int_pow and mode == 0 and s < 0:
                continue
            xs = E.nonneg_exponent(x) if (int_pow and mode == 1) else x
            src = D.upload(xs) if xs is not x else xd
            fill = fills[i % len(fills)]
            fill = E.nonneg_exponent(np.array([fill]))[0] if (int_pow and mode == 1) else fill
            of = _out_fill(func, out_dt, fill, s) if mode == 0 else _out_fill(func, out_dt, s, fill)
            vals, flags = Kn.ew_map(code, mode, src, T.type(s), of, out_dt)
            got, fl = D.download(vals), D.download(flags)
            full = np.full(len(xs), s, T)
            what = f"ew_map mode {mode}, scalar {s!r}"
            if mode == 0:
                _check(name, T, got, xs, full, what)
            else:
                _check(name, T, got, full, xs, what)
            _check_flags(got, fl, of, what)
    # dense gather, both operand orders
    n = len(a)
    for swap in (0, 1):
        sv, dv = (a, b) if swap == 0 else (b, a)
        of = _out_fill(func, out_dt, fills[1], fills[2] if not int_pow else T.type(7))
        keys, vals, flags = Kn.ew_dense(code, bool(swap), Kn.iota(n), D.upload(sv), 1, D.upload(dv), (n,), [1], of,
                                        out_dt)
        got = D.download(vals)
        assert np.array_equal(D.download(keys), np.arange(n))
        _check(name, T, got, a, b, f"ew_dense swap {swap}")
        _check_flags(got, D.download(flags), of, f"ew_dense swap {swap}")
    # fused merge: key 3i holds (a_i, b_i), 3i + 1 only a_i, 3i + 2 only b_i
    idx = np.arange(n, dtype=np.int64) * 3
    ka = np.sort(np.concatenate([idx, idx + 1]))
    kb = np.sort(np.concatenate([idx, idx + 2]))
    da = np.empty(2 * n, T)
    db = np.empty(2 * n, T)
    da[0::2], da[1::2] = a, a
    db[0::2], db[1::2] = b, b
    for j in range(len(fills)):
        fa, fb = fills[j], fills[(j + 1) % len(fills)] if j else fills[0]
        if int_pow:
            fb = E.nonneg_exponent(np.array([fb]))[0]
        of = _out_fill(func, out_dt, fa, fb)
        _merge_check(Kn, D, name, T, out_dt, code, ka, da, 1, kb, db, 1, fa, fb, of,
                     f"ew_merge_fused fills ({fa!r}, {fb!r})")


@gpu
@pytest.mark.parametrize("name,T", UN_CASES)
def test_unary_op_table(name, T):
    Kn, D = _kn()
    func = _func(name, False)
    code = _tables()._UNARY[func]
    out_dt = np.dtype(np.bool_) if name in E.PREDICATES_UN else T
    _needs_long_double(name, T)
    x = E.unary_set(T, _rng(name, T))
    xd = D.upload(x)
    for fill in E.fill_values(T):
        of = _out_fill(func, out_dt, fill)
        vals, flags = Kn.ew_map(code, 2, xd, None, of, out_dt)
        got = D.download(vals)
        _check(name, T, got, x, None, f"ew_map unary, fill {fill!r}")
        _check_flags(got, D.download(flags), of, f"ew_map unary, fill {fill!r}")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: merge structure
# ---------------------------------------------------------------------------------------------------------------------
STRUCT_OPS = [("add", np.dtype(np.int64)), ("not_equal", np.dtype(np.int64)), ("maximum", np.dtype(np.float64))]


def _data(name, T, n, rng):
    if T.kind == "i":
        return rng.integers(-50, 51, size=n).astype(T)
    v = rng.standard_normal(n)
    v[rng.random(n) < 0.05] = np.nan
    v[rng.random(n) < 0.05] = 0.0
    v[rng.random(n) < 0.05] = -0.0
    return v.astype(T)


def _struct_check(Kn, D, name, T, ka, da, Ra, kb, db, Rb, fa=0, fb=0, what=""):
    code = _tables()._BINARY[_func(name, True)]
    out_dt = np.dtype(np.bool_) if name in E.PREDICATES_BIN else T
    of = _out_fill(_func(name, True), out_dt, T.type(fa), T.type(fb))
    keys, vals = _merge_check(Kn, D, name, T, out_dt, code, ka, da, Ra, kb, db, Rb, fa, fb, of, what)
    wk, wv, _, _, _ = E.union_oracle(name, ka, da, Ra, kb, db, Rb, T.type(fa), T.type(fb), of)
    assert np.array_equal(keys, wk), f"{what}: kept keys"
    assert np.array_equal(E.bits(vals), E.bits(wv)), f"{what}: values"
    return keys


@gpu
@pytest.mark.parametrize("name,T", STRUCT_OPS, ids=[f"{n}-{t.name}" for n, t in STRUCT_OPS])
def test_merge_pairs_split_at_tile_boundaries(name, T):
    Kn, D = _kn()
    rng = np.random.default_rng(11)
    for s in range(7):
        ka, kb = E.split_pair_streams(s, 3 * E.TILE + 5)
        _struct_check(Kn, D, name, T, ka, _data(name, T, len(ka), rng), 1, kb, _data(name, T, len(kb), rng), 1,
                      7 if T.kind == "i" else 1.5, -1 if T.kind == "i" else -0.0, what=f"s={s}")


@gpu
@pytest.mark.parametrize("name,T", STRUCT_OPS, ids=[f"{n}-{t.name}" for n, t in STRUCT_OPS])
@pytest.mark.parametrize("tiles", [1, 2, 63, 64, 65, 129, 5003])
def test_merge_tile_counts(name, T, tiles):
    Kn, D = _kn()
    rng = np.random.default_rng(tiles)
    ka, kb = E.tile_count_streams(tiles, rng)
    _struct_check(Kn, D, name, T, ka, _data(name, T, len(ka), rng), 1, kb, _data(name, T, len(kb), rng), 1,
                  what=f"{tiles} tiles")


@gpu
@pytest.mark.parametrize("name,T", STRUCT_OPS, ids=[f"{n}-{t.name}" for n, t in STRUCT_OPS])
def test_merge_runs_of_pruned_tiles(name, T):
    Kn, D = _kn()
    rng = np.random.default_rng(5)
    ka, kb, cancel = E.pruned_tile_streams(PRUNED_PATTERN, rng)
    da = _data(name, T, len(ka), rng)
    if name == "maximum":
        da[cancel] = -1 - rng.random(int(cancel.sum()))  # max(negative, +0) = +0: the fill value
        da[~cancel] = np.abs(da[~cancel]) + 1      # kept: max(positive, +0)
        db = np.zeros(len(kb), T)
    else:
        da[~cancel] = np.where(da[~cancel] == 0, 3, da[~cancel])  # kept entries: a + 0 != 0 and a != 0
        db = -da[cancel] if name == "add" else da[cancel].copy()
    keys = _struct_check(Kn, D, name, T, ka, da, 1, kb, db, 1, what="pruned runs")
    assert len(keys) == int((~cancel).sum())


@gpu
@pytest.mark.parametrize("name,T", STRUCT_OPS, ids=[f"{n}-{t.name}" for n, t in STRUCT_OPS])
@pytest.mark.parametrize("R", [2, 3, 7, 64, 1000, 65537])
def test_merge_virtual_trailing_broadcast(name, T, R):
    Kn, D = _kn()
    rng = np.random.default_rng(R)
    for both in (False, True):
        for top in (False, True):
            n = max(2, 200_000 // R)
            pa, Ra, kb, Rb = E.broadcast_streams(R, both, n, rng, top=top)
            da, db = _data(name, T, len(pa), rng), _data(name, T, len(kb), rng)
            _struct_check(Kn, D, name, T, pa, da, Ra, kb, db, Rb, what=f"both={both} top={top}")
            _struct_check(Kn, D, name, T, kb, db, Rb, pa, da, Ra, what=f"swapped, both={both} top={top}")


@gpu
@pytest.mark.parametrize("name,T", STRUCT_OPS, ids=[f"{n}-{t.name}" for n, t in STRUCT_OPS])
def test_merge_small_operands(name, T):
    Kn, D = _kn()
    rng = np.random.default_rng(2)
    e = np.zeros(0, np.int64)
    big = np.sort(rng.choice(4_000_000, size=1_000_000, replace=False)).astype(np.int64)
    cases = [(e, np.array([5, 9], np.int64)), (np.array([5, 9], np.int64), e), (np.array([4]), np.array([4])),
             (np.array([4]), np.array([3])), (np.array([4]), np.array([5])), (big[500_000:500_001], big),
             (big, big[-1:]), (np.array([big[0] - 1]), big), (np.array([big[-1] + 1]), big)]
    for ka, kb in cases:
        ka, kb = np.asarray(ka, np.int64), np.asarray(kb, np.int64)
        _struct_check(Kn, D, name, T, ka, _data(name, T, len(ka), rng), 1, kb, _data(name, T, len(kb), rng), 1,
                      7 if T.kind == "i" else 1.5, 0, what=f"{len(ka)} x {len(kb)}")
    assert Kn.ew_merge_fused(0, D.upload(e), D.upload(np.zeros(0, T)), 1, D.upload(e), D.upload(np.zeros(0, T)), 1,
                             T.type(0), T.type(0), T.type(0), T, (1,), want_coords=False)[1].shape[0] == 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU: dense gather
# ---------------------------------------------------------------------------------------------------------------------
def _dense_case(Kn, D, shape, dshape, keys, R, T, rng, swap):
    """ew_dense with `subtract` (order-sensitive, exact) against NumPy's unravel + broadcast lookup."""
    shape = tuple(int(s) for s in shape)
    sv = _data("subtract", T, len(keys), rng)
    dense = _data("subtract", T, int(np.prod(dshape)), rng).reshape(dshape)
    code = _tables()._BINARY[np.subtract]
    strides = _tables()._dense_strides_over(shape, tuple(dshape))
    ok, ov, of = Kn.ew_dense(code, bool(swap), D.upload(keys), D.upload(sv), R, D.upload(dense.reshape(-1)), shape,
                             strides, T.type(0), T)
    ok, ov = D.download(ok), D.download(ov)
    ek = E.expand(keys, R)
    assert np.array_equal(ok, ek)
    coords = np.unravel_index(ek, shape)
    off = len(shape) - len(dshape)
    idx = tuple(np.where(dshape[d] == 1, 0, coords[d + off]) for d in range(len(dshape)))
    dv = dense[idx] if len(dshape) else np.full(len(ek), dense.reshape(()), T)
    s_rep = np.repeat(sv, R)
    want = (dv - s_rep) if swap else (s_rep - dv)
    assert np.array_equal(E.bits(ov), E.bits(want)) or T.kind == "f" and np.array_equal(ov, want, equal_nan=True)


@gpu
@pytest.mark.parametrize("T", [np.dtype(np.int64), np.dtype(np.float32)], ids=lambda t: t.name)
@pytest.mark.parametrize("ndim", range(1, 17))
def test_dense_every_ndim(T, ndim):
    Kn, D = _kn()
    rng = np.random.default_rng(ndim)
    ext = [3, 5, 2, 7, 1, 6, 3, 2, 5, 1, 3, 2, 1, 3, 2, 1]
    shape = tuple(ext[(i + ndim) % len(ext)] for i in range(ndim))
    while np.prod(shape) > 2_000_000:
        shape = tuple(max(1, s - 1) for s in shape)
    total = int(np.prod(shape))
    for trial in range(4):
        # dense operand: leading axes absent, extent 1 (zero stride) on a random subset of the rest
        lead = int(rng.integers(0, ndim))
        dshape = tuple(1 if rng.random() < 0.4 else s for s in shape[lead:])
        R = shape[-1] if trial % 2 else 1
        keys = np.sort(rng.choice(total // R, size=min(total // R, 5000), replace=False)).astype(np.int64)
        _dense_case(Kn, D, shape, dshape, keys, R, T, rng, swap=trial >= 2)


@gpu
@pytest.mark.parametrize("R", [1, 7])
def test_dense_keys_near_2_to_62(R):
    """A huge broadcast shape against a tiny dense operand: keys above 2^61, so every divmod of the index walk is a
    64-bit FastDiv by a non-power-of-two extent."""
    Kn, D = _kn()
    rng = np.random.default_rng(R)
    shape = (3, 1048573, 5, 1048583, 6, 6007, 7)
    total = 1
    for s in shape:
        total *= s
    assert 2 ** 61 < total < 2 ** 62
    dshape = (3, 1, 5, 1, 6, 1, 7)
    n = 3000
    hi = total // R
    keys = np.unique(np.concatenate([rng.integers(0, hi, size=n, dtype=np.int64),
                                     np.arange(hi - 50, hi, dtype=np.int64), np.arange(50, dtype=np.int64)]))
    assert keys.max() * R > 2 ** 61
    for swap in (0, 1):
        _dense_case(Kn, D, shape, dshape, keys, R, np.dtype(np.int64), rng, swap)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: broadcast expansion
# ---------------------------------------------------------------------------------------------------------------------
EXPAND_CASES = [
    ("leading", (4, 3, 5), (3, 5)),
    ("middle", (6, 4, 7), (6, 1, 7)),
    ("trailing", (5, 7, 3), (5, 1, 1)),
    ("mixed", (3, 2, 5, 1, 4, 3), (2, 1, 1, 4, 1)),
    ("all", (3, 4), (1, 1)),
]


@gpu
@pytest.mark.parametrize("idx", [np.int32, np.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("case", EXPAND_CASES, ids=[c[0] for c in EXPAND_CASES])
def test_expand(case, idx):
    import torch

    Kn, D = _kn()
    _, shape, xshape = case
    rng = np.random.default_rng(len(shape))
    nd, off = len(shape), len(shape) - len(xshape)
    total = int(np.prod(xshape))
    lin = np.sort(rng.choice(total, size=max(1, total * 2 // 3), replace=False))
    xc = np.stack(np.unravel_index(lin, xshape)) if len(xshape) else np.zeros((0, len(lin)), np.int64)
    n = len(lin)
    # a coordinate array whose row stride (n + 13) is not nnz
    wide = np.full((len(xshape), n + 13), -99, dtype=idx)
    wide[:, :n] = xc
    coords = D.upload(wide)[:, :n]
    assert coords.stride(0) == n + 13 and coords.stride(1) == 1
    bcast = [shape[d] > 1 and (d < off or xshape[d - off] != shape[d]) for d in range(nd)]
    src_row = [(d - off if (d >= off and not bcast[d]) else -1) for d in range(nd)]
    is_b = [1 if (bcast[d] or src_row[d] < 0) else 0 for d in range(nd)]
    keys, src = Kn.ew_expand(coords, shape, is_b, src_row)
    keys, src = D.download(keys), D.download(src)
    # NumPy's enumeration: entry e, then the broadcast axes' coordinates in C order
    baxes = [d for d in range(nd) if is_b[d]]
    bc = np.stack(np.unravel_index(np.arange(int(np.prod([shape[d] for d in baxes]))),
                                   tuple(shape[d] for d in baxes))) if baxes else np.zeros((0, 1), np.int64)
    R = bc.shape[1]
    full = np.zeros((nd, n * R), np.int64)
    for d in range(nd):
        if is_b[d]:
            full[d] = np.tile(bc[baxes.index(d)], n)
        else:
            full[d] = np.repeat(xc[src_row[d]], R)
    assert torch.is_tensor(coords)
    assert np.array_equal(src, np.repeat(np.arange(n), R))
    assert np.array_equal(keys, np.ravel_multi_index(tuple(full), shape))


# ---------------------------------------------------------------------------------------------------------------------
# end to end through the public API (mock kernels on a CPU box, CUDA kernels on an H100)
# ---------------------------------------------------------------------------------------------------------------------
def _int_coo(sp, T, rng, lo=-9, hi=10, edges=True):
    """A (40, 30) integer COO, half its positions zero; with `edges`, row 0 starts with 1, -1, MIN, MAX, 2."""
    d = rng.integers(lo, hi, size=(40, 30)).astype(T)
    d[rng.random(d.shape) < 0.5] = 0
    if edges:
        d[0, :5] = np.array([1, -1, np.iinfo(T).min, np.iinfo(T).max, 2], T)
    return d, sp.COO.from_numpy(d)


def _check_api(res, want, what):
    """Values and dtype equal NumPy's on the dense array; exactly the positions whose bits differ from the fill value
    are stored.  A dense result (func(fill, ndarray) not constant) is compared as it is."""
    assert res.dtype == want.dtype, f"{what}: dtype {res.dtype} != {want.dtype}"
    if isinstance(res, np.ndarray):
        assert np.array_equal(E.bits(res), E.bits(want)), f"{what}: values"
        return
    dense = res.todense()
    assert np.array_equal(E.bits(dense), E.bits(want)), f"{what}: values"
    fill = np.array([res.fill_value], dtype=res.dtype)
    stored = np.zeros(want.shape, bool)
    stored[tuple(np.asarray(res.coords))] = True
    differ = E.bits(want) != E.bits(fill)[0]
    assert (stored >= differ).all(), f"{what}: a value that differs from the fill value is not stored"
    assert not (E.bits(np.asarray(res.data)) == E.bits(fill)[0]).any(), f"{what}: a stored value equals the fill"


@pytest.mark.parametrize("T", E.INTS, ids=lambda t: t.name)
@pytest.mark.parametrize("name", ["floor", "ceil", "trunc", "reciprocal"])
def test_api_integer_unary(sp, name, T):  # noqa: F811
    d, x = _int_coo(sp, T, np.random.default_rng(1))
    f = getattr(np, name)
    with np.errstate(all="ignore"):
        want = f(d)
    _check_api(f(x), want, name)


@pytest.mark.parametrize("T", E.INTS, ids=lambda t: t.name)
def test_api_integer_power(sp, T):  # noqa: F811
    rng = np.random.default_rng(2)
    d, x = _int_coo(sp, T, rng)
    with np.errstate(all="ignore"):
        for k in (0, 1, 2, 3, 5, 31, 63, 64):
            _check_api(x ** k, d ** T.type(k), f"x ** {k}")
        dn, xn = _int_coo(sp, T, rng, lo=0, hi=70, edges=False)
        for k in (0, 1, -1, 2, 3, -3, 7):
            _check_api(k ** xn, T.type(k) ** dn, f"{k} ** x")
        e, y = _int_coo(sp, T, rng, lo=0, hi=9, edges=False)
        _check_api(x ** y, d ** e, "x ** y")
        _check_api(x ** e, d ** e, "x ** dense")


@pytest.mark.parametrize("T", E.INTS, ids=lambda t: t.name)
def test_api_integer_power_refuses_negative_exponents(sp, T):  # noqa: F811
    rng = np.random.default_rng(3)
    _, x = _int_coo(sp, T, rng)                          # stored entries include -1 and MIN
    dn, xn = _int_coo(sp, T, rng, lo=0, hi=5, edges=False)
    msg = "Integers to negative integer powers are not allowed"
    neg_fill = sp.COO.from_numpy(np.where(dn == 0, -2, dn).astype(T), fill_value=T.type(-2))
    dense_neg = dn.copy()
    dense_neg[3, 4] = -1
    calls = [("scalar", lambda: xn ** -1), ("stored entry", lambda: 2 ** x), ("sparse ** sparse", lambda: xn ** x),
             ("fill value", lambda: 2 ** neg_fill), ("dense operand", lambda: xn ** dense_neg),
             ("dense ** sparse", lambda: np.power(dn + 1, x))]
    for what, call in calls:
        with pytest.raises(ValueError, match=msg):
            call()
            pytest.fail(what)


@pytest.mark.parametrize("name", ["rad2deg", "deg2rad"])
def test_api_float32_degrees(sp, name):  # noqa: F811
    rng = np.random.default_rng(4)
    d = (rng.standard_normal((50, 40)) * 100).astype(np.float32)
    d[rng.random(d.shape) < 0.6] = 0
    x = sp.COO.from_numpy(d)
    _check_api(getattr(np, name)(x), getattr(np, name)(d), name)
