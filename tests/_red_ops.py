"""Key streams, value sets and the restated reference for the grouped reduction (K7, csrc/reduce_fused.cu).  CPU only:
NumPy, no torch.

The reduction's contract, as the tests below check it:
- group id = key // ncols; a group's value is its stored values folded in stored order;
- the fill-value step of SparseArray.reduce (_sparse_array.py:405-422): add / multiply get fill * n_fill / fill ** n_fill
  computed in the type NumPy promotes T and int64 to (float64 for float32), the ufunc's identity where n_fill == 0, and
  one rounding to T at the end; every other op gets op(v, fill) where the group is incomplete;
- the result fill is super_ufunc(fill, ncols) with the fill in T and ncols a Python int, as the reference's n_cols is
  (so a float32 fill ** ncols stays in float32 arithmetic); results are pruned by bit pattern (`equivalent`).
Float add and multiply are compared bit for bit on exactly representable values (every association order then gives
the same bits) and within a rounding-error bound on random values.  maximum / minimum / fmax / fmin are compared bit for
bit with a LEFT fold that keeps the earlier operand: the first of equal values (+0.0 before -0.0 or the other way
round) and the first NaN (payload included); the fill value is the right operand.  NumPy's own reduceat does not pin
these bits: its SIMD loops return the later of two equal zeros, and which NaN depends on the length.
"""
import functools
import re

import numpy as np

TILE = 2048           # entries per tile (RD_TILE = RD_THREADS * RD_ITEMS)
ITEMS = 8             # consecutive entries per thread
THREADS = 256         # threads per tile
CARRY_WINDOW = 32     # predecessor tiles per step of the single-pass kernel's carry-in look-back
HEADS_WINDOW = 64     # predecessor tiles per step of its head-count look-back
TWO_PASS_MAX_NCOLS = 2048  # default form: count / scan / emit up to this group width, single pass above

NCOLS_TWO_PASS = (1, 2, 3, 7, 8, 2047, 2048)
NCOLS_SINGLE = (2049, 4096, 10**6 + 3, 2**33, 2**40 + 1)
NCOLS = NCOLS_TWO_PASS + NCOLS_SINGLE

OPS = {0: np.add, 1: np.multiply, 2: np.maximum, 3: np.minimum, 4: np.logical_and, 5: np.logical_or,
       6: np.bitwise_and, 7: np.bitwise_or, 8: np.bitwise_xor, 9: np.fmax, 10: np.fmin}
SUPER = {np.add: np.multiply, np.multiply: np.power}
EXTREMA = {np.maximum, np.minimum, np.fmax, np.fmin}


def parse_geometry(src):
    """The constants above as reduce_fused.cu states them."""
    threads = int(re.search(r"constexpr int RD_THREADS = (\d+);", src).group(1))
    items = int(re.search(r"constexpr int RD_ITEMS = (\d+);", src).group(1))
    assert re.search(r"constexpr int RD_TILE = RD_THREADS \* RD_ITEMS;", src)
    carry = [int(v) for v in re.findall(r"\bq -= (\d+);", src)]
    heads = [int(v) for v in re.findall(r"\bp -= (\d+);", src)]
    assert re.search(r"i1 = p - (\d+) - lane", src).group(1) == str(heads[0] // 2)
    form = re.search(r"g_reduce_form == 0 \? \(ncols <= (\w+)\)", src).group(1)
    return {"threads": threads, "items": items, "tile": threads * items, "carry": carry, "heads": heads,
            "form_max": threads * items if form == "RD_TILE" else int(form)}


# ---------------------------------------------------------------------------------------------------------------------
# key streams: a stream is a list of run lengths, laid out on the keys of a given ncols
# ---------------------------------------------------------------------------------------------------------------------
LENGTHS = (1, 7, 8, 9, 255, 256, 257, 2047, 2048, 2049)


def _random_runs(total, rng, long_every=40):
    """Run lengths summing to `total`: mostly 1..130, every `long_every`-th one 1000..5000."""
    out, s = [], 0
    while s < total:
        L = int(rng.integers(1000, 5001)) if len(out) % long_every == long_every - 1 else int(rng.integers(1, 131))
        L = min(L, total - s)
        out.append(L)
        s += L
    return out


@functools.lru_cache(maxsize=None)
def streams():
    """name -> run lengths.  Runs start and end at every offset relative to a thread's 8 entries, a warp's 256 and a
    tile's 2048; tiles exactly filled by one run and runs ending on a tile's last entry; runs spanning 31 .. 300 tiles
    (around both look-back windows); one run over everything; tile counts 1 .. ~5000; tiny n."""
    rng = np.random.default_rng(2048)
    out = {}
    runs = []
    for k in range(11):  # each cycle shifts the next cycle's start by 6887 = 7 mod 8, 231 mod 256, 743 mod 2048
        runs += list(np.roll(LENGTHS, k))
    out["lengths"] = [3] + runs
    out["tile_fill"] = [2048] * 3 + [1, 2047, 2047, 1, 5, 2043, 2048, 1000, 1048, 4096, 2048 * 3, 3, 2045, 2048]
    span = [5]
    for t in (31, 32, 33, 63, 64, 65, 300):
        span += [TILE * t + 17, 3]
    out["span"] = span
    out["whole"] = [TILE * 100 + 17]
    for tiles in (1, 2, 31, 32, 33, 64, 65, 5000):
        r = np.random.default_rng(tiles)
        out[f"tiles{tiles}"] = _random_runs((tiles - 1) * TILE + int(r.integers(1, TILE + 1)), r)
    for n in (1, 7, 8, 2047, 2048, 2049):
        out[f"n{n}"] = _random_runs(n, np.random.default_rng(n), long_every=3)
    return out


_STREAMS = {}


def stream_keys(name, ncols):
    """layout() of streams()[name], cached: every case runs the same keys."""
    if (name, ncols) not in _STREAMS:
        names = list(streams())
        _STREAMS[(name, ncols)] = layout(streams()[name], ncols, seed=names.index(name))
        _STREAMS[(name, ncols)].flags.writeable = False
    return _STREAMS[(name, ncols)]


def layout(runs, ncols, seed=0):
    """Sorted int64 keys for the run lengths on groups of width ncols.  A run longer than ncols becomes full groups
    (the rest in one more).  Group ids grow by 1 or 2; the columns of a run are spread over its group: a group of
    length L gets columns shift + i * (ncols // L), i < L, so full groups are complete and the others are not."""
    runs = np.asarray(runs, np.int64)
    full, rest = runs // ncols, runs % ncols
    lens = np.repeat(np.stack([np.full(len(runs), ncols), rest], 1).reshape(-1),
                     np.stack([full, (rest > 0).astype(np.int64)], 1).reshape(-1))
    rng = np.random.default_rng(seed + ncols % 1000003)
    gid = np.cumsum(rng.integers(1, 3, size=len(lens))) - 1
    assert gid[-1] < (2**63 - 1) // ncols, "keys would overflow int64"
    step = np.maximum(ncols // lens, 1)
    room = ncols - 1 - (lens - 1) * step
    shift = (rng.random(len(lens)) * (room + 1)).astype(np.int64)
    run_of = np.repeat(np.arange(len(lens)), lens)
    pos = np.arange(int(lens.sum())) - np.repeat(np.cumsum(lens) - lens, lens)
    keys = gid[run_of] * np.int64(ncols) + shift[run_of] + pos * step[run_of]
    return keys


def heads(keys, ncols):
    g = keys // ncols
    h = np.ones(len(g), bool)
    h[1:] = g[1:] != g[:-1]
    return g, np.flatnonzero(h)


# ---------------------------------------------------------------------------------------------------------------------
# values
# ---------------------------------------------------------------------------------------------------------------------
def qnans(T):
    """Three quiet NaNs with distinct payloads (one negative)."""
    T = np.dtype(T)
    q = 0x7FC00000 if T == np.float32 else 0x7FF8000000000000
    sign = 1 << (8 * T.itemsize - 1)
    return np.array([q | 1, q | 0x1234, q | sign | 7], dtype=f"u{T.itemsize}").view(T)


def bits(x):
    x = np.ascontiguousarray(x)
    return x.view(f"u{x.dtype.itemsize}")


def exact_sum_values(T, n, rng):
    """Quarters in [-1, 1]: every partial sum of a run of up to 2^21 entries is exact in float32."""
    return (rng.integers(-4, 5, size=n) / 4.0).astype(T)


def exact_prod_values(T, n, rng):
    """+-2^e with e = P_i - P_(i-1) for random P_i in [0, 3]: every contiguous product is +-2^k, |k| <= 3, so every
    association order gives the same bits."""
    P = rng.integers(0, 4, size=n + 1)
    return (np.ldexp(1.0, np.diff(P)) * rng.choice([-1.0, 1.0], size=n)).astype(T)


def random_floats(T, n, rng):
    """Normal values scaled by 2^U(-20, 20): cancellation and mixed magnitudes, no overflow."""
    return (rng.standard_normal(n) * np.exp2(rng.uniform(-20, 20, size=n))).astype(T)


def random_factors(T, n, rng):
    """+-2^U(-1/16, 1/16) with random mantissas: products of a few hundred thousand stay far from overflow and from
    the subnormals (the exponent is a random walk with steps below 1/16)."""
    return (np.exp2(rng.uniform(-1 / 16, 1 / 16, size=n)) * rng.choice([-1.0, 1.0], size=n)).astype(T)


def extrema_values(T, keys, ncols, rng):
    """+0.0 / -0.0 ties, +-inf, +-1, 2 and NaNs with distinct payloads; NaNs only in every other group, so that half
    the groups are decided by the tie rule."""
    n = len(keys)
    pool = np.array([0.0, -0.0, 0.0, -0.0, 1.0, -1.0, 2.0, np.inf, -np.inf], T)
    v = pool[rng.integers(0, len(pool), size=n)]
    nan_ok = ((keys // ncols) % 2) == 0
    m = nan_ok & (rng.random(n) < 0.1)
    v[m] = qnans(T)[rng.integers(0, 3, size=int(m.sum()))]
    return v


def int_values(T, n, rng):
    """The whole range of T, its minimum and maximum, and small values."""
    T = np.dtype(T)
    ii = np.iinfo(T)
    v = rng.integers(ii.min, ii.max, size=n, dtype=T, endpoint=True)
    m = rng.random(n)
    v[m < 0.05] = ii.min
    v[(m >= 0.05) & (m < 0.1)] = ii.max
    small = (m >= 0.1) & (m < 0.3)
    v[small] = rng.integers(-3, 4, size=int(small.sum())).astype(T)
    return v


def bool_values(keys, ncols, rng):
    """Mostly True in every other group (all / logical_and see whole-True groups), half and half elsewhere."""
    p = np.where((keys // ncols) % 2 == 0, 0.002, 0.5)
    return rng.random(len(keys)) >= p


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
def first_wins(method, a, b):
    """The two-operand rule of the ordered fold (a is the earlier operand): maximum / minimum keep a NaN, the first
    one of two; fmax / fmin keep the number, the first NaN of two; ties keep a."""
    with np.errstate(invalid="ignore"):
        if method in (np.maximum, np.fmax):
            pick = a >= b
        else:
            pick = a <= b
        if method in (np.maximum, np.minimum):
            return np.where(np.isnan(a) | (~np.isnan(b) & pick), a, b)
        return np.where(pick | np.isnan(b), a, b)


def ordered_reduceat(method, v, starts):
    """Left fold of every group in stored order with first_wins: for maximum / minimum the first NaN if there is one,
    for fmax / fmin the first NaN if there is nothing else; otherwise the first entry equal (by value) to the extreme."""
    n = len(v)
    idx = np.arange(n, dtype=np.int64)
    big = np.int64(n)
    nan = np.isnan(v)
    first_nan = np.minimum.reduceat(np.where(nan, idx, big), starts)
    num = np.where(nan, -np.inf if method in (np.maximum, np.fmax) else np.inf, v)
    ext = (np.fmax if method in (np.maximum, np.fmax) else np.fmin).reduceat(num, starts)
    ends = np.r_[starts[1:], n]
    grp = np.repeat(np.arange(len(starts)), ends - starts)
    first_ext = np.minimum.reduceat(np.where(~nan & (v == ext[grp]), idx, big), starts)
    if method in (np.maximum, np.minimum):
        pick = np.where(first_nan < big, first_nan, first_ext)
    else:
        pick = np.where(first_ext < big, first_ext, first_nan)
    return v[pick]


def result_fill(method, fill, ncols, T):
    """super_ufunc(fill, ncols) with the fill in T and ncols a Python int, as the reference's n_cols (its shapes are
    Python ints): a float32 fill stays in float32 arithmetic.  The fill itself for the other ops."""
    sup = SUPER.get(method)
    if sup is None:
        return np.asarray(fill).astype(T)[()]
    with np.errstate(all="ignore"):
        return np.asarray(sup(np.asarray(fill).astype(T)[()], int(ncols))).astype(T)[()]


def apply_fill(method, data, counts, ncols, fill, ordered):
    """_sparse_array.py:405-422 on grouped results `data` (in T) of `counts` entries each."""
    T = data.dtype
    n_fill = np.int64(ncols) - counts.astype(np.int64)
    with np.errstate(all="ignore"):
        sup = SUPER.get(method)
        if sup is None:
            data = data.copy()
            m = n_fill != 0
            if ordered and method in EXTREMA:
                data[m] = first_wins(method, data[m], T.type(fill))
            else:
                data[m] = method(data[m], fill).astype(T)
            return data
        contribution = sup(fill, n_fill)
        contribution = np.where(n_fill == 0, method.identity, contribution)
        return method(data, contribution).astype(T)


def restate(method, keys, vals, ncols, fill, ordered=True):
    """The grouped reduction of sorted `keys` / `vals` (already in the work dtype T), fill step applied:
    (group ids, values in T, counts, result fill).  `ordered` pins extrema to the ordered fold; otherwise reduceat."""
    g, starts = heads(keys, ncols)
    T = vals.dtype
    with np.errstate(all="ignore"):
        if ordered and method in EXTREMA and T.kind == "f":
            data = ordered_reduceat(method, vals, starts)
        else:
            data = method.reduceat(vals, starts).astype(T)
    counts = np.diff(np.r_[starts, len(keys)])
    data = apply_fill(method, data, counts, ncols, fill, ordered)
    return g[starts], data, counts, result_fill(method, fill, ncols, T)


def n_equal(vals, rfill):
    return int((bits(vals) == bits(np.array([rfill], vals.dtype))[0]).sum())


def gamma(T, counts):
    """gamma_{n+1} = k u / (1 - k u), k = n + 1, for the n = count + 1 roundings of a group and its fill step."""
    u = float(np.finfo(T).eps) / 2
    k = counts.astype(np.float64) + 2
    return k * u / (1 - k * u)


FRACTION_MAX = 64  # longest group the exact rational fallback checks ...
FRACTION_GROUPS = 4000  # ... and how many of them (the first ones)


def long_double_ok():
    return np.finfo(np.longdouble).nmant >= 63


def group_errors(method, got, vals, starts, ncols, fill, T, fraction=None):
    """For float add / multiply: (checked groups, |got - exact|, bound).  The bound is
    gamma_{n+1} (sum |x_i| + |fill| n_fill) + (n + 2) smallest subnormal for a sum and gamma_{n+1} |exact| + the same
    subnormal slack for a product (the fill of a product must be +-1 here).  The exact value is taken in float64 for
    float32 data and in long double (at least 63 mantissa bits) for float64 data; without such a long double, or with
    `fraction`, it is a `fractions.Fraction` sum / product over the first FRACTION_GROUPS groups of at most FRACTION_MAX
    entries only."""
    import fractions

    T = np.dtype(T)
    fi = np.finfo(T)
    counts = np.diff(np.r_[starts, len(vals)])
    n_fill = np.int64(ncols) - counts
    slack = (counts.astype(np.float64) + 2) * float(fi.smallest_subnormal)
    g = gamma(T, counts)
    if method is np.multiply:
        assert abs(float(fill)) == 1.0, "random products take a fill of +-1"
    if fraction is None:
        fraction = T == np.float64 and not long_double_ok()
    if not fraction:
        H = np.float64 if T == np.float32 else np.longdouble
        x = vals.astype(H)
        with np.errstate(all="ignore"):
            if method is np.add:
                exact = np.add.reduceat(x, starts) + H(fill) * n_fill.astype(H)
                scale = np.add.reduceat(np.abs(x), starts).astype(np.float64) + abs(float(fill)) * n_fill
            else:
                exact = np.multiply.reduceat(x, starts) * np.where((n_fill % 2 == 1) & (float(fill) < 0), -1, 1)
                scale = np.abs(exact).astype(np.float64)
            err = np.abs(got.astype(H) - exact).astype(np.float64)
        return np.ones(len(starts), bool), err, g * scale + slack
    checked = (counts <= FRACTION_MAX) & (np.cumsum(counts <= FRACTION_MAX) <= FRACTION_GROUPS)
    err = np.full(len(starts), np.inf)
    scale = np.zeros(len(starts))
    F = fractions.Fraction
    for i in np.flatnonzero(checked):
        xs = [F(float(v)) for v in vals[starts[i]:starts[i] + counts[i]]]
        if method is np.add:
            exact = sum(xs, F(0)) + F(float(fill)) * int(n_fill[i])
            scale[i] = float(sum((abs(v) for v in xs), F(0)) + abs(F(float(fill))) * int(n_fill[i]))
        else:
            exact = F(1)
            for v in xs:
                exact *= v
            exact *= F(float(fill)) ** (int(n_fill[i]) % 2)
            scale[i] = float(abs(exact))
        if np.isfinite(got[i]):
            err[i] = float(abs(F(float(got[i])) - exact))
    return checked, err, g * scale + slack


# ---------------------------------------------------------------------------------------------------------------------
# the public API restated
# ---------------------------------------------------------------------------------------------------------------------
def restate_api(coords, data, shape, fill, method, axis, ordered=False):
    """SparseArray.reduce on a COO given by (coords, data, shape, fill): transpose the reduced axes last, group by the
    kept-axes key, reduce in key order, apply the fill step, prune by bit pattern (integers by value).  Returns (result
    coordinates, values, result fill, result shape)."""
    ndim = len(shape)
    axis = tuple(range(ndim)) if axis is None else tuple(a % ndim for a in (axis if isinstance(axis, tuple) else (axis,)))
    kept = tuple(d for d in range(ndim) if d not in axis)
    kshape = tuple(shape[d] for d in kept)
    ncols = int(np.prod([shape[d] for d in axis], dtype=np.int64))
    perm_shape = kshape + tuple(shape[d] for d in axis)
    coords = np.asarray(coords, np.int64).reshape(ndim, -1)
    keys = np.ravel_multi_index(tuple(coords[d] for d in kept + axis), perm_shape) if len(data) else np.zeros(0, np.int64)
    order = np.argsort(keys, kind="stable")
    keys, data = keys[order], np.asarray(data)[order]
    with np.errstate(all="ignore"):
        T = method.reduce(np.zeros(1, data.dtype)).dtype
    fill = np.asarray(fill)[()]
    rf = result_fill(method, fill, ncols, T)
    if len(data) == 0:
        return np.zeros((len(kept), 0), np.int64), np.zeros(0, T), rf, kshape
    g, starts = heads(keys, ncols)
    with np.errstate(all="ignore"):
        if ordered and method in EXTREMA and data.dtype.kind == "f":
            red = ordered_reduceat(method, data, starts)
        else:
            red = method.reduceat(data, starts)
    counts = np.diff(np.r_[starts, len(keys)])
    out = apply_fill(method, red.astype(T), counts, ncols, fill, ordered)
    if T.kind in "fc":
        keep = bits(out) != bits(np.array([rf], T))[0]
    else:
        keep = out != rf
    gids = g[starts][keep]
    rc = np.stack(np.unravel_index(gids, kshape)) if kshape else np.zeros((0, len(gids)), np.int64)
    return rc.astype(np.int64), out[keep], rf, kshape
