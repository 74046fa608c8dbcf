"""Value sets, references and comparison rules for the element-wise op table (K5, csrc/elemwise.cu), and key-stream
generators for its fused merge kernel.  CPU only: NumPy, no torch.

Ops are named by `__name__` of the functions in sparse_b200._elemwise._BINARY / _UNARY.  Every op is either EXACT
(correctly rounded or exact everywhere: compared bit for bit with NumPy in the compute dtype T) or TRANSCENDENTAL
(compared with a float64 reference for float32 inputs and a long double one for float64 inputs, within the ulp
budgets below).  Exceptions to bit equality, and why:
- a computed NaN is compared as a NaN only: the GPU's canonical NaN is not x86's (DESIGN.md section 4);
- ops that pass an operand through (PASS_THROUGH) keep its bits exactly, NaN payload included -- `where` relies on it.
  When both operands of maximum / minimum / fmax / fmin are NaN, the FIRST operand is returned (NumPy's rule);
- fmax / fmin of +0.0 and -0.0 are compared by value: NumPy's own answer depends on the array length there;
- integer edge results are pinned as literals (int_literals), not read from the NumPy that runs the test.
"""
import numpy as np

TILE = 1792      # positions per tile of the fused merge (EW_THREADS * EW_ITEMS)
ITEMS = 7        # positions per thread
LOOKBACK = 64    # predecessors the look-back reads per step

FLOATS = (np.dtype(np.float32), np.dtype(np.float64))
INTS = (np.dtype(np.int32), np.dtype(np.int64))
DTYPES = FLOATS + INTS

PREDICATES_BIN = {"greater", "greater_equal", "less", "less_equal", "equal", "not_equal", "logical_and",
                  "logical_or", "logical_xor"}
PREDICATES_UN = {"isnan", "isinf", "isfinite", "logical_not", "signbit"}
PASS_THROUGH = {"positive", "nan_replace", "_sel_x", "_sel_y", "_bitor_raw", "maximum", "minimum", "fmax", "fmin"}

# Maximum ulp error of the CUDA 12 math library on sm_90 ("CUDA C++ Programming Guide", appendix "Mathematical
# Functions", tables "Single-Precision Mathematical Standard Library Functions with Maximum ULP Error" and the
# double-precision one; full range, without -use_fast_math).  (float32, float64).  The guide states these maxima as the
# distance to the CORRECTLY ROUNDED result; measured at the unrounded reference, as here, that allows half an ulp more
# (ROUNDING_SLACK).  The H100 uses that half ulp: e.g. float64 log1p(-0.453207756284789) is 1.24 ulp from the exact
# value but 1 ulp from the rounded one, and expm1, log2, log10, tanh, cosh (float64) and expm1, cbrt (float32) show
# the same, between 1.0 and 1.24 ulp where the budget is 1.
ULP_BUDGET = {
    "exp": (2, 1), "expm1": (1, 1), "exp2": (2, 1), "log": (1, 1), "log1p": (1, 1), "log2": (1, 1),
    "log10": (2, 1), "sin": (2, 2), "cos": (2, 2), "tan": (4, 2), "sinh": (3, 2), "cosh": (2, 1), "tanh": (2, 1),
    "arcsin": (2, 2), "arctan": (2, 2), "arcsinh": (3, 3), "arctanh": (3, 2), "cbrt": (1, 1), "power": (4, 2),
}
ROUNDING_SLACK = 0.5
TRANSCENDENTAL = set(ULP_BUDGET)


def ubits(dt):
    return np.dtype(f"u{np.dtype(dt).itemsize}")


def bits(x):
    x = np.ascontiguousarray(x)
    return x.view(ubits(x.dtype))


def from_bits(b, dt):
    return np.array(b, dtype=ubits(dt)).view(np.dtype(dt))


def hp_dtype(T):
    """Reference precision for compute dtype T."""
    return np.dtype(np.float64) if np.dtype(T) == np.float32 else np.dtype(np.longdouble)


def is_transcendental(name, T):
    return name in TRANSCENDENTAL and np.dtype(T).kind == "f"


# ---------------------------------------------------------------------------------------------------------------------
# value sets
# ---------------------------------------------------------------------------------------------------------------------
def float_specials(T):
    T = np.dtype(T)
    fi = np.finfo(T)
    f32 = T == np.float32
    qnan = 0x7FC00000 if f32 else 0x7FF8000000000000
    nans = from_bits([qnan, qnan | 0x1234, qnan | (1 << (T.itemsize * 8 - 1))], T)
    one = T.type(1)
    vals = [0.0, -0.0, np.inf, -np.inf,
            fi.smallest_subnormal, -fi.smallest_subnormal,
            fi.smallest_normal - fi.smallest_subnormal, fi.smallest_normal, -fi.smallest_normal, fi.max, -fi.max,
            1.0, -1.0, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 3.0, -8.0, 1.0 / 3.0, 2.0, -2.0,
            2.0 ** 24 - 1, 2.0 ** 24 + 1, 2.0 ** 53 - 1, 2.0 ** 53 + 1,
            0.1, -0.1, 1e22, -1e22,
            np.nextafter(one, T.type(0)), np.nextafter(one, T.type(2)), 1.0 + 1e-3, 1.0 - 1e-3, -0.999,
            np.nextafter(-one, T.type(0)), 0.75, -0.75, 1e-5, 88.5, 710.0, -745.0]
    return np.concatenate([np.array(vals, dtype=np.float64).astype(T), nans])


def int_specials(T):
    T = np.dtype(T)
    ii = np.iinfo(T)
    nb = 8 * T.itemsize
    vals = [0, 1, -1, 2, -2, ii.min, ii.min + 1, ii.max, -1, nb - 1, nb, nb + 1, 64, 3, 7, -7]
    return np.array(sorted(set(vals)), dtype=T)


def specials(T):
    return float_specials(T) if np.dtype(T).kind == "f" else int_specials(T)


def random_values(T, n, rng):
    """n values: for floats a third raw bit patterns, a third log-uniform magnitudes in [2^-40, 2^40] and a third
    small half-integers; for integers a third over the whole range, a third in [-70, 70] (shift counts, small
    divisors) and a third in [-2^20, 2^20]."""
    T = np.dtype(T)
    k = n // 3
    if T.kind == "f":
        raw = rng.integers(0, np.iinfo(ubits(T)).max, size=k, dtype=ubits(T), endpoint=True).view(T)
        mag = np.exp2(rng.uniform(-40, 40, size=k)) * rng.choice([-1.0, 1.0], size=k)
        half = rng.integers(-40, 41, size=n - 2 * k) / 2.0
        return np.concatenate([raw, mag.astype(T), half.astype(T)])
    ii = np.iinfo(T)
    full = rng.integers(ii.min, ii.max, size=k, dtype=T, endpoint=True)
    small = rng.integers(-70, 71, size=k).astype(T)
    mid = rng.integers(-(1 << 20), (1 << 20) + 1, size=n - 2 * k).astype(T)
    return np.concatenate([full, small, mid])


def unary_set(T, rng, n=100_000):
    return np.concatenate([specials(T), random_values(T, n, rng)])


def pair_set(T, rng, n=100_000):
    """(a, b): the full cartesian product of the special set, then n random pairs."""
    s = specials(T)
    a = np.repeat(s, len(s))
    b = np.tile(s, len(s))
    return np.concatenate([a, random_values(T, n, rng)]), np.concatenate([b, random_values(T, n, rng)])


def nonneg_exponent(x):
    """Integer `power` refuses negative exponents: map them onto non-negative ones (~x), keeping 0, MAX and the shift
    edge counts."""
    return np.where(x < 0, ~x, x)


def fill_values(T):
    T = np.dtype(T)
    if T.kind == "f":
        return [T.type(v) for v in (0.0, 1.5, -0.0, np.nan, -3.0)]
    return [T.type(v) for v in (0, -1, 7, np.iinfo(T).min)]


def scalar_set(T):
    """The scalars the map kernel is run with, on each side."""
    T = np.dtype(T)
    if T.kind == "f":
        return [T.type(v) for v in (0.0, -0.0, 1.0, -1.5, 2.5, np.inf, np.nan, 0.1, 1e22)]
    nb = 8 * T.itemsize
    return [T.type(v) for v in (0, 1, -1, 3, nb - 1, nb, np.iinfo(T).min, np.iinfo(T).max)]


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------
def _where_nan_first(a, b, pick):
    """maximum / minimum: a NaN operand wins, the first one when both are NaN; a +-0 tie returns the SECOND operand
    (the kernel's rule, elemwise.cu, which NumPy's x86 loops follow)."""
    return np.where(np.isnan(a), a, np.where(np.isnan(b), b, np.where(pick(a, b), a, b)))


def _where_number_first(a, b, pick):
    """fmax / fmin: a NaN operand loses; both NaN returns the first."""
    return np.where(np.isnan(b), a, np.where(np.isnan(a), b, np.where(pick(a, b), a, b)))


def _bitor_raw(a, b):
    return (bits(a) | bits(b)).view(a.dtype)


def int_literals(name, a, b=None):
    """Integer edge results pinned as literals: x // 0 = 0, x % 0 = 0, MIN // -1 = MIN, MIN % -1 = 0, and
    reciprocal(x) = (T)(1.0 / x): 1 -> 1, -1 -> -1, 0 -> MIN (what x86-64 NumPy gives), 0 otherwise.
    Returns (mask of pinned positions, their values) or None."""
    T = a.dtype
    lo = np.iinfo(T).min
    if name == "floor_divide":
        m = (b == 0) | ((b == -1) & (a == lo))
        return m, np.where(b == 0, T.type(0), T.type(lo))
    if name == "remainder":
        m = (b == 0) | (b == -1)
        return m, np.zeros_like(a)
    if name == "reciprocal":
        return np.ones(len(a), bool), np.where(a == 1, T.type(1), np.where(a == -1, T.type(-1),
                                                                           np.where(a == 0, T.type(lo), T.type(0))))
    return None


def exact_reference(name, a, b=None):
    """NumPy's result of an exact op in its output dtype (the pinned rules above applied)."""
    T = a.dtype
    with np.errstate(all="ignore"):
        if name in ("maximum", "minimum", "fmax", "fmin") and T.kind == "f":
            pick = np.greater if name in ("maximum", "fmax") else np.less
            rule = _where_nan_first if name in ("maximum", "minimum") else _where_number_first
            return rule(a, b, pick).astype(T)
        if name == "nan_replace":
            return np.where(np.isnan(a), b, a)
        if name == "_sel_x":
            return np.where(a != 0, b, T.type(0))
        if name == "_sel_y":
            return np.where(a != 0, T.type(0), b)
        if name == "_bitor_raw":
            return _bitor_raw(a, b)
        if name == "power" and T.kind == "i":
            assert (b >= 0).all(), "integer power with a negative exponent"
        if T.kind == "i":
            pinned = int_literals(name, a, b)
            if pinned is not None:
                m, v = pinned
                safe_b = None if b is None else np.where(m, T.type(1), b)
                r = (getattr(np, name)(a, safe_b) if b is not None else np.zeros_like(a))
                return np.where(m, v, r)
        f = getattr(np, name)
        return f(a) if b is None else f(a, b)


def hp_reference(name, a, b=None):
    """Transcendental reference at higher precision (float64 for float32, long double for float64)."""
    H = hp_dtype(a.dtype)
    with np.errstate(all="ignore"):
        f = getattr(np, name)
        return f(a.astype(H)) if b is None else f(a.astype(H), b.astype(H))


def ulp_error(got, ref, T):
    """|got - ref| in ulps of T at the unrounded reference value `ref` (a finite high-precision array).  An infinite
    `got` counts as +-2^(emax+1), the first value past the largest finite one."""
    T = np.dtype(T)
    fi = np.finfo(T)
    H = ref.dtype
    g = got.astype(H)
    top = np.ldexp(H.type(1), fi.maxexp)
    g = np.where(np.isinf(g), np.copysign(top, g), g)
    _, e = np.frexp(np.abs(ref))            # |ref| = m * 2^e, m in [0.5, 1)
    e = np.where(ref == 0, fi.minexp, np.maximum(e.astype(np.int64) - 1, fi.minexp))
    ulp = np.ldexp(np.ones(len(ref), H), (e - fi.nmant).astype(np.int32))
    return np.abs(g - ref) / ulp


def special_input(*xs):
    m = np.zeros(len(xs[0]), bool)
    for x in xs:
        m |= np.isnan(x) | np.isinf(x) | (x == 0)
    return m


def mismatches(name, T, got, a, b=None):
    """Boolean mask: where `got` (the kernel's values for op `name` on operands a[, b] in T) breaks the contract."""
    T = np.dtype(T)
    got = np.asarray(got)
    if name in PREDICATES_BIN or name in PREDICATES_UN:
        with np.errstate(all="ignore"):
            want = getattr(np, name)(a) if b is None else getattr(np, name)(a, b)
        return got.astype(bool) != want
    if is_transcendental(name, T):
        ref = hp_reference(name, a, b)
        rT = ref.astype(T)
        # special inputs, and results that are NaN, infinite or zero: class, sign and value exactly
        exact = special_input(a, *(() if b is None else (b,))) | np.isnan(ref) | np.isinf(ref) | (ref == 0)
        bad = np.zeros(len(got), bool)
        nan_both = np.isnan(got) & np.isnan(rT)
        bad[exact] = ~(nan_both[exact] | (bits(got)[exact] == bits(rT)[exact]))
        close = ~exact
        budget = ULP_BUDGET[name][0 if T == np.float32 else 1] + ROUNDING_SLACK
        with np.errstate(all="ignore"):
            err = ulp_error(got[close], ref[close], T)
        overflow = np.isinf(got[close]) & (got[close] == rT[close])  # a finite reference that rounds to +-inf in T
        bad[close] = ~((err <= budget) | overflow)
        return bad
    want = exact_reference(name, a, b)
    if want.dtype != T:
        raise AssertionError(f"{name} on {T}: NumPy result dtype {want.dtype}")
    bad = bits(got) != bits(want)
    if T.kind == "f":
        if name not in PASS_THROUGH:
            bad &= ~(np.isnan(got) & np.isnan(want))
        if name in ("fmax", "fmin"):
            bad &= ~((got == 0) & (want == 0))
    return bad


def worst(name, T, got, a, b=None, k=5):
    """The first k offending inputs, for an assertion message."""
    bad = np.flatnonzero(mismatches(name, T, got, a, b))[:k]
    rows = []
    for i in bad:
        ins = f"a={a[i]!r} ({bits(a[i:i + 1])[0]:#x})" + ("" if b is None else f", b={b[i]!r} ({bits(b[i:i + 1])[0]:#x})")
        rows.append(f"{ins}: got {got[i]!r} ({bits(got[i:i + 1])[0]:#x})")
    return f"{name} on {np.dtype(T)}: {int(mismatches(name, T, got, a, b).sum())} bad; " + "; ".join(rows)


# ---------------------------------------------------------------------------------------------------------------------
# key streams for the fused merge
# ---------------------------------------------------------------------------------------------------------------------
def expand(keys, R):
    """Virtual trailing broadcast made explicit: key * R + r, r < R."""
    keys = np.asarray(keys, np.int64)
    return (keys[:, None] * np.int64(R) + np.arange(R, dtype=np.int64)[None, :]).reshape(-1)


def merged_sources(ka, kb):
    """NumPy replay of the merge path: for each merged position, True when it is taken from A (ties go to A)."""
    order = np.argsort(np.concatenate([ka, kb]), kind="stable")
    return order < len(ka), np.concatenate([ka, kb])[order]


def tiles_of(total):
    return -(-total // TILE)


def split_pair_streams(s, pairs):
    """A and B share `pairs` keys and A has s unmatched keys in front.  A's copy of shared key k sits at merged
    position s + 2k, B's copy at s + 2k + 1: for odd s every tile boundary (and for every s some 7-position thread
    boundary, at an offset that moves with s) falls between the two copies of one key."""
    ka = np.arange(s + pairs, dtype=np.int64) * 3
    kb = ka[s:].copy()
    return ka, kb


def tile_count_streams(tiles, rng):
    """A and B (about a third shared keys) whose merge has exactly `tiles` tiles."""
    total = (tiles - 1) * TILE + int(rng.integers(1, TILE + 1))
    keys = np.sort(rng.choice(4 * total, size=total, replace=False)).astype(np.int64)
    kind = rng.integers(0, 3, size=len(keys))            # 0: A only, 1: B only, 2: both
    # shared keys count twice: trim the key set until A + B is exactly `total`
    count = np.cumsum(np.where(kind == 2, 2, 1))
    n = int(np.searchsorted(count, total, side="right"))
    keys, kind = keys[:n], kind[:n]
    if count[n - 1] < total:                             # one short: one more A-only key past the last
        keys = np.append(keys, keys[-1] + 1)
        kind = np.append(kind, 0)
    ka, kb = keys[kind != 1], keys[kind != 0]
    assert len(ka) + len(kb) == total
    return ka, kb


def pruned_tile_streams(pattern, rng):
    """Streams laid out tile by tile from `pattern` ("P": every position of the tile is one copy of a shared key whose
    result is pruned; "K": A-only keys, kept).  Returns ka, kb and the mask of A entries that must cancel."""
    ka, kb, cancel = [], [], []
    k = 0
    for c in pattern:
        if c == "P":
            keys = np.arange(k, k + TILE // 2, dtype=np.int64)
            ka.append(keys)
            kb.append(keys)
            cancel.append(np.ones(len(keys), bool))
            k += TILE // 2
        else:
            keys = np.arange(k, k + TILE, dtype=np.int64)
            ka.append(keys)
            cancel.append(np.zeros(len(keys), bool))
            k += TILE
    return np.concatenate(ka), np.concatenate(kb) if kb else np.zeros(0, np.int64), np.concatenate(cancel)


def broadcast_streams(R, both, n, rng, top=False):
    """Prefix keys for a virtual trailing broadcast by R on A (and on B when `both`; otherwise B holds expanded keys
    directly).  With `top` the largest expanded key is 2^63 - 1 - small."""
    hi = (np.iinfo(np.int64).max // R) if top else max(4 * n, 16)
    lo = hi - 4 * n if top else 0
    pa = np.sort(rng.choice(np.arange(lo, hi, dtype=np.int64), size=n, replace=False))
    if both:  # B keeps every other prefix of A and adds its own
        pb = np.union1d(pa[::2], rng.choice(np.arange(lo, hi, dtype=np.int64), size=n // 2 + 1, replace=False))
        return pa, R, pb, R
    ea = expand(pa, R)
    pool = np.union1d(ea[:: 3], expand(np.arange(lo, hi, 7, dtype=np.int64)[:n], R)[:: 2])
    kb = np.sort(rng.choice(pool, size=min(len(pool), n * R), replace=False))
    return pa, R, kb, 1


def union_oracle(name, ka, da, Ra, kb, db, Rb, fill_a, fill_b, out_fill):
    """elemwise on key streams, restated: union of the (expanded) keys, f(a or fill_a, b or fill_b) with the exact
    reference, keep what differs from out_fill by bit pattern.  Returns keys, values, va, vb over the whole union."""
    ea, eb = expand(ka, Ra), expand(kb, Rb)
    xa, xb = np.repeat(da, Ra), np.repeat(db, Rb)
    keys = np.union1d(ea, eb)
    va = np.full(len(keys), fill_a, dtype=da.dtype)
    vb = np.full(len(keys), fill_b, dtype=db.dtype)
    va[np.searchsorted(keys, ea)] = xa
    vb[np.searchsorted(keys, eb)] = xb
    r = exact_reference(name, va, vb) if name not in PREDICATES_BIN else getattr(np, name)(va, vb)
    keep = bits(r) != bits(np.array([out_fill], dtype=r.dtype))[0]
    return keys[keep], r[keep], keys, va, vb
