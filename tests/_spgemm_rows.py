"""Seeded CSR pairs (A, B) whose rows reach every path of the CSR x CSR kernels (spgemm.cu), for
tests/test_spgemm_rows_gpu.py.

The kernels pick their path per A row from two numbers: the entry count n of the row and its product count P (the sum
of the lengths of the B rows it references).  Rows with P <= 256 go to the warp-per-row kernel, which takes the row in
one piece when n <= 32 and in chunks of 32 entries otherwise, and sizes its shared-memory table H from P (64 slots up to
P = 16, then 128, 256, 512 at P = 17, 33, 65).  Rows with P > 256 go to the CTA-per-row kernel, which stages 256 A
entries at a time and their products in tiles of 2,048.  A row is described here by the list of B-row lengths its
entries reference, in order, so n and P are exact; B holds a pool of rows of every length a kind needs and is shuffled.

`make_pair` deals the kinds out down the rows in a period coprime with 4 (the warp kernel deals rows 4 to a ticket), so
that every kind meets every position of a ticket and every neighbour in the warp's row pipeline.  Besides the plain
kinds it places special B rows: columns that all land in one bucket of the warp table (hash_small) or of the CTA table
(hash_col), some buckets close to H - 1 so that probes wrap; columns all owned by one warp of the CTA kernel; pairs of
B rows with negated values, referenced with equal A values, whose products cancel to +0; and rows whose sums cancel in
float32 / lose bits in float64 (the `wide` accumulator's cases)."""
import numpy as np

WARP_PMAX = 256         # a row with more products goes to the CTA-per-row kernel
WARP_HMAX = 512         # the warp kernel's largest table
CTA_WARPS = 8           # warps of the CTA-per-row kernel; column k belongs to warp (hash_col(k) >> 20) % 8
CTA_THREADS = 256       # A entries the CTA kernel stages at a time
CTA_TILE = 2048         # products per staged tile

POOL = 24               # B rows of each length the kinds use
WIDE_SPAN = 5003        # columns of the ordinary B rows: half of them in [0, 5003), half in [0, 61) (both prime)
NARROW_SPAN = 61


# ---------------------------------------------------------------------------------------------------------------------
# the kernels' hashes and table sizes, restated
# ---------------------------------------------------------------------------------------------------------------------
def hash_small(k):
    """hash_small<I> of the warp kernel (the high-word fold is a no-op below 2^32, so this serves I = int32 too)."""
    k = np.asarray(k, np.int64).astype(np.uint64)
    x = (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    x ^= (k >> np.uint64(32)).astype(np.uint32) * np.uint32(0x85EBCA6B)
    return (x * np.uint32(0x9E3779B1)) >> np.uint32(20)


def hash_col(k):
    """hash_col<I> of the CTA kernel: the high word of k * 0x9E3779B97F4A7C15 (mod 2^64)."""
    k = np.asarray(k, np.int64).astype(np.uint64)
    return ((k * np.uint64(0x9E3779B97F4A7C15)) >> np.uint64(32)).astype(np.uint32)


def cta_owner(k):
    return (hash_col(k) >> np.uint32(20)) % np.uint32(CTA_WARPS)


def warp_table(P):
    """Slots of the warp kernel's table for a row of P products: load <= 1/4 while it fits, <= 1/2 always."""
    H = 64
    while H < 4 * P and H < WARP_HMAX:
        H *= 2
    return H


def cta_table(P, n_col):
    """Slots of the CTA kernel's global table for a row of P products."""
    cap = min(P, n_col)
    H = 64
    while H < 2 * cap:
        H *= 2
    return H


def pick_columns(pred, n, start=0, block=1 << 20):
    """The first n integers >= start for which pred(array) holds."""
    out = []
    got = 0
    while got < n:
        k = np.arange(start, start + block, dtype=np.int64)
        hit = k[pred(k)]
        out.append(hit[:n - got])
        got += len(out[-1])
        start += block
    return np.concatenate(out)


# ---------------------------------------------------------------------------------------------------------------------
# row kinds
# ---------------------------------------------------------------------------------------------------------------------
def holes(n):
    """Positions of an A row that reference empty B rows: lane 0, lane 31 and the last entry of every 32-entry chunk,
    a run of 8 entries, and the row's last entry."""
    if n < 3:
        return []
    h = {0, n - 1} | set(range(31, n, 32))
    if n > 16:
        h |= set(range(8, 16))
    return sorted(h)


def row_lengths(n, P, with_holes=True):
    """B-row lengths of an A row of n entries and P products: P is spread as evenly as possible over the entries
    outside `holes(n)` (the first P of them get 1 when P is smaller than their count)."""
    lens = np.zeros(n, np.int64)
    if n == 0:
        return lens
    live = np.setdiff1d(np.arange(n), holes(n) if with_holes and P > 0 else [])
    base, rem = divmod(P, len(live))
    lens[live] = base
    lens[live[:rem]] += 1
    assert lens.sum() == P
    return lens


# (entries, products, holes).  Every table edge of the warp kernel (P = 16/17, 32/33, 64/65, 256), entries 0, 1, 31,
# 32, 33, 64, 65 and more than 256 on both sides of one_chunk, P = 0 rows with and without entries.
SHORT_KINDS = [
    (0, 0, False), (3, 0, True), (40, 0, True),
    (1, 1, False), (1, 16, False), (31, 17, True), (32, 32, False), (1, 33, False), (2, 64, False),
    (32, 65, True), (31, 255, True), (1, 256, False), (32, 256, True), (32, 16, True),
    (33, 16, True), (33, 33, True), (64, 17, True), (64, 64, True), (65, 65, True), (65, 255, True),
    (100, 256, True), (300, 256, True), (33, 32, False), (64, 1, True), (65, 128, False),
]
# P > 256: the CTA kernel.  P = 257 exactly; chunk_total (products of 256 staged A entries) of exactly one and two
# 2,048-product tiles; A rows of 257 .. 600 entries (two or three staged chunks).
LONG_KINDS = [
    (1, 257, False), (33, 257, True), (2, 600, False), (256, 2048, False), (512, 4096, False), (256, 4096, False),
    (300, 2400, False), (257, 257, False), (600, 1000, True), (9, 3000, False), (40, 300, True),
]
assert len(SHORT_KINDS) % 2 == 1 and len(LONG_KINDS) % 2 == 1


def special_rows():
    """name -> columns of the special B rows (the value of each entry is set by `special_values`)."""
    rows = {}
    # one bucket of the warp table, for each table size; buckets 60, 126, 250, 509 sit close to H - 1 so probes wrap
    for H, bucket, n in ((64, 60, 16), (128, 126, 32), (256, 250, 64), (512, 509, 128)):
        c = pick_columns(lambda k, H=H, b=bucket: (hash_small(k) & np.uint32(H - 1)) == b, n, start=WIDE_SPAN)
        rows[f"c{H}"] = c
        rows[f"c{H}r"] = c[::-1].copy()
    # one bucket of the CTA table (H = 1024 for P = 300) and one owning warp
    c = pick_columns(lambda k: ((hash_col(k) & np.uint32(1023)) == 1021) & (cta_owner(k) == 5), 150, start=WIDE_SPAN)
    rows["cc"], rows["ccr"] = c, c[::-1].copy()
    c = pick_columns(lambda k: cta_owner(k) == 2, 400, start=WIDE_SPAN)
    rows["co"], rows["cor"] = c, np.random.default_rng(3).permutation(c)
    # twins: the same columns, negated values
    for n in (5, 40):
        c = np.arange(n, dtype=np.int64) * 7 % WIDE_SPAN
        rows[f"t{n}"], rows[f"t{n}n"] = c, c.copy()
    # the accumulator rows: three B rows over the same four columns
    for w in ("w1", "w2", "w3"):
        rows[w] = np.array([11, 22, 33, 44], np.int64)
    return rows


# special kinds: the B rows referenced (names or lengths); `ties` = entry pairs with equal A values, `ones` = entries
# whose A value is 1
SPECIAL_KINDS = [
    dict(refs=["c64"]), dict(refs=["c128"]), dict(refs=["c256"]), dict(refs=["c512", "c512r"]),
    dict(refs=["c64", "c64r", 0, "c64"]),                               # P = 48: H = 256, chains over 16 slots
    dict(refs=[0] * 32 + ["c256", 0]),                                  # collisions in a row's second chunk
    dict(refs=["cc", "ccr"]), dict(refs=["co", "cor", "co"]),           # CTA kernel: one bucket / one owner warp
    dict(refs=["t5", "t5n"], ties=[(0, 1)]), dict(refs=["t40", 3, 0, "t40n"], ties=[(0, 3)]),
    dict(refs=["w1", "w2", "w3"], ones=[0, 1, 2]),
]
assert len(SPECIAL_KINDS) % 2 == 1


KINDS = SHORT_KINDS + LONG_KINDS + SPECIAL_KINDS


def kind_refs(kind):
    if isinstance(kind, dict):
        return kind["refs"]
    n, P, h = kind
    return [int(x) for x in row_lengths(n, P, h)]


def row_kinds(M, long_every, special_every=0):
    """Index into KINDS of every row: SHORT_KINDS cycled (odd period), every `long_every`-th row (from row 3) a long
    kind, every `special_every`-th row (from row 5) a special kind."""
    ns, nl = len(SHORT_KINDS), len(LONG_KINDS)
    kinds = np.arange(M, dtype=np.int64) % ns
    if long_every:
        r = np.arange(3, M, long_every)
        kinds[r] = ns + np.arange(len(r)) % nl
    if special_every:
        r = np.arange(5, M, special_every)
        kinds[r] = ns + nl + np.arange(len(r)) % len(SPECIAL_KINDS)
    return kinds


# ---------------------------------------------------------------------------------------------------------------------
# values
# ---------------------------------------------------------------------------------------------------------------------
_WIDE_VALUES = {  # rows w1, w2, w3 over columns 11, 22, 33, 44
    # float32: 1e8 + 1 - 1e8 is 0 in float32 and 1 in float64; likewise 3; the last column agrees
    "f": [[1e8, 1e8, 3.0, 0.5], [1.0, 3.0, 1e8, 0.25], [-1e8, -1e8, -1e8, 1e-9]],
    # int64: 2^60 + 1 - 2^60 is 0 in float64 and 1 in int64; 2^53 + 1 rounds in float64
    "i8": [[2**60, 2**53, 5, 7], [1, 1, 3, 2**62], [-2**60, 0, -5, -2**62]],
    # int32: 2^30 + 2^30 wraps in int32 and not in float64
    "i4": [[2**30, 2**30, 5, 7], [2**30, 1, 3, -7], [-5, -2**30, -5, 0]],
}


def values(rng, n, dtype, mode):
    """n random values.  mode 'plain': floats in [-1, 1) (every 11th -0.0), integers in [-5, 5] (zeros included);
    'special': floats as plain plus NaN, +Inf and -Inf sprinkled; 'wrap': integers over the whole range, so products
    and sums wrap."""
    dt = np.dtype(dtype)
    if dt.kind == "f":
        v = (rng.random(n) * 2 - 1).astype(dt)
        v[::11] = -0.0
        if mode == "special":
            v[5::997] = np.nan
            v[7::1009] = np.inf
            v[9::1013] = -np.inf
        return v
    if mode == "wrap":
        info = np.iinfo(dt)
        return rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
    return rng.integers(-5, 6, n).astype(dt)


def special_values(name, cols, dtype, rng, mode):
    dt = np.dtype(dtype)
    if name[0] == "w":
        key = "f" if dt.kind == "f" else ("i8" if dt.itemsize == 8 else "i4")
        return np.array(_WIDE_VALUES[key][int(name[1]) - 1], dt)
    return values(rng, len(cols), dt, mode)


# ---------------------------------------------------------------------------------------------------------------------
# the pair
# ---------------------------------------------------------------------------------------------------------------------
def make_pair(rng, kinds, dtype, mode="plain"):
    """(A, B, n_col) for rows of the given kinds (indices into KINDS); A = (data, indices, indptr), B likewise, int64
    indices.

    A row's entries reference B rows as its kind lists them: a length picks one of POOL B rows of that length (256 for
    lengths 0 and 1) at random, a name the special B row.  B's rows are shuffled.  n_col is one past the largest
    column."""
    special = special_rows()
    kref = [kind_refs(k) for k in KINDS]
    lens = sorted({r for rr in kref for r in rr if not isinstance(r, str)} | {0, 1})
    # B rows: the pools, then the special rows; then shuffled
    b_len, b_name = [], []
    for ln in lens:
        cnt = 256 if ln <= 1 else POOL
        b_len += [ln] * cnt
        b_name += [None] * cnt
    for name, cols in special.items():
        b_len.append(len(cols))
        b_name.append(name)
    nb = len(b_len)
    perm = rng.permutation(nb)  # B row perm[i] is the i-th row built above
    b_len = np.array(b_len, np.int64)
    lens_sorted = np.empty(nb, np.int64)
    lens_sorted[perm] = b_len
    bp = np.zeros(nb + 1, np.int64)
    np.cumsum(lens_sorted, out=bp[1:])
    bi = np.empty(bp[-1], np.int64)
    bd = np.empty(bp[-1], np.dtype(dtype))
    pools = {}
    for i, (ln, name) in enumerate(zip(b_len.tolist(), b_name)):
        r = perm[i]
        s, e = bp[r], bp[r + 1]
        if name is None:
            pools.setdefault(ln, []).append(r)
            span = NARROW_SPAN if (i % 2 and ln <= NARROW_SPAN) else WIDE_SPAN
            stride = int(rng.integers(1, span))
            bi[s:e] = (int(rng.integers(0, span)) + np.arange(ln, dtype=np.int64) * stride) % span
        else:
            pools[name] = r
            bi[s:e] = special[name]
    bd[:] = values(rng, len(bd), dtype, mode)
    for name, cols in special.items():
        r = pools[name]
        bd[bp[r]:bp[r + 1]] = special_values(name, cols, dtype, rng, mode)
        if name[0] == "t" and name.endswith("n"):
            tw = pools[name[:-1]]
            bd[bp[r]:bp[r + 1]] = -bd[bp[tw]:bp[tw + 1]]
    # A: every entry looks up its reference in the flattened kind table
    kinds = np.asarray(kinds, np.int64)
    M = len(kinds)
    klen = np.array([len(rr) for rr in kref], np.int64)
    kstart = np.cumsum(klen) - klen
    flat = [r for rr in kref for r in rr]
    want = np.array([-1 if isinstance(r, str) else r for r in flat], np.int64)   # a length, or -1 for a name
    named = np.array([pools[r] if isinstance(r, str) else -1 for r in flat], np.int64)
    a_len = klen[kinds]
    ap = np.zeros(M + 1, np.int64)
    np.cumsum(a_len, out=ap[1:])
    row = np.repeat(np.arange(M, dtype=np.int64), a_len)
    t = kstart[kinds[row]] + (np.arange(ap[-1], dtype=np.int64) - ap[row])
    ai = named[t]
    for ln in lens:
        sel = np.flatnonzero(want[t] == ln)
        pool_rows = np.array(pools[ln], np.int64)
        ai[sel] = pool_rows[rng.integers(0, len(pool_rows), len(sel))]
    ad = values(rng, len(ai), dtype, mode)
    for kk, k in enumerate(KINDS):
        if isinstance(k, dict):
            s = ap[:-1][kinds == kk]
            for i, j in k.get("ties", []):
                ad[s + j] = ad[s + i]
            for i in k.get("ones", []):
                ad[s + i] = 1
    return (ad, ai, ap), (bd, bi, bp), int(bi.max()) + 1


def products(a, b):
    """P of every A row."""
    _, ai, ap = a
    _, _, bp = b
    per = bp[ai + 1] - bp[ai]
    c = np.zeros(len(per) + 1, np.int64)
    np.cumsum(per, out=c[1:])
    return c[ap[1:]] - c[ap[:-1]]


def chunk_totals(a, b, row):
    """Products of each group of CTA_THREADS A entries of a row (the CTA kernel's chunk_total)."""
    _, ai, ap = a
    _, _, bp = b
    per = (bp[ai + 1] - bp[ai])[ap[row]:ap[row + 1]]
    return np.add.reduceat(per, np.arange(0, len(per), CTA_THREADS)) if len(per) else per


# ---------------------------------------------------------------------------------------------------------------------
# occupancy of the warp kernel (the persistent grid is SMs x CTAs per SM, 4 warps per CTA, 4 rows per ticket)
# ---------------------------------------------------------------------------------------------------------------------
ROWS_WARPS = 4
ROWS_PER_TICKET = 4


def rows_kernel_ctas_per_sm(value_bytes, index_bytes, wide, regs):
    """CTAs per SM of spgemm_rows_kernel: the shared-memory bound of OrderedSmem (227 KB per SM, 1 KB reserved per
    CTA), the register bound (64 K registers per SM, allocated per warp in units of 256) and 64 warps per SM."""
    a16 = lambda x: (x + 15) // 16 * 16
    H = WARP_HMAX
    per_warp = a16(H * index_bytes) + a16(H * (8 if wide else value_bytes)) + a16(H // 2 * 2)
    by_smem = (227 * 1024) // (per_warp * ROWS_WARPS + 1024)
    by_regs = 65536 // (ROWS_WARPS * ((regs * 32 + 255) // 256 * 256)) if regs else 64
    return min(by_smem, by_regs, 64 // ROWS_WARPS)


def tickets_per_warp(M, sms, ctas_per_sm):
    return (-(-M // ROWS_PER_TICKET)) / (sms * ctas_per_sm * ROWS_WARPS)
