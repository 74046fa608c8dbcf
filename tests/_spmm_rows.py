"""Row streams with known per-panel run lengths for the CSR x dense kernels (tests/test_spmm_row_streams_gpu.py).

The tiled passes (spmm_panel.cu) split every row into P K-panels of `width = ceil(K / P)` columns (the panel of column
c is min(c // width, P - 1)) and walk each panel's run in chunks of L entries, one row after another per group of L
lanes.  `panel_rows` builds sorted CSR rows whose run in each panel has a chosen length, so that the chunk boundaries,
empty chunks and the rows-per-group walk are known exactly; `walk` replays that walk on the CPU."""
import numpy as np

BLOCK = 64  # rows per block of the block pattern


def panel_width(K, P):
    return max(1, -(-K // P))


def panel_of(cols, K, P):
    return np.minimum(np.asarray(cols, np.int64) // panel_width(K, P), P - 1)


def panel_ranges(K, P):
    """[lo, hi) columns of each panel (empty for the trailing panels when P does not fit K)."""
    w = panel_width(K, P)
    lo = np.minimum(np.arange(P, dtype=np.int64) * w, K)
    hi = np.minimum(lo + w, K)
    hi[-1] = K
    return lo, hi


def run_cycle(L):
    """Run lengths cycled through down the rows: 0, 1, L-1, L, L+1, 2L, 2L+1 and a long run, with a second 0 to make
    the period 9, which is coprime with the 32 / L groups of a warp (L in 4, 8, 16, 32)."""
    return np.array([0, 1, L - 1, L, 0, L + 1, 2 * L, 2 * L + 1, 5 * L + 3], np.int64)


def run_lengths(M, K, P, L):
    """(M, P) run lengths.  Row r takes cycle[(r + p) % 9] in panel p, except in its block b = r // 64:
    b % 8 == 3: the row is empty;  b % 8 == 5: empty in panel (b // 8) % P;
    b % 8 == 1: entries in the first panel only;  b % 8 == 6: entries in the last panel with columns only.
    Panels without columns (P > K) get 0."""
    cyc = run_cycle(L)
    r = np.arange(M, dtype=np.int64)[:, None]
    p = np.arange(P, dtype=np.int64)[None, :]
    R = cyc[(r + p) % len(cyc)]
    lo, hi = panel_ranges(K, P)
    has_cols = hi > lo
    last = int(np.flatnonzero(has_cols)[-1])
    b = r[:, 0] // BLOCK
    kind = b % 8
    R[kind == 3] = 0
    sel = np.flatnonzero(kind == 5)
    R[sel, (b[sel] // 8) % P] = 0
    R[np.ix_(kind == 1, np.arange(P) != 0)] = 0
    R[np.ix_(kind == 6, np.arange(P) != last)] = 0
    R[:, ~has_cols] = 0
    return R


def panel_rows(rng, M, K, P, L, dtype):
    """Sorted CSR (data, indices, indptr; int64 indices) with run lengths run_lengths(M, K, P, L).

    Within a run, columns are sorted random draws from the panel (repeats allowed).  Every third row pins its runs to
    the panel's first and last column, twice each when the run has 4 or more entries: columns p*width - 1, p*width
    and K - 1 all occur, and repeated columns sit on both sides of panel boundaries.  Every 7th value is -0.0."""
    R = run_lengths(M, K, P, L)
    lo, hi = panel_ranges(K, P)
    n = R.ravel()
    nnz = int(n.sum())
    run = np.repeat(np.arange(M * P, dtype=np.int64), n)  # (row, panel) id of every entry
    row, pan = run // P, run % P
    span = (hi - lo)[pan]
    cols = lo[pan] + np.minimum((rng.random(nnz) * span).astype(np.int64), span - 1)
    cols = np.sort(row * K + cols) - row * K  # rows are ascending; sort each row by column
    starts = np.zeros(M * P + 1, np.int64)
    np.cumsum(n, out=starts[1:])
    pos = np.arange(nnz, dtype=np.int64) - starts[run]
    pin = (row % 3 == 0)
    ln = n[run]
    first = pin & ((pos == 0) | ((pos == 1) & (ln >= 4)))
    lastp = pin & ((pos == ln - 1) | ((pos == ln - 2) & (ln >= 4)))
    cols[first] = lo[pan[first]]
    cols[lastp] = hi[pan[lastp]] - 1
    indptr = np.zeros(M + 1, np.int64)
    np.cumsum(R.sum(axis=1), out=indptr[1:])
    data = (rng.random(nnz) * 2 - 1).astype(dtype)
    data[::7] = -0.0
    return data, cols, indptr


def measured_runs(indices, indptr, K, P):
    """(M, P) run lengths recomputed from the CSR with the pre-pass's panel formula."""
    M = len(indptr) - 1
    row = np.repeat(np.arange(M, dtype=np.int64), np.diff(indptr))
    return np.bincount(row * P + panel_of(indices, K, P), minlength=M * P).reshape(M, P)


def pass_grid(M, L, sms, ctas_per_sm):
    """Row stride of a tiled pass: min(sms * ctas, ceil(M / (8 * 32 / L))) CTAs of 8 warps, 32 / L rows per warp."""
    rpw = 32 // L
    blocks = min(sms * ctas_per_sm, -(-M // (8 * rpw)))
    return blocks * 8 * rpw


def walk(runs, L, stride):
    """Replay one pass's walk: group g (rows g, g + stride, ...) takes one chunk per step, a row without entries
    being one empty chunk and a row of n entries ceil(n / L); groups g // (32 / L) share a warp, which stops once
    every one of its groups is past M.  Returns (fewest rows a group walks, warp steps whose chunks are all empty
    while some group is still below M, warps whose groups walk different numbers of chunks)."""
    M = len(runs)
    rpw = 32 // L
    S = -(-M // stride)
    pad = np.zeros(S * stride, np.int64)
    pad[:M] = runs
    n = pad.reshape(S, stride)  # n[k, g]: row g + k * stride
    valid = (np.arange(S * stride) < M).reshape(S, stride)
    chunks = np.where(valid, np.maximum(1, -(-n // L)), 0)
    start = np.cumsum(chunks, axis=0) - chunks
    total = chunks.sum(axis=0)
    T = int(total.max()) + 1
    empty = np.ones((stride, T), bool)  # past its rows a group walks empty rows
    active = np.arange(T)[None, :] < total[:, None]
    empty[active] = False
    k, g = np.nonzero(valid & (n == 0))
    empty[g, start[k, g]] = True
    w = stride // rpw
    skips = int((empty.reshape(w, rpw, T).all(axis=1) & active.reshape(w, rpw, T).any(axis=1)).sum())
    uneven = int((total.reshape(w, rpw).min(axis=1) != total.reshape(w, rpw).max(axis=1)).sum())
    return int(valid.sum(axis=0).min()), skips, uneven
