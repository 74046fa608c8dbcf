// spmm_panel.cu -- K1p: CSR x dense in (column tile x K panel) passes that serve the B-row gathers from L2.
//
// Same contract as K1 (bit-identical to _dot_csr_ndarray, sparse/numba_backend/_common.py:720-755).  At C2 (B is
// 1e6 x 128 fp32 = 512 MB, L2 is 50 MB) the one-pass kernel gathers one 512-byte row of B per stored entry and almost
// every gather misses L2: ~50 GB of HBM traffic for ~1.8 GB of compulsory bytes.  Here B is cut both ways:
//   * a column tile of TB bytes (default 128 B = one cache line: 32 fp32 / 16 fp64 columns), and
//   * P panels of the K axis (rows of B), so that one panel x one tile of B (K/P x TB bytes) fits in L2.
// One launch per (tile, panel), tiles outer, panels inner.  Pass (t, p) computes, for every row of A, the stored entries
// whose column falls into panel p, for the columns of tile t.  Rows are sorted by column, so these form the run
// [off[p][row], off[p+1][row]) that a pre-pass computes once per call.  Partial sums are carried through C in T: a store
// followed by a load of the same float is exact, panels are visited in ascending column order, and each run is taken
// in stored order, so every out[i,j] is still ((+0 + a0*b0) + a1*b1) + ... with separate roundings, as in K1.
// DRAM traffic: B once, A once per tile, C (2P-1) x per tile (reads and writes of one tile's columns).
//
// Any row with a descending column pair sets a device flag in the pre-pass; the passes then return at entry and the
// one-pass kernel, launched behind them with the same flag as its guard, computes the whole product.  No host sync.
#include "common.cuh"

namespace b2s {

template <typename T, int VEC>
struct alignas(sizeof(T) * VEC) PPack {
    T v[VEC];
};

__device__ __forceinline__ uint4 ldg_cs_v4(const void *p) {
    uint4 r;
    asm volatile("ld.global.cs.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

__device__ __forceinline__ uint64_t policy_evict_normal() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
    return p;
}

// Pre-pass: one warp per row.  off is panel-major, (P+1) x M: off[p*M + row] = first position of the row whose column is
// in panel >= p (off[0] = indptr[row], off[P] = indptr[row+1]).  Each lane handles one position j and writes off[p] = j
// for the panels p in (panel(j-1), panel(j)]; the position j = end closes the row with panel P.  A sorted row therefore
// writes each of its P+1 offsets exactly once.  *unsorted |= 1 if a row has a descending neighbour pair.
template <typename I>
__global__ void __launch_bounds__(256)
panel_offsets_kernel(int64_t M, const I *__restrict__ indptr, const I *__restrict__ indices, int64_t width, int P,
                     I *__restrict__ off, int *__restrict__ unsorted) {
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    bool bad = false;
    for (int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < M; row += nwarps) {
        const int64_t s = (int64_t)ldg_stream(indptr + row), e = (int64_t)ldg_stream(indptr + row + 1);
        if (lane == 0) __stcs(off + row, (I)s);
        I carry_c = 0;
        int carry_q = 0;
        for (int64_t j0 = s; j0 <= e; j0 += 32) {
            const int64_t j = j0 + lane;
            const bool valid = j < e;
            I c = 0;
            int q = P;  // positions at or past the end close the row
            if (valid) {
                c = ldg_stream(indices + j);
                bad |= c < 0;
                int64_t qq;
                if constexpr (sizeof(I) == 4) qq = width > 0xffffffffll ? 0 : (int64_t)((uint32_t)c / (uint32_t)width);
                else qq = (int64_t)((uint64_t)c / (uint64_t)width);
                q = qq < P - 1 ? (int)qq : P - 1;
            }
            I cp = __shfl_up_sync(FULL, c, 1);
            int qp = __shfl_up_sync(FULL, q, 1);
            if (lane == 0) {
                cp = carry_c;
                qp = carry_q;
            }
            if (valid && j > s && c < cp) bad = true;
            if (j <= e)
                for (int p = qp + 1; p <= q; ++p) __stcs(off + (int64_t)p * M + row, (I)j);
            carry_c = __shfl_sync(FULL, c, 31);
            carry_q = __shfl_sync(FULL, q, 31);
        }
    }
    if (__any_sync(FULL, bad) && lane == 0) atomicOr(unsorted, 1);
}

// 16-byte B gather straight into r when pred is set; otherwise no request is issued and r keeps its value.  Writing
// the destination in the load itself (no copy behind it) lets L of these issue back to back into L distinct packs.
__device__ __forceinline__ void ldg_nc_v4_hint_if(uint4 &r, const void *p, bool pred, uint64_t pol) {
    asm volatile(
        "{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %5, 0;\n\t"
        "@q ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %6;\n\t}"
        : "+r"(r.x), "+r"(r.y), "+r"(r.z), "+r"(r.w)
        : "l"(p), "r"((int)pred), "l"(pol));
}

// One chunk of up to L stored entries of one row of a pass, as one lane of the row's group sees it.
template <typename T, typename I>
struct PassChunk {
    I col;     // column of entry base + sub (0 past the chunk's end)
    T val;
    int step;  // the row is row0 + step * stride
    int info;  // entries in the chunk (0..L) | kHead | kTail | kTouched
};

// CTAs of 256 threads per SM the register budget is sized for: two (<= 128 registers) while the ring (2L packs of 4
// registers) leaves room, one for L = 16.  Either way 1024 (L <= 8) or 512 (L = 16) gathers can be in flight per SM.
constexpr int tile_pass_min_blocks(int L) { return L <= 8 ? 2 : 1; }

// One pass (column tile at col_base, K panel [off_lo, off_hi)).  A group of L lanes owns one row and one tile of L x 16
// bytes; lane `sub` holds columns col_base + sub*VEC .. +VEC.  Persistent warps walk rows with a static stride; each
// group walks its own stream of chunks (L stored entries of one row; a row without entries in this panel is one empty
// chunk, so pass 0 still writes its +0) independently of the other groups of its warp, with no barrier between rows.
// Software pipeline, one chunk per step, per lane:
//   * the L gathers of chunk k+1 issue into one half of a two-chunk register ring (2L packs of 16 bytes) before the
//     FMAs of chunk k consume the other half, so up to 2L gathers are in flight per lane across row boundaries;
//   * A entries are loaded two chunks ahead of their gathers, the offsets of a row two rows ahead of its A;
//   * the C partial of a row is loaded right after the previous chunk's FMAs (and its row's store), one step ahead.
template <typename T, typename I, int L>
__global__ void __launch_bounds__(256, tile_pass_min_blocks(L))
spmm_tile_pass_kernel(int64_t M, int64_t N, const T *__restrict__ a_data, const I *__restrict__ a_indices,
                      const I *__restrict__ off_lo, const I *__restrict__ off_hi, const T *__restrict__ B, int64_t ldb,
                      T *__restrict__ C, int64_t ldc, int64_t col_base, int first, int hint,
                      const int *__restrict__ unsorted) {
    if (*unsorted) return;  // the one-pass kernel behind the passes computes this call
    constexpr int VEC = 16 / sizeof(T);
    constexpr int RPW = 32 / L;  // rows per warp
    constexpr unsigned FULL = 0xffffffffu;
    // chunk info: first / last chunk of its row; the row has entries in this panel
    constexpr int kHead = 1 << 8, kTail = 2 << 8, kTouched = 4 << 8, kCnt = 0xff;
    const int lane = threadIdx.x & 31;
    const int sub = lane & (L - 1);
    const int grp = lane / L;
    const int64_t col0 = col_base + (int64_t)sub * VEC;
    const bool col_ok = col0 < N;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t stride = nwarps * RPW;
    const int64_t row0 = warp0 * RPW + grp;
    const uint64_t pol_b = hint ? policy_evict_last() : policy_evict_normal();
    const T *bcol = B + col0;
    // a grid has at least 8 warps of at least 2 rows (stride >= 16), so every step used, <= M / 16 + 3, fits an int
    auto row_of = [&](int step) { return row0 + (int64_t)step * stride; };
    auto crow = [&](int step) { return C + row_of(step) * ldc + col0; };

    // walker: the next chunk whose A entries are loaded (row row_of(ws), entries [wb, we)), the offsets of the next two
    // rows, and the info bits of the chunk; rows at or past M are empty
    auto offsets = [&](int step, I &s, I &e) {
        const int64_t r = row_of(step);
        s = e = 0;
        if (r < M) {
            s = ldg_stream(off_lo + r);
            e = ldg_stream(off_hi + r);
        }
    };
    int ws = 0;
    I wb, we, ns, ne, n2s, n2e;
    offsets(0, wb, we);
    offsets(1, ns, ne);
    offsets(2, n2s, n2e);
    int wflags = kHead | (wb < we ? kTouched : 0);
    auto next_chunk = [&]() {
        PassChunk<T, I> c;
        const int64_t rem = (int64_t)we - (int64_t)wb;
        c.step = ws;
        c.info = wflags | (rem > L ? L : (rem > 0 ? (int)rem : 0)) | (rem > L ? 0 : kTail);
        c.col = 0;
        c.val = T(0);
        if (sub < rem) {
            c.col = ldg_stream(a_indices + (int64_t)wb + sub);
            c.val = ldg_stream(a_data + (int64_t)wb + sub);
        }
        if (rem > L) {
            wb += L;
            wflags = kTouched;
        } else {
            ++ws;
            wb = ns;
            we = ne;
            ns = n2s;
            ne = n2e;
            offsets(ws + 2, n2s, n2e);
            wflags = kHead | (wb < we ? kTouched : 0);
        }
        return c;
    };

    // a step whose chunks are all empty (rows without entries in this panel) skips the shuffles, gathers and FMAs
    auto issue = [&](uint4(&ring)[L], const PassChunk<T, I> &c) {
        if (!__any_sync(FULL, c.info & kCnt)) return;
#pragma unroll
        for (int u = 0; u < L; ++u) {
            const I cu = __shfl_sync(FULL, c.col, u, L);
            ldg_nc_v4_hint_if(ring[u], bcol + (int64_t)cu * ldb, u < (c.info & kCnt) && col_ok, pol_b);
        }
    };
    uint4 part = make_uint4(0, 0, 0, 0);  // C partial of the next chunk's row (later passes)
    auto load_partial = [&](const PassChunk<T, I> &c) {
        if ((c.info & kHead) && !first && (c.info & kTouched) && col_ok) part = ldg_cs_v4(crow(c.step));
    };
    PPack<T, VEC> acc;
    auto consume = [&](const uint4(&ring)[L], const PassChunk<T, I> &c) {
        if (c.info & kHead) {
            const uint4 a0 = (!first && (c.info & kTouched) && col_ok) ? part : make_uint4(0, 0, 0, 0);
            memcpy(&acc, &a0, 16);
        }
        if (__any_sync(FULL, c.info & kCnt)) {
#pragma unroll
            for (int u = 0; u < L; ++u) {
                const T v = __shfl_sync(FULL, c.val, u, L);
                if (u < (c.info & kCnt)) {
                    PPack<T, VEC> b;
                    memcpy(&b, &ring[u], 16);
#pragma unroll
                    for (int k = 0; k < VEC; ++k) acc.v[k] = add_rn(acc.v[k], mul_rn(v, b.v[k]));
                }
            }
        }
        // pass 0 writes every row (rows without entries get +0, as in K1); later passes only rows they touched
        if ((c.info & kTail) && row_of(c.step) < M && col_ok && (first || (c.info & kTouched))) {
            uint4 u;
            memcpy(&u, &acc, 16);
            stg_cs_v4(crow(c.step), u);
        }
    };

    uint4 ring0[L], ring1[L];
#pragma unroll
    for (int u = 0; u < L; ++u) ring0[u] = ring1[u] = make_uint4(0, 0, 0, 0);
    PassChunk<T, I> c0 = next_chunk(), c1 = next_chunk(), c2 = next_chunk();
    // one step: c0's gathers are in `cur`; c1's go into `nxt`
    auto step = [&](const uint4(&cur)[L], uint4(&nxt)[L]) {
        if (!__any_sync(FULL, row_of(c0.step) < M)) return false;
        issue(nxt, c1);
        const PassChunk<T, I> c3 = next_chunk();
        consume(cur, c0);
        load_partial(c1);
        c0 = c1;
        c1 = c2;
        c2 = c3;
        return true;
    };
    issue(ring0, c0);
    load_partial(c0);
    while (step(ring0, ring1) && step(ring1, ring0)) {
    }
}

// rows sorted by column? (flag[0] |= 1 when some row has a descending neighbour pair)
template <typename I>
__global__ void rows_sorted_kernel(int64_t M, const I *__restrict__ indptr, const I *__restrict__ indices,
                                   int *__restrict__ flag) {
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    bool bad = false;
    for (int64_t row = warp; row < M; row += nwarps) {
        const int64_t s = (int64_t)indptr[row], e = (int64_t)indptr[row + 1];
        for (int64_t p = s + lane; p + 1 < e; p += 32) bad |= indices[p + 1] < indices[p];
    }
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(flag, 1);
}

template <typename I>
__global__ void max_row_kernel(int64_t M, const I *__restrict__ indptr, unsigned long long *__restrict__ out) {
    unsigned long long m = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < M; r += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long n = (unsigned long long)((int64_t)indptr[r + 1] - (int64_t)indptr[r]);
        m = n > m ? n : m;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long v = __shfl_xor_sync(0xffffffffu, m, o);
        m = v > m ? v : m;
    }
    if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

// ---------------------------------------------------------------------------
// selection and host-side driver
// ---------------------------------------------------------------------------
// Defaults from tools/tune_panels.py on an H100 80GB HBM3 at 700 W (one-pass kernel 16.19 ms at C2 in the same run).
// C2 with 128-byte tiles: 14.89 / 12.34 / 10.90 / 10.17 / 10.03 / 10.94 ms at 8 / 12 / 16 / 24 / 32 / 48 MB per pass
// (24 MB kept: at a 400 W limit 24 MB gave 12.4-12.8 ms and 32 MB 13.7-14.4 ms over two runs); 64-byte tiles never
// below 20.8 ms (A is read once per tile, and a 4-entry chunk carries the same per-step cost), 256-byte tiles not below
// 12.86 ms.  With every column inside one 16 MB panel (all gathers after the first touch are L2 hits) the passes take
// 9.44 ms = 42 G line-gathers/s, 7 % below C2: the L2 line rate is the limit.  Forced passes vs the one-pass kernel
// around the thresholds: nnz / K = 10: 4.08 vs 1.81 ms, 30: 5.45 vs 5.08, 50: 7.04 vs 8.30, 70: 8.34 vs 11.48; K = 1e5
// (B about one L2): 1.54 vs 1.22 ms at nnz / K = 100, 2.95 vs 2.68 at 300; fp64 N = 64: 11.45 vs 17.17 ms.
constexpr int64_t kPanelBytes = 24ll << 20;  // B bytes (one panel x one tile) per pass
constexpr int kTileBytes = 128;               // column tile: one cache line per gather
constexpr int kL2Multiple = 2;                // tiled only when B is larger than this many L2s ...
constexpr int64_t kMinReuse = 48;             // ... and each B row is used at least this often (nnz / K)

static int64_t g_panel_bytes = 0;  // b2s_spmm_set_tiling (0 = default)
static int g_tile_bytes = 0;
int g_tile_hint = 1;  // 0: the passes load B with no L2 policy (b2s_spmm_set_variant(4, ...), for the sweep)

static int64_t l2_bytes() {
    static int64_t cached = 0;
    if (cached == 0) {
        int dev = 0, v = 0;
        if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, dev) == cudaSuccess &&
            v > 0)
            cached = v;
        else
            cached = 50ll << 20;  // H100 SXM
    }
    return cached;
}

// lanes per row group for a tile of `tile_bytes` (clamped to what N needs)
static int tile_lanes(int64_t N, size_t es) {
    const int tb = g_tile_bytes > 0 ? g_tile_bytes : kTileBytes;
    int lanes = tb <= 64 ? 4 : (tb <= 128 ? 8 : 16);
    const int64_t packs = (N * (int64_t)es + 15) / 16;
    while (lanes > 4 && packs <= lanes / 2) lanes /= 2;
    return lanes;
}

// Number of K panels of the tiled path for this call, or 0 for the one-pass kernel.
static int choose_panels(int dtype, int64_t K, int64_t N, int64_t nnz, bool vec_ok, int long_rows, int n_panels,
                         int rows_sorted) {
    if ((dtype != B2S_F32 && dtype != B2S_F64) || !vec_ok || rows_sorted == 0) return 0;
    if (n_panels >= 2) return n_panels;
    if (n_panels != 0 || long_rows || nnz < 0 || K <= 0) return 0;
    const size_t es = dtype_size(dtype);
    if (K * N * (int64_t)es <= kL2Multiple * l2_bytes() || nnz < kMinReuse * K) return 0;
    const int64_t slice_row = (int64_t)tile_lanes(N, es) * 16;  // B bytes of one row within one tile
    const int64_t budget = g_panel_bytes > 0 ? g_panel_bytes : kPanelBytes;
    const int64_t P = (K * slice_row + budget - 1) / budget;
    return (int)(P < 1 ? 1 : (P > 4096 ? 4096 : P));
}

template <typename T, typename I, int L>
static int launch_passes(int64_t M, int64_t N, const void *ad, const void *ai, const I *off, int P, const void *b,
                         int64_t ldb, void *out, int64_t ldc, const int *unsorted, cudaStream_t s) {
    constexpr int VEC = 16 / sizeof(T);
    constexpr int64_t TILE = (int64_t)L * VEC;  // columns per tile
    auto kern = spmm_tile_pass_kernel<T, I, L>;
    int occ = 1;
    B2S_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 256, 0));
    int64_t blocks = (int64_t)num_sms() * (occ < 1 ? 1 : occ);
    const int64_t need = (M + 8 * (32 / L) - 1) / (8 * (32 / L));
    if (blocks > need) blocks = need;
    for (int64_t c0 = 0; c0 < N; c0 += TILE) {
        for (int p = 0; p < P; ++p) {
            kern<<<(unsigned)blocks, 256, 0, s>>>(M, N, (const T *)ad, (const I *)ai, off + (int64_t)p * M,
                                                  off + (int64_t)(p + 1) * M, (const T *)b, ldb, (T *)out, ldc, c0,
                                                  p == 0 ? 1 : 0, g_tile_hint, unsorted);
            B2S_CHECK_LAUNCH();
        }
    }
    return B2S_OK;
}

template <typename T, typename I>
static int run_tiled(int dtype, int idx_bytes, int64_t M, int64_t K, int64_t N, const void *ad, const void *ai,
                     const void *ap, const void *b, int64_t ldb, void *out, int64_t ldc, int P, cudaStream_t s) {
    // scratch: the unsorted flag (16 bytes) then the (P+1) x M offsets
    void *scr = nullptr;
    int rc = scratch_alloc(&scr, 16 + (size_t)(P + 1) * M * sizeof(I), s);
    if (rc) return rc;
    int *flag = (int *)scr;
    I *off = (I *)((char *)scr + 16);
    B2S_CUDA(cudaMemsetAsync(flag, 0, 4, s));
    {
        int64_t blocks = (M * 32 + 255) / 256;
        const int64_t cap = (int64_t)num_sms() * 16;
        if (blocks > cap) blocks = cap;
        const int64_t width = (K + P - 1) / P;
        panel_offsets_kernel<I><<<(unsigned)blocks, 256, 0, s>>>(M, (const I *)ap, (const I *)ai, width < 1 ? 1 : width,
                                                                P, off, flag);
        B2S_CHECK_LAUNCH();
    }
    const int lanes = tile_lanes(N, sizeof(T));
    if (lanes == 4) rc = launch_passes<T, I, 4>(M, N, ad, ai, off, P, b, ldb, out, ldc, flag, s);
    else if (lanes == 8) rc = launch_passes<T, I, 8>(M, N, ad, ai, off, P, b, ldb, out, ldc, flag, s);
    else rc = launch_passes<T, I, 16>(M, N, ad, ai, off, P, b, ldb, out, ldc, flag, s);
    if (rc) return rc;
    // the one-pass kernel, which returns at entry unless some row was unsorted
    set_call_skew(0);
    set_call_guard(flag);
    rc = spmm_csr_dense_impl(dtype, idx_bytes, M, K, N, ad, ai, ap, b, ldb, out, ldc, s);
    set_call_guard(nullptr);
    set_call_skew(-1);
    if (rc) return rc;
    return scratch_free(scr, s);
}

}  // namespace b2s

using namespace b2s;

extern "C" {

/* 1 if every row of the CSR has non-decreasing column indices. Synchronises. */
int b2s_csr_rows_sorted(int idx_bytes, int64_t M, const void *indptr_dev, const void *indices_dev, int *sorted_host,
                        void *stream) {
    B2S_REQUIRE(sorted_host != nullptr, B2S_ERR_INVALID, "csr_rows_sorted: NULL output");
    *sorted_host = 1;
    if (M == 0) return B2S_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int *flag = nullptr;
    int rc = scratch_alloc((void **)&flag, 4, s);
    if (rc) return rc;
    B2S_CUDA(cudaMemsetAsync(flag, 0, 4, s));
    int64_t blocks = (M * 32 + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    if (idx_bytes == 4) rows_sorted_kernel<int32_t><<<(unsigned)blocks, 256, 0, s>>>(M, (const int32_t *)indptr_dev, (const int32_t *)indices_dev, flag);
    else rows_sorted_kernel<int64_t><<<(unsigned)blocks, 256, 0, s>>>(M, (const int64_t *)indptr_dev, (const int64_t *)indices_dev, flag);
    B2S_CHECK_LAUNCH();
    int h = 0;
    B2S_CUDA(cudaMemcpyAsync(&h, flag, 4, cudaMemcpyDeviceToHost, s));
    B2S_CUDA(cudaStreamSynchronize(s));
    scratch_free(flag, s);
    *sorted_host = h ? 0 : 1;
    return B2S_OK;
}

/* Largest number of stored entries in a row (decides whether the nnz-balanced long-row path is worth enabling). */
int b2s_csr_max_row_nnz(int idx_bytes, int64_t M, const void *indptr_dev, int64_t *max_host, void *stream) {
    B2S_REQUIRE(max_host != nullptr, B2S_ERR_INVALID, "csr_max_row_nnz: NULL output");
    *max_host = 0;
    if (M == 0) return B2S_OK;
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long *d = nullptr;
    int rc = scratch_alloc((void **)&d, 8, s);
    if (rc) return rc;
    B2S_CUDA(cudaMemsetAsync(d, 0, 8, s));
    int64_t blocks = (M + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    if (idx_bytes == 4) max_row_kernel<int32_t><<<(unsigned)blocks, 256, 0, s>>>(M, (const int32_t *)indptr_dev, d);
    else max_row_kernel<int64_t><<<(unsigned)blocks, 256, 0, s>>>(M, (const int64_t *)indptr_dev, d);
    B2S_CHECK_LAUNCH();
    unsigned long long h = 0;
    B2S_CUDA(cudaMemcpyAsync(&h, d, 8, cudaMemcpyDeviceToHost, s));
    B2S_CUDA(cudaStreamSynchronize(s));
    scratch_free(d, s);
    *max_host = (int64_t)h;
    return B2S_OK;
}

int b2s_spmm_set_tiling(int64_t panel_bytes, int tile_bytes) {
    B2S_REQUIRE(panel_bytes >= 0 && (tile_bytes == 0 || tile_bytes == 64 || tile_bytes == 128 || tile_bytes == 256),
                B2S_ERR_INVALID, "spmm_set_tiling: panel_bytes >= 0, tile_bytes in {0, 64, 128, 256}");
    g_panel_bytes = panel_bytes;
    g_tile_bytes = tile_bytes;
    return B2S_OK;
}

/*
 * K1 with explicit scheduling control.  n_panels == 1: the one-pass kernel.  n_panels >= 2: tiled passes with that many
 * K panels (fp32/fp64 with 16-byte aligned operands; otherwise the one-pass kernel).  n_panels == 0: tiled passes for
 * fp32/fp64 when B is larger than kL2Multiple L2s and nnz >= kMinReuse x K (P from the panel budget), else the one-pass
 * kernel.
 * rows_sorted is advisory (0 = known unsorted: skip the passes); the passes check the order on the device themselves.
 */
int b2s_spmm_csr_dense_ex(int dtype, int idx_bytes, int64_t M, int64_t K, int64_t N, int64_t nnz,
                          const void *a_data_dev, const void *a_indices_dev, const void *a_indptr_dev,
                          const void *b_dev, int64_t ldb, void *out_dev, int64_t ldc, int n_panels, int rows_sorted,
                          int long_rows, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    const size_t es = dtype_size(dtype);
    const bool vec_ok = (dtype == B2S_F32 || dtype == B2S_F64) && es != 0 && (N * es) % 16 == 0 &&
                        (ldb * es) % 16 == 0 && (ldc * es) % 16 == 0 && (((uintptr_t)b_dev | (uintptr_t)out_dev) & 15) == 0;
    B2S_REQUIRE(M >= 0 && K >= 0 && N >= 0, B2S_ERR_INVALID, "spmm: negative dimension");
    B2S_REQUIRE(ldb >= N && ldc >= N, B2S_ERR_INVALID, "spmm: ldb/ldc smaller than N");
    const int P = (M == 0 || N == 0) ? 0 : choose_panels(dtype, K, N, nnz, vec_ok, long_rows, n_panels, rows_sorted);
    if (P == 0) {
        set_call_skew(long_rows ? 1 : 0);
        const int rc = spmm_csr_dense_impl(dtype, idx_bytes, M, K, N, a_data_dev, a_indices_dev, a_indptr_dev, b_dev,
                                           ldb, out_dev, ldc, s);
        set_call_skew(-1);
        return rc;
    }
    B2S_REQUIRE(idx_bytes == 4 || idx_bytes == 8, B2S_ERR_INVALID, "spmm: idx_bytes must be 4 or 8");
#define B2S_TILED(T, I) \
    run_tiled<T, I>(dtype, idx_bytes, M, K, N, a_data_dev, a_indices_dev, a_indptr_dev, b_dev, ldb, out_dev, ldc, P, s)
    if (dtype == B2S_F32) return idx_bytes == 4 ? B2S_TILED(float, int32_t) : B2S_TILED(float, int64_t);
    return idx_bytes == 4 ? B2S_TILED(double, int32_t) : B2S_TILED(double, int64_t);
#undef B2S_TILED
}

}  // extern "C"
