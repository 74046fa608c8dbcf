// spmm.cu -- K1: CSR x dense -> dense, exact-order (bit-identical to the reference loop).
//
// Replaces _dot_csr_ndarray (sparse/numba_backend/_common.py:720-755).
//
// Work decomposition ("row-split"): a group of G lanes (G = 32 for N*sizeof(T) >= 512 B) owns one
// row of A and a tile of G*VEC output columns; lane l keeps VEC accumulators in registers for the
// whole row, so every out[i,j] is summed in the stored order of row i with separate product and
// sum roundings (mul_rn/add_rn) -- the same operation sequence as the reference, hence bit-exact.
//
// Memory behaviour (fp32, N = 128): one nnz = one 512-byte row of B = one 16-byte load per lane
// (4 full 128-B lines per warp request).  The A stream (indices + data) is read coalesced, 32
// entries at a time, broadcast with shuffles, and prefetched one chunk ahead.  U independent
// B-row loads are in flight per warp (Little's law on H100: 3.35 TB/s x ~1 us over 132 SMs needs ~25 KB in flight per SM).
// B rows carry an L2 evict_last policy (B is the only operand with reuse), the A stream and the
// C stores are streaming (evict-first).
#include "common.cuh"

namespace b2s {

template <typename T, int VEC>
struct alignas(sizeof(T) * VEC) Pack {
    T v[VEC];
};

template <typename T, int VEC>
__device__ __forceinline__ Pack<T, VEC> load_b(const T *p, uint64_t pol) {
    Pack<T, VEC> r;
    if constexpr (sizeof(T) * VEC == 16) {
        uint4 u = ldg_nc_v4_hint(p, pol);
        memcpy(&r, &u, 16);
    } else {
        static_assert(VEC == 1, "only 16-byte or scalar packs");
        r.v[0] = __ldg(p);
    }
    return r;
}

template <typename T, int VEC>
__device__ __forceinline__ void store_c(T *p, const T (&acc)[VEC]) {
    if constexpr (sizeof(T) * VEC == 16) {
        uint4 u;
        memcpy(&u, acc, 16);
        stg_cs_v4(p, u);
    } else {
        p[0] = acc[0];
    }
}

// ---------------------------------------------------------------------------
// Variant 1: register-staged gather (LDG.128, U loads in flight per group)
// ---------------------------------------------------------------------------
template <typename T, typename I, int VEC, int G, int U>
__global__ void __launch_bounds__(256)
spmm_csr_dense_kernel(int64_t M, int64_t N, const T *__restrict__ a_data, const I *__restrict__ a_indices,
                      const I *__restrict__ a_indptr, const T *__restrict__ B, int64_t ldb, T *__restrict__ C,
                      int64_t ldc, const uint8_t *__restrict__ skip, const int *__restrict__ guard) {
    static_assert(G >= 1 && G <= 32 && (G & (G - 1)) == 0, "G must be a power of two <= 32");
    static_assert(U <= G && G % U == 0, "U must divide G");
    if (guard != nullptr && *guard == 0) return;  // the tiled passes (spmm_panel.cu) computed this call
    constexpr unsigned FULL = 0xffffffffu;
    constexpr int ROWS_PER_WARP = 32 / G;
    const int lane = threadIdx.x & 31;
    const int sub = lane & (G - 1);
    const int64_t warp_global = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t row = warp_global * ROWS_PER_WARP + lane / G;
    const int64_t col0 = ((int64_t)blockIdx.y * G + sub) * VEC;
    const bool row_ok = row < M;
    const bool col_ok = col0 < N;

    int64_t base = 0, end = 0;
    // rows marked in `skip` are long rows handled by the column-split kernel (spmm_skew.cu)
    const bool skipped = skip != nullptr && row_ok && skip[row] != 0;
    if (row_ok && !skipped) {
        base = (int64_t)a_indptr[row];
        end = (int64_t)a_indptr[row + 1];
    }
    const uint64_t pol_b = policy_evict_last();
    const T *bcol = B + col0;

    T acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = T(0);

    // prefetch the first chunk of the row's (index, value) stream
    I col_n = 0;
    T val_n = T(0);
    if (base + sub < end) {
        col_n = ldg_stream(a_indices + base + sub);
        val_n = ldg_stream(a_data + base + sub);
    }

    auto any = [&](bool p) -> bool {
        if constexpr (G == 32) return p;  // whole warp shares the row: already uniform
        else return __any_sync(FULL, p);
    };

    while (any(base < end)) {
        const I col = col_n;
        const T val = val_n;
        int64_t rem = end - base;
        const int cnt = rem > G ? G : (rem > 0 ? (int)rem : 0);
        const int64_t nb = base + G;
        if (nb + sub < end) {  // prefetch the next chunk while this one is consumed
            col_n = ldg_stream(a_indices + nb + sub);
            val_n = ldg_stream(a_data + nb + sub);
        }
#pragma unroll 1
        for (int j = 0; j < G; j += U) {
            if (!any(j < cnt)) break;
            Pack<T, VEC> bv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const I c = __shfl_sync(FULL, col, j + u, G);
                if (j + u < cnt && col_ok) bv[u] = load_b<T, VEC>(bcol + (int64_t)c * ldb, pol_b);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const T v = __shfl_sync(FULL, val, j + u, G);
                if (j + u < cnt) {
#pragma unroll
                    for (int k = 0; k < VEC; ++k) acc[k] = add_rn(acc[k], mul_rn(v, bv[u].v[k]));
                }
            }
        }
        base = nb;
    }
    if (row_ok && col_ok && !skipped) store_c<T, VEC>(C + row * ldc + col0, acc);
}

template <typename T, typename I, int VEC, int G, int U, int MINB>
__global__ void __launch_bounds__(256, MINB)
spmm_csr_dense_dyn_kernel(int64_t M, int64_t N, const T *__restrict__ a_data, const I *__restrict__ a_indices,
                      const I *__restrict__ a_indptr, const T *__restrict__ B, int64_t ldb, T *__restrict__ C,
                      int64_t ldc, const uint8_t *__restrict__ skip, unsigned int *__restrict__ row_counter,
                      const int *__restrict__ guard) {
    static_assert(G >= 1 && G <= 32 && (G & (G - 1)) == 0, "G must be a power of two <= 32");
    static_assert(U <= G && G % U == 0, "U must divide G");
    if (guard != nullptr && *guard == 0) return;  // the tiled passes (spmm_panel.cu) computed this call
    constexpr unsigned FULL = 0xffffffffu;
    constexpr int ROWS_PER_WARP = 32 / G;
    const int lane = threadIdx.x & 31;
    const int sub = lane & (G - 1);
    static_assert(G == 32, "the dynamic-row variant is warp per row");
    const int64_t col0 = ((int64_t)blockIdx.y * G + sub) * VEC;
    const bool col_ok = col0 < N;
    constexpr unsigned ROWS_PER_TICKET = 2;
    for (;;) {
    // rows are dealt out two at a time by a global counter: a warp that drew a long row simply draws fewer rows, so
    // no CTA sits on one busy warp (skewed matrices: the row-split grid's static 8 rows per CTA idles 7 warps)
    unsigned first = 0;
    if (lane == 0) first = atomicAdd(row_counter + blockIdx.y, ROWS_PER_TICKET);
    first = __shfl_sync(FULL, first, 0);
    if ((int64_t)first >= M) break;
    for (unsigned rr = 0; rr < ROWS_PER_TICKET; ++rr) {
    const int64_t row = (int64_t)first + rr;
    const bool row_ok = row < M;

    int64_t base = 0, end = 0;
    // rows marked in `skip` are long rows handled by the column-split kernel (spmm_skew.cu)
    const bool skipped = skip != nullptr && row_ok && skip[row] != 0;
    if (row_ok && !skipped) {
        base = (int64_t)a_indptr[row];
        end = (int64_t)a_indptr[row + 1];
    }
    const uint64_t pol_b = policy_evict_last();
    const T *bcol = B + col0;

    T acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = T(0);

    // prefetch the first chunk of the row's (index, value) stream
    I col_n = 0;
    T val_n = T(0);
    if (base + sub < end) {
        col_n = ldg_stream(a_indices + base + sub);
        val_n = ldg_stream(a_data + base + sub);
    }

    auto any = [&](bool p) -> bool {
        if constexpr (G == 32) return p;  // whole warp shares the row: already uniform
        else return __any_sync(FULL, p);
    };

    while (any(base < end)) {
        const I col = col_n;
        const T val = val_n;
        int64_t rem = end - base;
        const int cnt = rem > G ? G : (rem > 0 ? (int)rem : 0);
        const int64_t nb = base + G;
        if (nb + sub < end) {  // prefetch the next chunk while this one is consumed
            col_n = ldg_stream(a_indices + nb + sub);
            val_n = ldg_stream(a_data + nb + sub);
        }
#pragma unroll 1
        for (int j = 0; j < G; j += U) {
            if (!any(j < cnt)) break;
            Pack<T, VEC> bv[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const I c = __shfl_sync(FULL, col, j + u, G);
                if (j + u < cnt && col_ok) bv[u] = load_b<T, VEC>(bcol + (int64_t)c * ldb, pol_b);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const T v = __shfl_sync(FULL, val, j + u, G);
                if (j + u < cnt) {
#pragma unroll
                    for (int k = 0; k < VEC; ++k) acc[k] = add_rn(acc[k], mul_rn(v, bv[u].v[k]));
                }
            }
        }
        base = nb;
    }
    if (row_ok && col_ok && !skipped) store_c<T, VEC>(C + row * ldc + col0, acc);
    }
    }
}

// ---------------------------------------------------------------------------
// Variant 2: 1-D bulk-TMA gather (cp.async.bulk -> shared-memory ring, mbarrier complete_tx).
// One warp per row; ring of 32 stages of ROWB bytes per warp; position p of the row's nnz stream
// uses stage p % 32 and its lane p % 32 is both the holder of (col, val) for p and the issuer of
// the bulk copy, so 32 B-row copies are always in flight per warp without any register staging.
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar, uint64_t pol) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
            "r"(dst),
        "l"(src), "r"(bytes), "r"(bar), "l"(pol)
        : "memory");
}

template <typename T, typename I, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
spmm_csr_dense_tma_kernel(int64_t M, int N, const T *__restrict__ a_data, const I *__restrict__ a_indices,
                          const I *__restrict__ a_indptr, const T *__restrict__ B, int64_t ldb, T *__restrict__ C,
                          int64_t ldc) {
    // N * sizeof(T) == 512 (one 16-byte pack per lane), checked by the host.
    constexpr int VEC = 16 / sizeof(T);
    constexpr int ROWB = 512;
    constexpr unsigned FULL = 0xffffffffu;
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    unsigned char *ring = smem + (size_t)warp * 32 * ROWB;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + (size_t)WARPS * 32 * ROWB) + warp * 32;
    const uint32_t my_bar = smem_u32(bars + lane);
    const uint32_t my_stage = smem_u32(ring + lane * ROWB);
    mbar_init(my_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();

    const uint64_t pol_b = policy_evict_last();
    uint32_t phase = 0;  // parity of the ring pass (same for every stage: stages advance in lock step per chunk)

    const int64_t warps_total = (int64_t)gridDim.x * WARPS;
    for (int64_t row = (int64_t)blockIdx.x * WARPS + warp; row < M; row += warps_total) {
        int64_t base = (int64_t)a_indptr[row];
        const int64_t end = (int64_t)a_indptr[row + 1];
        T acc[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) acc[k] = T(0);

        // fill: every lane issues the copy for its own position of the first chunk
        I col = 0;
        T val = T(0);
        if (base + lane < end) {
            col = ldg_stream(a_indices + base + lane);
            val = ldg_stream(a_data + base + lane);
            mbar_expect_tx(my_bar, ROWB);
            bulk_g2s(my_stage, B + (int64_t)col * ldb, ROWB, my_bar, pol_b);
        }
        while (base < end) {
            const int64_t rem = end - base;
            const int cnt = rem > 32 ? 32 : (int)rem;
            const int64_t nb = base + 32;
            // (col, val) of the NEXT chunk, needed by this lane when its stage is released
            I col_n = 0;
            T val_n = T(0);
            const bool has_next = nb + lane < end;
            if (has_next) {
                col_n = ldg_stream(a_indices + nb + lane);
                val_n = ldg_stream(a_data + nb + lane);
            }
            for (int j = 0; j < cnt; ++j) {
                const uint32_t bar_j = smem_u32(bars + j);
                mbar_wait(bar_j, phase);
                Pack<T, VEC> bv;
                {
                    const uint4 u = *reinterpret_cast<const uint4 *>(ring + j * ROWB + lane * 16);
                    memcpy(&bv, &u, 16);
                }
                const T v = __shfl_sync(FULL, val, j);
                __syncwarp();  // all lanes have read stage j: it may be overwritten
                if (lane == j && has_next) {
                    mbar_expect_tx(my_bar, ROWB);
                    bulk_g2s(my_stage, B + (int64_t)col_n * ldb, ROWB, my_bar, pol_b);
                }
#pragma unroll
                for (int k = 0; k < VEC; ++k) acc[k] = add_rn(acc[k], mul_rn(v, bv.v[k]));
            }
            // stages j >= cnt were not used in this pass: keep every barrier's parity in lock step
            // by completing an empty phase on them (only happens on the last chunk of a row).
            if (lane >= cnt) {
                asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(my_bar) : "memory");
            }
            phase ^= 1;
            col = col_n;
            val = val_n;
            base = nb;
        }
        store_c<T, VEC>(C + row * ldc + lane * VEC, acc);
    }
}

// ---------------------------------------------------------------------------
// host-side dispatch
// ---------------------------------------------------------------------------
static int g_variant = 1;
static int g_unroll = 8;
static int g_skew = 0;  // process-wide default of the long-row (nnz-balanced) path; per-call override below
static int g_dyn_form = 0;     // tuning of the dynamic-row kernel (see dispatch_g)
static int g_static_rows = 0;  // 1 = the static one-row-per-warp grid instead of the dynamic-row default (A/B, tests)
static thread_local int t_skew = -1;
void set_call_skew(int v) { t_skew = v; }
static thread_local const int *t_guard = nullptr;
void set_call_guard(const int *guard) { t_guard = guard; }

// spmm_skew.cu
template <typename T, typename I>
int skew_begin(int64_t M, int64_t N, const void *ad, const void *ai, const void *ap, const void *b, int64_t ldb,
               void *out, int64_t ldc, cudaStream_t s, uint8_t **skip_out, bool aligned16);
int skew_end(cudaStream_t s, uint8_t *skip);
unsigned int *skew_row_counter();  // 64 zero-initialisable counters of the in-flight call (nullptr: unavailable)

template <typename T, typename I, int VEC, int G, int U>
static int launch_v1(int64_t M, int64_t N, const void *ad, const void *ai, const void *ap, const void *b, int64_t ldb,
                     void *out, int64_t ldc, cudaStream_t s, const uint8_t *skip = nullptr) {
    constexpr int THREADS = 256;
    constexpr int rows_per_block = (THREADS / 32) * (32 / G);
    const int64_t gx = (M + rows_per_block - 1) / rows_per_block;
    const int64_t gy = (N + (int64_t)G * VEC - 1) / ((int64_t)G * VEC);
    B2S_REQUIRE(gx <= 2147483647LL && gy <= 65535, B2S_ERR_OVERFLOW, "spmm: grid too large (M=%lld N=%lld)",
                (long long)M, (long long)N);
    dim3 grid((unsigned)gx, (unsigned)gy);
    spmm_csr_dense_kernel<T, I, VEC, G, U><<<grid, THREADS, 0, s>>>(M, N, (const T *)ad, (const I *)ai, (const I *)ap,
                                                                    (const T *)b, ldb, (T *)out, ldc, skip, t_guard);
    B2S_CHECK_LAUNCH();
    return B2S_OK;
}

template <typename T, typename I, int VEC>
static int dispatch_g(int64_t M, int64_t N, const void *ad, const void *ai, const void *ap, const void *b, int64_t ldb,
                      void *out, int64_t ldc, cudaStream_t s) {
    const int64_t packs = (N + VEC - 1) / VEC;  // column packs per row
#define B2S_GO(G, U) return launch_v1<T, I, VEC, G, U>(M, N, ad, ai, ap, b, ldb, out, ldc, s)
    if (packs >= 32) {
        // Default for wide B rows: PERSISTENT warps that draw rows two at a time from a global counter
        // (spmm_csr_dense_dyn_kernel).  Written for skewed matrices, it also wins on the uniform C2 matrix: on an H100 SXM
        // (700 W) 16.19 ms vs 16.59 ms for the static one-row-per-warp grid (no tail of partially idle CTAs);
        // bit-identical, since the per-row loop is the same code.
        const bool skew = (t_skew >= 0 ? t_skew : g_skew) && g_variant == 1 && M >= 4096;
        const int64_t gy = (N + (int64_t)32 * VEC - 1) / ((int64_t)32 * VEC);
        if (g_variant == 1 && g_unroll == 8 && g_static_rows == 0 && gy <= 64) {
            // nnz-balanced mode on top: rows longer than max(512, 4 x mean) go to the column-split kernel on a side
            // stream (they start first and run concurrently with the row kernel, which skips them)
            uint8_t *skip = nullptr;
            int rc = B2S_OK;
            unsigned int *counter = nullptr;
            if (skew) {
                rc = skew_begin<T, I>(M, N, ad, ai, ap, b, ldb, out, ldc, s, &skip, VEC > 1);
                if (rc) return rc;
                counter = skew_row_counter();
            }
            unsigned int *own = nullptr;
            if (counter == nullptr) {
                if ((rc = scratch_alloc((void **)&own, 64 * sizeof(unsigned int), s))) return rc;
                counter = own;
            }
            B2S_CUDA(cudaMemsetAsync(counter, 0, 64 * sizeof(unsigned int), s));
            // g_dyn_form (tuning): 0 = 8 gathers in flight per lane, 4 CTAs per SM (the default); 1 = 16 in flight, 4 CTAs;
            // 2 = 8 in flight, 5 CTAs per SM; 3 = 16 in flight, 3 CTAs per SM.  H100 SXM at C2: 16.19 / 23.65 / 17.80 /
            // 18.36 ms (tools/tune_k1_dyn.py)
            using KernT = void (*)(int64_t, int64_t, const T *, const I *, const I *, const T *, int64_t, T *, int64_t,
                                   const uint8_t *, unsigned int *, const int *);
            KernT kern = spmm_csr_dense_dyn_kernel<T, I, VEC, 32, 8, 4>;
            if (g_dyn_form == 1) kern = spmm_csr_dense_dyn_kernel<T, I, VEC, 32, 16, 4>;
            else if (g_dyn_form == 2) kern = spmm_csr_dense_dyn_kernel<T, I, VEC, 32, 8, 5>;
            else if (g_dyn_form == 3) kern = spmm_csr_dense_dyn_kernel<T, I, VEC, 32, 16, 3>;
            int occ = 1;
            B2S_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 256, 0));
            const int occ_cached = occ < 1 ? 1 : occ;
            int64_t blocks = (int64_t)num_sms() * occ_cached;
            const int64_t need = (M + 15) / 16;  // 8 warps x 2 rows per ticket
            if (blocks > need) blocks = need > 0 ? need : 1;
            dim3 grid((unsigned)blocks, (unsigned)gy);
            kern<<<grid, 256, 0, s>>>(M, N, (const T *)ad, (const I *)ai, (const I *)ap, (const T *)b, ldb, (T *)out, ldc,
                                      skip, counter, t_guard);
            B2S_CHECK_LAUNCH();
            if (own) scratch_free(own, s);
            return skew ? skew_end(s, skip) : B2S_OK;
        }
        if (g_unroll == 4) B2S_GO(32, 4);
        if (g_unroll == 16) B2S_GO(32, 16);
        if (g_unroll == 32) B2S_GO(32, 32);
        B2S_GO(32, 8);
    }
    if (packs > 8) B2S_GO(16, 8);
    if (packs > 4) B2S_GO(8, 8);
    if (packs > 2) B2S_GO(4, 4);
    if (packs > 1) B2S_GO(2, 2);
    B2S_GO(1, 1);
#undef B2S_GO
}

template <typename T, typename I>
static int dispatch_vec(int64_t M, int64_t N, const void *ad, const void *ai, const void *ap, const void *b,
                        int64_t ldb, void *out, int64_t ldc, cudaStream_t s) {
    constexpr int VEC = 16 / sizeof(T);
    const bool vec_ok = (N % VEC == 0) && (ldb % VEC == 0) && (ldc % VEC == 0) && (((uintptr_t)b & 15) == 0) &&
                        (((uintptr_t)out & 15) == 0);
    if (vec_ok) {
        if (g_variant == 2 && N * (int64_t)sizeof(T) == 512) {
            constexpr int WARPS = 4;
            const size_t smem = (size_t)WARPS * 32 * 512 + (size_t)WARPS * 32 * 8;
            auto kern = spmm_csr_dense_tma_kernel<T, I, WARPS>;
            B2S_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            int64_t blocks = (M + WARPS - 1) / WARPS;
            const int64_t cap = (int64_t)num_sms() * 3;  // 3 x 66 KB CTAs per SM, persistent over rows
            if (blocks > cap) blocks = cap;
            kern<<<(unsigned)blocks, WARPS * 32, smem, s>>>(M, (int)N, (const T *)ad, (const I *)ai, (const I *)ap,
                                                            (const T *)b, ldb, (T *)out, ldc);
            B2S_CHECK_LAUNCH();
            return B2S_OK;
        }
        return dispatch_g<T, I, VEC>(M, N, ad, ai, ap, b, ldb, out, ldc, s);
    }
    return dispatch_g<T, I, 1>(M, N, ad, ai, ap, b, ldb, out, ldc, s);
}

template <typename T>
static int dispatch_idx(int idx_bytes, int64_t M, int64_t N, const void *ad, const void *ai, const void *ap,
                        const void *b, int64_t ldb, void *out, int64_t ldc, cudaStream_t s) {
    if (idx_bytes == 4) return dispatch_vec<T, int32_t>(M, N, ad, ai, ap, b, ldb, out, ldc, s);
    return dispatch_vec<T, int64_t>(M, N, ad, ai, ap, b, ldb, out, ldc, s);
}

int spmm_csr_dense_impl(int dtype, int idx_bytes, int64_t M, int64_t K, int64_t N, const void *ad, const void *ai,
                        const void *ap, const void *b, int64_t ldb, void *out, int64_t ldc, cudaStream_t s) {
    B2S_REQUIRE(M >= 0 && K >= 0 && N >= 0, B2S_ERR_INVALID, "spmm: negative dimension");
    B2S_REQUIRE(idx_bytes == 4 || idx_bytes == 8, B2S_ERR_INVALID, "spmm: idx_bytes must be 4 or 8");
    B2S_REQUIRE(ldb >= N && ldc >= N, B2S_ERR_INVALID, "spmm: ldb/ldc smaller than N");
    if (M == 0 || N == 0) return B2S_OK;
    switch (dtype) {
        case B2S_F32: return dispatch_idx<float>(idx_bytes, M, N, ad, ai, ap, b, ldb, out, ldc, s);
        case B2S_F64: return dispatch_idx<double>(idx_bytes, M, N, ad, ai, ap, b, ldb, out, ldc, s);
        case B2S_I32: return dispatch_idx<int32_t>(idx_bytes, M, N, ad, ai, ap, b, ldb, out, ldc, s);
        case B2S_I64: return dispatch_idx<int64_t>(idx_bytes, M, N, ad, ai, ap, b, ldb, out, ldc, s);
        default: set_error("spmm: unsupported dtype %d", dtype); return B2S_ERR_UNSUPPORTED;
    }
}

// int64 -> int32 narrowing of index arrays on the device (host arrays are np.intp)
__global__ void narrow_i64_i32_kernel(const int64_t *__restrict__ in, int32_t *__restrict__ out, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = (int32_t)in[i];
}

int narrow_i64_i32(const int64_t *in, int32_t *out, int64_t n, cudaStream_t s) {
    if (n == 0) return B2S_OK;
    int64_t blocks = (n + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    narrow_i64_i32_kernel<<<(unsigned)blocks, 256, 0, s>>>(in, out, n);
    B2S_CHECK_LAUNCH();
    return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_spmm_set_skew(int enabled) {
    g_skew = enabled ? 1 : 0;
    return B2S_OK;
}

int b2s_spmm_set_variant(int variant, int unroll) {
    g_variant = (variant == 2) ? 2 : 1;
    g_static_rows = (variant == 3) ? 1 : 0;
    g_dyn_form = (variant >= 10 && variant <= 13) ? variant - 10 : 0;  // 10..13: forms of the dynamic-row kernel
    g_unroll = (unroll == 4 || unroll == 16 || unroll == 32) ? unroll : 8;
    g_tile_hint = (variant == 4) ? 0 : 1;  // 4: tiled passes load B with no L2 policy (evict_last A/B)
    return B2S_OK;
}

int b2s_spmm_csr_dense(int dtype, int idx_bytes, int64_t M, int64_t K, int64_t N, const void *a_data_dev,
                       const void *a_indices_dev, const void *a_indptr_dev, const void *b_dev, int64_t ldb,
                       void *out_dev, int64_t ldc, void *stream) {
    return spmm_csr_dense_impl(dtype, idx_bytes, M, K, N, a_data_dev, a_indices_dev, a_indptr_dev, b_dev, ldb, out_dev,
                               ldc, (cudaStream_t)stream);
}

}  // extern "C"
