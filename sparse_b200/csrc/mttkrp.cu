// mttkrp.cu -- K10: mode-n MTTKRP of a sparse tensor of order 2..8, nnz-balanced and in a fixed order.
//
//   out[i, r] = sum over stored e with i_n(e) = i of  v_e * prod_{m != n} U_m[i_m(e), r]
//
// Input is the mode stream S_n: the tensor's entries ordered by coordinate n (stable in C order), as N coordinate
// arrays plus the values.  The stream is cut into chunks of B2S_MTTKRP_CHUNK consecutive entries; a group of G lanes
// owns one (chunk, column tile) and walks its chunk in stream order, so the work per group is the same whatever the
// slice lengths are (a 100-slice mode of a 1e8-entry tensor is as balanced as a 1e6-slice one).  Lane l of a group
// owns VEC consecutive columns; the (coordinates, value) stream is read G entries at a time with streaming loads and
// broadcast by shuffles (as K1 does), and the N-1 factor rows of U entries are gathered at once with 16-byte loads
// under an L2 evict_last policy (the factors are the reused operand).
//
// A row that starts and ends inside a chunk is written straight to `out`.  The first and the last row of a chunk may
// continue into the neighbouring chunk: their partials go to a scratch array (two slots per chunk), and a second
// kernel adds each crossing row's partials in chunk order.  Rows without entries are zeroed by the chunk that follows
// them in the stream (the last chunk zeroes the rows after it).  No atomics: the result is the order of
// include/sparse_b200.h, independent of grid size and scheduling.
#include "common.cuh"

namespace b2s {

constexpr int64_t kChunk = B2S_MTTKRP_CHUNK;
constexpr int kMaxOther = 7;  // order <= 8

// the N-1 gathered modes, in ascending mode order
template <typename I>
struct OtherModes {
    const I *coord[kMaxOther];
    const void *fac[kMaxOther];
    int64_t ld[kMaxOther];
};

template <typename T, int VEC>
struct alignas(sizeof(T) * VEC) MPack {
    T v[VEC];
};

template <typename T, int VEC>
__device__ __forceinline__ MPack<T, VEC> m_load(const T *p, uint64_t pol) {
    MPack<T, VEC> r;
    if constexpr (sizeof(T) * VEC == 16) {
        const uint4 u = ldg_nc_v4_hint(p, pol);
        memcpy(&r, &u, 16);
    } else {
        static_assert(VEC == 1, "only 16-byte or scalar packs");
        r.v[0] = __ldg(p);
    }
    return r;
}

template <typename T, int VEC>
__device__ __forceinline__ void m_store(T *p, const T (&v)[VEC]) {
    if constexpr (sizeof(T) * VEC == 16) {
        uint4 u;
        memcpy(&u, v, 16);
        *reinterpret_cast<uint4 *>(p) = u;
    } else {
        p[0] = v[0];
    }
}

template <typename T, int VEC>
__device__ __forceinline__ void m_zero_rows(T *out, int64_t ldo, int64_t from, int64_t to, int64_t col0) {
    T z[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) z[k] = T(0);
    for (int64_t r = from; r < to; ++r) m_store<T, VEC>(out + r * ldo + col0, z);
}

template <typename T, typename I, int VEC, int G, int U>
__global__ void __launch_bounds__(256)
mttkrp_mode_kernel(const OtherModes<I> om, const int n_other, const I *__restrict__ rowc, const T *__restrict__ vals,
                   const int64_t nnz, const int64_t rows, const int64_t R, T *__restrict__ out, const int64_t ldo,
                   T *__restrict__ pieces, const int64_t ldp) {
    static_assert(G >= 1 && G <= 32 && (G & (G - 1)) == 0, "G must be a power of two <= 32");
    static_assert(U <= G && G % U == 0, "U must divide G");
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int sub = lane & (G - 1);
    const int64_t chunk = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * (32 / G) + lane / G;
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    const int64_t col0 = ((int64_t)blockIdx.y * G + sub) * VEC;
    const bool col_ok = col0 < R;

    int64_t base = 0, end = 0, row_first = 0, row_last = 0;
    bool head_cross = false, tail_cross = false;
    if (chunk < nchunks) {
        base = chunk * kChunk;
        end = base + kChunk < nnz ? base + kChunk : nnz;
        row_first = (int64_t)rowc[base];
        row_last = (int64_t)rowc[end - 1];
        const int64_t prev = chunk > 0 ? (int64_t)rowc[base - 1] : -1;
        head_cross = prev == row_first;
        tail_cross = end < nnz && (int64_t)rowc[end] == row_last;
        if (col_ok) {
            m_zero_rows<T, VEC>(out, ldo, prev + 1, row_first, col0);
            if (end == nnz) m_zero_rows<T, VEC>(out, ldo, row_last + 1, rows, col0);
        }
    }
    const uint64_t pol = policy_evict_last();

    T acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = T(0);
    int64_t cur = row_first;

    // the first row of the chunk goes to slot 0 when it crosses either boundary, the last row to slot 1 when it
    // continues into the next chunk; every other row is complete here
    auto flush = [&](int64_t r) {
        if (!col_ok) return;
        T *dst;
        if (r == row_first && (head_cross || (r == row_last && tail_cross))) dst = pieces + (2 * chunk) * ldp + col0;
        else if (r == row_last && tail_cross) dst = pieces + (2 * chunk + 1) * ldp + col0;
        else dst = out + r * ldo + col0;
        m_store<T, VEC>(dst, acc);
    };

    auto any = [&](bool p) -> bool {
        if constexpr (G == 32) return p;  // one chunk per warp: already uniform
        else return __any_sync(FULL, p);
    };

    // prefetch the first G entries of the stream
    I rc_n = 0;
    I c_n[kMaxOther];
    T v_n = T(0);
#pragma unroll
    for (int m = 0; m < kMaxOther; ++m) c_n[m] = 0;
    if (base + sub < end) {
        rc_n = ldg_stream(rowc + base + sub);
        v_n = ldg_stream(vals + base + sub);
#pragma unroll
        for (int m = 0; m < kMaxOther; ++m)
            if (m < n_other) c_n[m] = ldg_stream(om.coord[m] + base + sub);
    }

    while (any(base < end)) {
        const I rc = rc_n;
        const T v = v_n;
        I c[kMaxOther];
#pragma unroll
        for (int m = 0; m < kMaxOther; ++m) c[m] = c_n[m];
        const int64_t rem = end - base;
        const int cnt = rem > G ? G : (rem > 0 ? (int)rem : 0);
        const int64_t nb = base + G;
        if (nb + sub < end) {  // next G entries while these are consumed
            rc_n = ldg_stream(rowc + nb + sub);
            v_n = ldg_stream(vals + nb + sub);
#pragma unroll
            for (int m = 0; m < kMaxOther; ++m)
                if (m < n_other) c_n[m] = ldg_stream(om.coord[m] + nb + sub);
        }
#pragma unroll 1
        for (int j = 0; j < G; j += U) {
            if (!any(j < cnt)) break;
            T p[U][VEC];
            int64_t rr[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const T vu = __shfl_sync(FULL, v, j + u, G);
                rr[u] = (int64_t)__shfl_sync(FULL, rc, j + u, G);
#pragma unroll
                for (int k = 0; k < VEC; ++k) p[u][k] = vu;
            }
            // (((v * U_a) * U_b) * ...) over the other modes in ascending order, each product rounded
#pragma unroll
            for (int m = 0; m < kMaxOther; ++m) {
                if (m < n_other) {
                    const T *fm = (const T *)om.fac[m] + col0;
                    const int64_t ldm = om.ld[m];
                    MPack<T, VEC> f[U];
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const I ix = __shfl_sync(FULL, c[m], j + u, G);
                        if (j + u < cnt && col_ok) f[u] = m_load<T, VEC>(fm + (int64_t)ix * ldm, pol);
                        else {
#pragma unroll
                            for (int k = 0; k < VEC; ++k) f[u].v[k] = T(0);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < U; ++u)
#pragma unroll
                        for (int k = 0; k < VEC; ++k) p[u][k] = mul_rn(p[u][k], f[u].v[k]);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (j + u < cnt) {
                    if (rr[u] != cur) {
                        flush(cur);
                        if (col_ok) m_zero_rows<T, VEC>(out, ldo, cur + 1, rr[u], col0);
                        cur = rr[u];
#pragma unroll
                        for (int k = 0; k < VEC; ++k) acc[k] = T(0);
                    }
#pragma unroll
                    for (int k = 0; k < VEC; ++k) acc[k] = add_rn(acc[k], p[u][k]);
                }
            }
        }
        base = nb;
    }
    if (chunk < nchunks) flush(cur);
}

// One warp per chunk boundary b: the row that crosses b and no earlier boundary adds its partials, chunk b-1's piece
// first, then the head pieces of chunks b .. last (found by bisection over the chunks' first entries).
template <typename T, typename I>
__global__ void __launch_bounds__(256)
mttkrp_combine_kernel(const I *__restrict__ rowc, const int64_t nnz, const int64_t R, const T *__restrict__ pieces,
                      const int64_t ldp, T *__restrict__ out, const int64_t ldo) {
    const int64_t b = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) + 1;
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    const int64_t col = (int64_t)blockIdx.y * 32 + (threadIdx.x & 31);
    if (b >= nchunks || col >= R) return;
    const int64_t p = b * kChunk;
    const I r = rowc[p];
    if (rowc[p - 1] != r) return;                  // no row crosses b
    if (b > 1 && rowc[p - kChunk - 1] == r) return;  // the row crosses b-1 too: that boundary owns it
    int64_t lo = b, hi = nchunks - 1;
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (rowc[mid * kChunk] == r) lo = mid;
        else hi = mid - 1;
    }
    const int64_t slot = rowc[p - kChunk] == r ? 0 : 1;
    T acc = T(0);
    acc = add_rn(acc, pieces[(2 * (b - 1) + slot) * ldp + col]);
#pragma unroll 8
    for (int64_t c = b; c <= lo; ++c) acc = add_rn(acc, pieces[(2 * c) * ldp + col]);
    out[(int64_t)r * ldo + col] = acc;
}

template <typename T, typename I, int VEC, int G, int U>
static void launch_mode(const OtherModes<I> &om, int n_other, const I *rowc, const T *vals, int64_t nnz, int64_t rows,
                        int64_t R, T *out, int64_t ldo, T *pieces, int64_t ldp, cudaStream_t s) {
    constexpr int chunks_per_block = 8 * (32 / G);
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    dim3 grid((unsigned)((nchunks + chunks_per_block - 1) / chunks_per_block),
              (unsigned)((R + (int64_t)G * VEC - 1) / ((int64_t)G * VEC)));
    mttkrp_mode_kernel<T, I, VEC, G, U><<<grid, 256, 0, s>>>(om, n_other, rowc, vals, nnz, rows, R, out, ldo, pieces,
                                                            ldp);
}

// group width from the column packs per row, as K1's dispatch_g: a narrow R puts several chunks in one warp
template <typename T, typename I, int VEC>
static void dispatch_mode(const OtherModes<I> &om, int n_other, const I *rowc, const T *vals, int64_t nnz,
                          int64_t rows, int64_t R, T *out, int64_t ldo, T *pieces, int64_t ldp, cudaStream_t s) {
    const int64_t packs = (R + VEC - 1) / VEC;
#define B2S_MM(G, U) return launch_mode<T, I, VEC, G, U>(om, n_other, rowc, vals, nnz, rows, R, out, ldo, pieces, ldp, s)
    if (packs > 16) B2S_MM(32, 8);
    if (packs > 8) B2S_MM(16, 8);
    if (packs > 4) B2S_MM(8, 8);
    if (packs > 2) B2S_MM(4, 4);
    if (packs > 1) B2S_MM(2, 2);
    B2S_MM(1, 1);
#undef B2S_MM
}

template <typename T, typename I>
static int mttkrp_mode_impl(int order, int mode, int64_t nnz, int64_t rows, int64_t R, const void *const *coords,
                            const void *vals, const void *const *factors, const int64_t *ld, void *out, int64_t ldo,
                            cudaStream_t s) {
    constexpr int VEC = 16 / sizeof(T);
    OtherModes<I> om{};
    int n_other = 0;
    bool aligned = R % VEC == 0 && ldo % VEC == 0 && ((uintptr_t)out & 15) == 0;
    for (int m = 0; m < order; ++m) {
        if (m == mode) continue;
        om.coord[n_other] = (const I *)coords[m];
        om.fac[n_other] = factors[m];
        om.ld[n_other] = ld[m];
        aligned = aligned && ((uintptr_t)factors[m] & 15) == 0 && ld[m] % VEC == 0;
        ++n_other;
    }
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    const int64_t ldp = (R + 3) & ~(int64_t)3;  // 16-byte aligned piece rows for both dtypes
    T *pieces = nullptr;
    int rc = scratch_alloc((void **)&pieces, (size_t)(2 * nchunks * ldp) * sizeof(T), s);
    if (rc) return rc;
    const I *rowc = (const I *)coords[mode];
    if (aligned) dispatch_mode<T, I, VEC>(om, n_other, rowc, (const T *)vals, nnz, rows, R, (T *)out, ldo, pieces, ldp, s);
    else dispatch_mode<T, I, 1>(om, n_other, rowc, (const T *)vals, nnz, rows, R, (T *)out, ldo, pieces, ldp, s);
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e == cudaSuccess && nchunks > 1) {
        const int64_t warps = nchunks - 1;
        dim3 grid((unsigned)((warps + 7) / 8), (unsigned)((R + 31) / 32));
        mttkrp_combine_kernel<T, I><<<grid, 256, 0, s>>>(rowc, nnz, R, pieces, ldp, (T *)out, ldo);
        e = cudaGetLastError();
        count_launch();
    }
    rc = scratch_free(pieces, s);  // stream-ordered: released after the kernels that use it
    B2S_REQUIRE(e == cudaSuccess, B2S_ERR_CUDA, "mttkrp_mode: kernel launch failed: %s", cudaGetErrorString(e));
    return rc;
}

// ---------------------------------------------------------------------------------------------------------------------
// K12: mode-n TTMc (tensor times matrix chain), the Kronecker counterpart of K10.
//
//   out[i, col] = sum over stored e with i_n(e) = i of  v_e * U_a[i_a, r_a] * U_b[i_b, r_b] * ... * U_z[i_z, r_z]
//   col = ((r_a * R_b + r_b) * R_c + r_c) ... (C order over the other modes a < b < ... < z)
//
// Same stream, chunks, flush and combine as K10; only the columns differ.  The W = R_a * ... * R_z columns of a row
// are cut into tiles of G * VEC; lane l of a group owns VEC consecutive columns, which (VEC dividing R_z) share the
// digits r_a .. r_y.  Per entry the lane gathers the scalars U_a[i_a, r_a] .. U_y[i_y, r_y] (the group reads the same
// factor rows), forms the prefix ((v * U_a) * ...) * U_y once, and multiplies it by one pack of U_z's row: the
// association of the order contract, so the vector and scalar forms are bit-identical.  The grid is flat with the column
// tiles of one chunk range adjacent, so the tiles that re-read a chunk's stream entries run together and mostly find
// them in L2.
// ---------------------------------------------------------------------------------------------------------------------

// ranks of the leading other modes (every other mode but the last), ascending
struct TtmcRanks {
    int r[kMaxOther];
};

template <typename T>
__device__ __forceinline__ T t_stream(const T *p, bool reread) {
    return reread ? __ldg(p) : ldg_stream(p);  // several column tiles read the stream: keep it in L2 for the others
}

template <typename T, typename I, int VEC, int G, int U>
__global__ void __launch_bounds__(256)
ttmc_mode_kernel(const OtherModes<I> lead, const TtmcRanks rk, const int n_lead, const I *__restrict__ lastc,
                 const T *__restrict__ fac_last, const int64_t ld_last, const int64_t R_last,
                 const I *__restrict__ rowc, const T *__restrict__ vals, const int64_t nnz, const int64_t rows,
                 const int64_t W, const int64_t ntiles, T *__restrict__ out, const int64_t ldo, T *__restrict__ pieces,
                 const int64_t ldp) {
    static_assert(G >= 1 && G <= 32 && (G & (G - 1)) == 0, "G must be a power of two <= 32");
    static_assert(U <= G && G % U == 0, "U must divide G");
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int sub = lane & (G - 1);
    const int64_t tile = (int64_t)blockIdx.x % ntiles;
    const int64_t cblock = (int64_t)blockIdx.x / ntiles;
    const int64_t chunk = (cblock * (blockDim.x >> 5) + (threadIdx.x >> 5)) * (32 / G) + lane / G;
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    const int64_t col0 = (tile * G + sub) * VEC;
    const bool col_ok = col0 < W;
    const bool reread = ntiles > 1;

    // this lane's digits: r_z0 .. r_z0 + VEC - 1 of the last mode, one digit of each leading mode
    int64_t q = col_ok ? col0 / R_last : 0;
    const int64_t rz0 = col_ok ? col0 - q * R_last : 0;
    int dig[kMaxOther];
#pragma unroll
    for (int m = kMaxOther - 1; m >= 0; --m) {
        dig[m] = 0;
        if (m < n_lead) {
            const int64_t qn = q / rk.r[m];
            dig[m] = (int)(q - qn * rk.r[m]);
            q = qn;
        }
    }

    int64_t base = 0, end = 0, row_first = 0, row_last = 0;
    bool head_cross = false, tail_cross = false;
    if (chunk < nchunks) {
        base = chunk * kChunk;
        end = base + kChunk < nnz ? base + kChunk : nnz;
        row_first = (int64_t)rowc[base];
        row_last = (int64_t)rowc[end - 1];
        const int64_t prev = chunk > 0 ? (int64_t)rowc[base - 1] : -1;
        head_cross = prev == row_first;
        tail_cross = end < nnz && (int64_t)rowc[end] == row_last;
        if (col_ok) {
            m_zero_rows<T, VEC>(out, ldo, prev + 1, row_first, col0);
            if (end == nnz) m_zero_rows<T, VEC>(out, ldo, row_last + 1, rows, col0);
        }
    }
    const uint64_t pol = policy_evict_last();

    T acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = T(0);
    int64_t cur = row_first;

    auto flush = [&](int64_t r) {
        if (!col_ok) return;
        T *dst;
        if (r == row_first && (head_cross || (r == row_last && tail_cross))) dst = pieces + (2 * chunk) * ldp + col0;
        else if (r == row_last && tail_cross) dst = pieces + (2 * chunk + 1) * ldp + col0;
        else dst = out + r * ldo + col0;
        m_store<T, VEC>(dst, acc);
    };

    auto any = [&](bool p) -> bool {
        if constexpr (G == 32) return p;
        else return __any_sync(FULL, p);
    };

    I rc_n = 0, cz_n = 0;
    I c_n[kMaxOther];
    T v_n = T(0);
#pragma unroll
    for (int m = 0; m < kMaxOther; ++m) c_n[m] = 0;
    if (base + sub < end) {
        rc_n = t_stream(rowc + base + sub, reread);
        v_n = t_stream(vals + base + sub, reread);
        cz_n = t_stream(lastc + base + sub, reread);
#pragma unroll
        for (int m = 0; m < kMaxOther; ++m)
            if (m < n_lead) c_n[m] = t_stream(lead.coord[m] + base + sub, reread);
    }

    const T *fz = fac_last + rz0;
    while (any(base < end)) {
        const I rc = rc_n, cz = cz_n;
        const T v = v_n;
        I c[kMaxOther];
#pragma unroll
        for (int m = 0; m < kMaxOther; ++m) c[m] = c_n[m];
        const int64_t rem = end - base;
        const int cnt = rem > G ? G : (rem > 0 ? (int)rem : 0);
        const int64_t nb = base + G;
        if (nb + sub < end) {
            rc_n = t_stream(rowc + nb + sub, reread);
            v_n = t_stream(vals + nb + sub, reread);
            cz_n = t_stream(lastc + nb + sub, reread);
#pragma unroll
            for (int m = 0; m < kMaxOther; ++m)
                if (m < n_lead) c_n[m] = t_stream(lead.coord[m] + nb + sub, reread);
        }
#pragma unroll 1
        for (int j = 0; j < G; j += U) {
            if (!any(j < cnt)) break;
            T pre[U];
            I rr[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                pre[u] = __shfl_sync(FULL, v, j + u, G);
                rr[u] = __shfl_sync(FULL, rc, j + u, G);
            }
            // the prefix ((v * U_a) * U_b) * ... over the leading modes, each product rounded
#pragma unroll
            for (int m = 0; m < kMaxOther; ++m) {
                if (m < n_lead) {
                    const T *fm = (const T *)lead.fac[m] + dig[m];
                    const int64_t ldm = lead.ld[m];
                    T f[U];
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const I ix = __shfl_sync(FULL, c[m], j + u, G);
                        f[u] = j + u < cnt && col_ok ? m_load<T, 1>(fm + (int64_t)ix * ldm, pol).v[0] : T(0);
                    }
#pragma unroll
                    for (int u = 0; u < U; ++u) pre[u] = mul_rn(pre[u], f[u]);
                }
            }
            MPack<T, VEC> f[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const I ix = __shfl_sync(FULL, cz, j + u, G);
                if (j + u < cnt && col_ok) f[u] = m_load<T, VEC>(fz + (int64_t)ix * ld_last, pol);
                else {
#pragma unroll
                    for (int k = 0; k < VEC; ++k) f[u].v[k] = T(0);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (j + u < cnt) {
                    if (rr[u] != cur) {
                        flush(cur);
                        if (col_ok) m_zero_rows<T, VEC>(out, ldo, cur + 1, rr[u], col0);
                        cur = rr[u];
#pragma unroll
                        for (int k = 0; k < VEC; ++k) acc[k] = T(0);
                    }
#pragma unroll
                    for (int k = 0; k < VEC; ++k) acc[k] = add_rn(acc[k], mul_rn(pre[u], f[u].v[k]));
                }
            }
        }
        base = nb;
    }
    if (chunk < nchunks) flush(cur);
}

template <typename T, typename I, int VEC, int G, int U>
static int launch_ttmc(const OtherModes<I> &lead, const TtmcRanks &rk, int n_lead, const I *lastc, const T *fac_last,
                       int64_t ld_last, int64_t R_last, const I *rowc, const T *vals, int64_t nnz, int64_t rows,
                       int64_t W, T *out, int64_t ldo, T *pieces, int64_t ldp, cudaStream_t s) {
    constexpr int chunks_per_block = 8 * (32 / G);
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    const int64_t ntiles = (W + (int64_t)G * VEC - 1) / ((int64_t)G * VEC);
    const int64_t blocks = (nchunks + chunks_per_block - 1) / chunks_per_block * ntiles;
    B2S_REQUIRE(blocks <= INT32_MAX, B2S_ERR_INVALID, "ttmc_mode: %lld chunks x %lld column tiles exceed one grid",
                (long long)nchunks, (long long)ntiles);
    ttmc_mode_kernel<T, I, VEC, G, U><<<(unsigned)blocks, 256, 0, s>>>(lead, rk, n_lead, lastc, fac_last, ld_last,
                                                                       R_last, rowc, vals, nnz, rows, W, ntiles, out,
                                                                       ldo, pieces, ldp);
    return B2S_OK;
}

template <typename T, typename I, int VEC>
static int dispatch_ttmc(const OtherModes<I> &lead, const TtmcRanks &rk, int n_lead, const I *lastc,
                         const T *fac_last, int64_t ld_last, int64_t R_last, const I *rowc, const T *vals, int64_t nnz,
                         int64_t rows, int64_t W, T *out, int64_t ldo, T *pieces, int64_t ldp, cudaStream_t s) {
    const int64_t packs = (W + VEC - 1) / VEC;
#define B2S_TT(G, U)                                                                                                 \
    return launch_ttmc<T, I, VEC, G, U>(lead, rk, n_lead, lastc, fac_last, ld_last, R_last, rowc, vals, nnz, rows, W, \
                                        out, ldo, pieces, ldp, s)
    // at most 16 lanes per group (two chunks per warp, 16 entries' gathers in flight): against 32 lanes, W = 256 and
    // 1024 in f32 ran 20 % faster on the H100, more than paying for twice the column tiles
    if (packs > 8) B2S_TT(16, 8);
    if (packs > 4) B2S_TT(8, 8);
    if (packs > 2) B2S_TT(4, 4);
    if (packs > 1) B2S_TT(2, 2);
    B2S_TT(1, 1);
#undef B2S_TT
}

template <typename T, typename I>
static int ttmc_mode_impl(int order, int mode, int64_t nnz, int64_t rows, const int64_t *ranks, int64_t W,
                          const void *const *coords, const void *vals, const void *const *factors, const int64_t *ld,
                          void *out, int64_t ldo, cudaStream_t s) {
    constexpr int VEC = 16 / sizeof(T);
    const int last = mode == order - 1 ? order - 2 : order - 1;
    OtherModes<I> lead{};
    TtmcRanks rk{};
    int n_lead = 0;
    for (int m = 0; m < last; ++m) {
        if (m == mode) continue;
        lead.coord[n_lead] = (const I *)coords[m];
        lead.fac[n_lead] = factors[m];
        lead.ld[n_lead] = ld[m];
        rk.r[n_lead] = (int)ranks[m];
        ++n_lead;
    }
    const int64_t R_last = ranks[last];
    const bool aligned = R_last % VEC == 0 && ld[last] % VEC == 0 && ((uintptr_t)factors[last] & 15) == 0 &&
                         ldo % VEC == 0 && ((uintptr_t)out & 15) == 0;
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    const int64_t ldp = (W + 3) & ~(int64_t)3;
    T *pieces = nullptr;
    int rc = scratch_alloc((void **)&pieces, (size_t)(2 * nchunks * ldp) * sizeof(T), s);
    if (rc) return rc;
    const I *rowc = (const I *)coords[mode];
    const I *lastc = (const I *)coords[last];
    const T *fl = (const T *)factors[last];
    if (aligned)
        rc = dispatch_ttmc<T, I, VEC>(lead, rk, n_lead, lastc, fl, ld[last], R_last, rowc, (const T *)vals, nnz, rows,
                                      W, (T *)out, ldo, pieces, ldp, s);
    else
        rc = dispatch_ttmc<T, I, 1>(lead, rk, n_lead, lastc, fl, ld[last], R_last, rowc, (const T *)vals, nnz, rows, W,
                                    (T *)out, ldo, pieces, ldp, s);
    cudaError_t e = cudaGetLastError();
    if (rc == B2S_OK) count_launch();
    if (rc == B2S_OK && e == cudaSuccess && nchunks > 1) {
        const int64_t warps = nchunks - 1;
        dim3 grid((unsigned)((warps + 7) / 8), (unsigned)((W + 31) / 32));
        mttkrp_combine_kernel<T, I><<<grid, 256, 0, s>>>(rowc, nnz, W, pieces, ldp, (T *)out, ldo);
        e = cudaGetLastError();
        count_launch();
    }
    const int frc = scratch_free(pieces, s);
    if (rc) return rc;
    B2S_REQUIRE(e == cudaSuccess, B2S_ERR_CUDA, "ttmc_mode: kernel launch failed: %s", cudaGetErrorString(e));
    return frc;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_mttkrp_mode_chunk(void) { return B2S_MTTKRP_CHUNK; }

int b2s_mttkrp_mode(int dtype, int idx_bytes, int order, int mode, int64_t nnz, int64_t rows, int64_t R,
                    const void *const *coords_host, const void *vals_dev, const void *const *factors_host,
                    const int64_t *ld_host, void *out_dev, int64_t ldo, void *stream) {
    B2S_REQUIRE(dtype == B2S_F32 || dtype == B2S_F64, B2S_ERR_UNSUPPORTED, "mttkrp_mode: dtype %d (f32/f64 only)",
                dtype);
    B2S_REQUIRE(idx_bytes == 4 || idx_bytes == 8, B2S_ERR_INVALID, "mttkrp_mode: idx_bytes");
    B2S_REQUIRE(order >= 2 && order <= 8, B2S_ERR_INVALID, "mttkrp_mode: order %d outside 2..8", order);
    B2S_REQUIRE(mode >= 0 && mode < order, B2S_ERR_INVALID, "mttkrp_mode: mode %d of an order-%d tensor", mode, order);
    B2S_REQUIRE(nnz >= 0 && rows >= 0 && R >= 0, B2S_ERR_INVALID, "mttkrp_mode: negative size");
    B2S_REQUIRE(ldo >= R, B2S_ERR_INVALID, "mttkrp_mode: ldo < R");
    if (rows == 0 || R == 0) return B2S_OK;
    B2S_REQUIRE(coords_host != nullptr && factors_host != nullptr && ld_host != nullptr, B2S_ERR_INVALID,
                "mttkrp_mode: NULL pointer array");
    for (int m = 0; m < order; ++m)
        B2S_REQUIRE(m == mode || ld_host[m] >= R, B2S_ERR_INVALID, "mttkrp_mode: ld of factor %d < R", m);
    cudaStream_t s = (cudaStream_t)stream;
    const size_t es = dtype_size(dtype);
    if (nnz == 0) {
        B2S_CUDA(cudaMemset2DAsync(out_dev, (size_t)ldo * es, 0, (size_t)R * es, (size_t)rows, s));
        return B2S_OK;
    }
#define B2S_MI(T, I) \
    return mttkrp_mode_impl<T, I>(order, mode, nnz, rows, R, coords_host, vals_dev, factors_host, ld_host, out_dev, ldo, s)
    if (dtype == B2S_F32) {
        if (idx_bytes == 4) B2S_MI(float, int32_t);
        B2S_MI(float, int64_t);
    }
    if (idx_bytes == 4) B2S_MI(double, int32_t);
    B2S_MI(double, int64_t);
#undef B2S_MI
}

int b2s_ttmc_mode_max_width(void) { return B2S_TTMC_MAX_W; }

int b2s_ttmc_mode(int dtype, int idx_bytes, int order, int mode, int64_t nnz, int64_t rows, const int64_t *ranks_host,
                  const void *const *coords_host, const void *vals_dev, const void *const *factors_host,
                  const int64_t *ld_host, void *out_dev, int64_t ldo, void *stream) {
    B2S_REQUIRE(dtype == B2S_F32 || dtype == B2S_F64, B2S_ERR_UNSUPPORTED, "ttmc_mode: dtype %d (f32/f64 only)", dtype);
    B2S_REQUIRE(idx_bytes == 4 || idx_bytes == 8, B2S_ERR_INVALID, "ttmc_mode: idx_bytes");
    B2S_REQUIRE(order >= 2 && order <= 8, B2S_ERR_INVALID, "ttmc_mode: order %d outside 2..8", order);
    B2S_REQUIRE(mode >= 0 && mode < order, B2S_ERR_INVALID, "ttmc_mode: mode %d of an order-%d tensor", mode, order);
    B2S_REQUIRE(nnz >= 0 && rows >= 0, B2S_ERR_INVALID, "ttmc_mode: negative size");
    B2S_REQUIRE(ranks_host != nullptr, B2S_ERR_INVALID, "ttmc_mode: NULL ranks");
    int64_t W = 1;
    for (int m = 0; m < order; ++m) {
        if (m == mode) continue;
        B2S_REQUIRE(ranks_host[m] >= 0, B2S_ERR_INVALID, "ttmc_mode: negative rank of mode %d", m);
        if (ranks_host[m] == 0) W = 0;
        else if (W > 0) W = W > B2S_TTMC_MAX_W / ranks_host[m] ? B2S_TTMC_MAX_W + 1 : W * ranks_host[m];
    }
    B2S_REQUIRE(W <= B2S_TTMC_MAX_W, B2S_ERR_INVALID, "ttmc_mode: width above B2S_TTMC_MAX_W = %d", B2S_TTMC_MAX_W);
    B2S_REQUIRE(ldo >= W, B2S_ERR_INVALID, "ttmc_mode: ldo < W");
    if (rows == 0 || W == 0) return B2S_OK;
    B2S_REQUIRE(coords_host != nullptr && factors_host != nullptr && ld_host != nullptr, B2S_ERR_INVALID,
                "ttmc_mode: NULL pointer array");
    for (int m = 0; m < order; ++m)
        B2S_REQUIRE(m == mode || ld_host[m] >= ranks_host[m], B2S_ERR_INVALID, "ttmc_mode: ld of factor %d < R_%d", m,
                    m);
    cudaStream_t s = (cudaStream_t)stream;
    const size_t es = dtype_size(dtype);
    if (nnz == 0) {
        B2S_CUDA(cudaMemset2DAsync(out_dev, (size_t)ldo * es, 0, (size_t)W * es, (size_t)rows, s));
        return B2S_OK;
    }
#define B2S_TI(T, I)                                                                                                \
    return ttmc_mode_impl<T, I>(order, mode, nnz, rows, ranks_host, W, coords_host, vals_dev, factors_host, ld_host, \
                                out_dev, ldo, s)
    if (dtype == B2S_F32) {
        if (idx_bytes == 4) B2S_TI(float, int32_t);
        B2S_TI(float, int64_t);
    }
    if (idx_bytes == 4) B2S_TI(double, int32_t);
    B2S_TI(double, int64_t);
#undef B2S_TI
}

}  // extern "C"
