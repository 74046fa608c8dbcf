// tensor_modes.cuh -- what the sparse-tensor kernels K10 / K12 (mttkrp.cu), K13 (tttp.cu), K15 (cp_completion.cu) and
// K16 (cp_apr.cu) share: the per-mode pointer arrays, the factor-row pack and its load, the argument checks and dtype x
// index-width dispatch of their C entry points, and the mode-stream chunk scheme of K10, K12, K15 and K16 with K10's
// combine kernel (one definition, so that K15's b_i and K16's sums stay mttkrp_mode's rows bit for bit).
#pragma once
#include "common.cuh"

namespace b2s {

__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }

constexpr int64_t kChunk = B2S_MTTKRP_CHUNK;
constexpr int kMaxOther = 7;  // order <= 8

// coordinate array, factor and factor row stride of up to N modes, passed to a kernel by value
template <typename I, int N>
struct ModeArrays {
    const I *coord[N];
    const void *fac[N];
    int64_t ld[N];
};

// the gathered other modes of a mode-stream kernel, in ascending mode order
template <typename I>
using OtherModes = ModeArrays<I, kMaxOther>;

// Chunk `chunk` of a mode stream (empty for ChunkSpan(c)): its entries base .. end - 1, the row before it (-1 for chunk
// 0), its first and last row, and whether they continue into the previous / next chunk.
struct ChunkSpan {
    int64_t base = 0, end = 0, row_first = 0, row_last = 0, prev = -1, chunk;
    bool head_cross = false, tail_cross = false;

    __device__ __forceinline__ explicit ChunkSpan(const int64_t c) : chunk(c) {}
    template <typename I>
    __device__ __forceinline__ ChunkSpan(const I *rowc, const int64_t nnz, const int64_t c) : chunk(c) {
        base = c * kChunk;
        end = base + kChunk < nnz ? base + kChunk : nnz;
        row_first = (int64_t)rowc[base];
        row_last = (int64_t)rowc[end - 1];
        if (c > 0) {
            prev = (int64_t)rowc[base - 1];
            head_cross = prev == row_first;
        }
        tail_cross = end < nnz && (int64_t)rowc[end] == row_last;
    }

    // where row r's sums go: piece row 2 chunk (the first row, crossing either boundary) or 2 chunk + 1 (the last row,
    // continuing into the next chunk) of `pieces`, else row r of `out`, as it is complete in this chunk
    template <typename T>
    __device__ __forceinline__ T *dest(T *pieces, const int64_t ldp, const int64_t r, T *out, const int64_t ldo) const {
        if (r == row_first && (head_cross || (r == row_last && tail_cross))) return pieces + (2 * chunk) * ldp;
        if (r == row_last && tail_cross) return pieces + (2 * chunk + 1) * ldp;
        return out + r * ldo;
    }
};

// False when no row crosses chunk boundary b >= 1, or when it crosses b-1 too (b-1 owns it).  Else b owns `row`, which
// adds piece row `first` (chunk b-1's), then the head pieces 2c of chunks c = b .. `last` (found by bisection).
template <typename I>
__device__ __forceinline__ bool crossing_row(const I *__restrict__ rowc, const int64_t nnz, const int64_t b,
                                             int64_t &row, int64_t &first, int64_t &last) {
    const int64_t p = b * kChunk;
    const I r = rowc[p];
    if (rowc[p - 1] != r) return false;                    // no row crosses b
    if (b > 1 && rowc[p - kChunk - 1] == r) return false;  // the row crosses b-1 too: that boundary owns it
    int64_t hi = (nnz + kChunk - 1) / kChunk - 1;
    for (last = b; last < hi;) {
        const int64_t mid = (last + hi + 1) >> 1;
        if (rowc[mid * kChunk] == r) last = mid;
        else hi = mid - 1;
    }
    row = (int64_t)r;
    first = 2 * (b - 1) + (rowc[p - kChunk] == r ? 0 : 1);
    return true;
}

// K10's combine, also K16's (the sums of both are b2s_mttkrp_mode's steps 4-5): one warp per chunk boundary b, one
// column per lane; the row that b owns (crossing_row) adds its pieces into `out`
template <typename T, typename I>
__global__ void __launch_bounds__(256)
mttkrp_combine_kernel(const I *__restrict__ rowc, const int64_t nnz, const int64_t R, const T *__restrict__ pieces,
                      const int64_t ldp, T *__restrict__ out, const int64_t ldo) {
    const int64_t b = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) + 1;
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    const int64_t col = (int64_t)blockIdx.y * 32 + (threadIdx.x & 31);
    if (b >= nchunks || col >= R) return;
    int64_t row, first, last;
    if (!crossing_row(rowc, nnz, b, row, first, last)) return;
    T acc = T(0);
    acc = add_rn(acc, pieces[first * ldp + col]);
#pragma unroll 8
    for (int64_t c = b; c <= last; ++c) acc = add_rn(acc, pieces[(2 * c) * ldp + col]);
    out[row * ldo + col] = acc;
}

// the combine launch of R columns over the nchunks - 1 chunk boundaries: a warp per boundary
template <typename T, typename I>
int launch_mttkrp_combine(const I *rowc, const int64_t nnz, const int64_t R, const T *pieces, const int64_t ldp,
                          const int64_t nchunks, T *out, const int64_t ldo, cudaStream_t s) {
    dim3 grid((unsigned)((nchunks - 1 + 7) / 8), (unsigned)((R + 31) / 32));
    mttkrp_combine_kernel<T, I><<<grid, 256, 0, s>>>(rowc, nnz, R, pieces, ldp, out, ldo);
    return B2S_OK;
}

// 2 piece rows per chunk, `width` rounded up to 4 (16-byte aligned rows), main(pieces, ldp), combine(pieces, ldp,
// nchunks) when there is more than one chunk, then the stream-ordered free; each callable launches one kernel
template <typename T, typename Main, typename Combine>
int chunked_launches(const char *op, const int64_t nnz, const int64_t width, cudaStream_t s, Main &&main,
                     Combine &&combine) {
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    const int64_t ldp = (width + 3) & ~(int64_t)3;
    T *pieces = nullptr;
    int rc = scratch_alloc((void **)&pieces, (size_t)(2 * nchunks * ldp) * sizeof(T), s);
    if (rc) return rc;
    rc = main(pieces, ldp);
    cudaError_t e = cudaGetLastError();
    if (rc == B2S_OK) count_launch();
    if (rc == B2S_OK && e == cudaSuccess && nchunks > 1) {
        rc = combine(pieces, ldp, nchunks);
        e = cudaGetLastError();
        if (rc == B2S_OK) count_launch();
    }
    const int frc = scratch_free(pieces, s);  // stream-ordered: released after the kernels that use it
    if (rc) return rc;
    B2S_REQUIRE(e == cudaSuccess, B2S_ERR_CUDA, "%s: kernel launch failed: %s", op, cudaGetErrorString(e));
    return frc;
}

template <typename T, int VEC>
struct alignas(sizeof(T) * VEC) MPack {
    T v[VEC];
};

// one 16-byte pack or one scalar of a factor row, under the L2 policy `pol`
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

// dtype, index width and order, named after the entry point `op`
inline int check_tensor(const char *op, int dtype, int idx_bytes, int order) {
    B2S_REQUIRE(dtype == B2S_F32 || dtype == B2S_F64, B2S_ERR_UNSUPPORTED, "%s: dtype %d (f32/f64 only)", op, dtype);
    B2S_REQUIRE(idx_bytes == 4 || idx_bytes == 8, B2S_ERR_INVALID, "%s: idx_bytes", op);
    B2S_REQUIRE(order >= 2 && order <= 8, B2S_ERR_INVALID, "%s: order %d outside 2..8", op, order);
    return B2S_OK;
}

// the host pointer arrays, and the row stride of every factor but `skip` (-1: none) against its rank: ranks[m], or R
// for every factor when `ranks` is NULL
inline int check_factors(const char *op, int order, int skip, const void *const *coords, const void *const *factors,
                         const int64_t *ld, int64_t R, const int64_t *ranks) {
    B2S_REQUIRE(coords != nullptr && factors != nullptr && ld != nullptr, B2S_ERR_INVALID, "%s: NULL pointer array",
                op);
    for (int m = 0; m < order; ++m)
        B2S_REQUIRE(m == skip || ld[m] >= (ranks ? ranks[m] : R), B2S_ERR_INVALID, "%s: ld of factor %d < its rank",
                    op, m);
    return B2S_OK;
}

// f(T{}, I{}) for the value type of `dtype` (f32 / f64) and the index type of `idx_bytes` (4 / 8)
template <typename F>
int dispatch_tensor(int dtype, int idx_bytes, F &&f) {
    if (dtype == B2S_F32) return idx_bytes == 4 ? f(float{}, int32_t{}) : f(float{}, int64_t{});
    return idx_bytes == 4 ? f(double{}, int32_t{}) : f(double{}, int64_t{});
}

}  // namespace b2s
