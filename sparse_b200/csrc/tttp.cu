// tttp.cu -- K13: a sparse tensor of order 2..8 times a CP (Kruskal) model at its stored entries (TTTP, the order-N
// SDDMM).
//
//   z_e = v_e * sum_r  U_0[i_0(e), r] * U_1[i_1(e), r] * ... * U_{N-1}[i_{N-1}(e), r]
//
// Each warp owns a block of 32 consecutive entries and walks the R columns in r-tiles of RT = 8 * VEC.  Per r-tile the
// warp takes its entries four at a time: a group of 8 lanes gathers one entry's RT-column segment of every factor row
// (16-byte packs, L2 evict_last: the factors are the reused operand), so each gather is one contiguous segment of a
// row, and multiplies the packs together in ascending mode order.  The products of the 32 entries go to shared memory
// (one padded row per entry), and then each lane adds its own entry's RT products in ascending r onto a running sum it
// carries across r-tiles.  The products q_r are independent; only that sum is serial, so the result is the order of
// include/sparse_b200.h whatever the grid, and the vector (VEC = 16 B / itemsize) and scalar (VEC = 1) forms are
// bit-identical.  No atomics, no scratch memory.
#include "tensor_modes.cuh"

namespace b2s {

constexpr int kMaxOrder = 8;
constexpr int kLanesPerEntry = 8;                    // lanes that gather one entry's r-tile
constexpr int kEntriesPerStep = 32 / kLanesPerEntry;  // entries a warp gathers at once
constexpr int kSteps = 32 / kEntriesPerStep;          // gather steps per block of 32 entries
constexpr int kWarps = 8;                            // warps per CTA

template <typename I>
using TttpModes = ModeArrays<I, kMaxOrder>;

template <typename T, typename I, int VEC>
__global__ void __launch_bounds__(kWarps * 32)
tttp_kernel(const TttpModes<I> md, const int order, const T *__restrict__ vals, const int64_t nnz, const int64_t R,
            T *__restrict__ out) {
    constexpr int RT = kLanesPerEntry * VEC;  // columns per r-tile
    constexpr int LDS = RT + 1;               // padded shared row: conflict-free column reads across the warp
    constexpr unsigned FULL = 0xffffffffu;
    __shared__ T prod[kWarps][32 * LDS];

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int grp = lane / kLanesPerEntry;  // which of the step's entries this lane gathers for
    const int sub = lane % kLanesPerEntry;  // which pack of the r-tile
    const int64_t base = ((int64_t)blockIdx.x * kWarps + warp) * 32;
    if (base >= nnz) return;  // warp-uniform
    const int cnt = nnz - base < 32 ? (int)(nnz - base) : 32;
    const bool own = lane < cnt;

    I c[kMaxOrder];
#pragma unroll
    for (int m = 0; m < kMaxOrder; ++m) c[m] = (m < order && own) ? ldg_stream(md.coord[m] + base + lane) : I(0);
    const T v = own ? ldg_stream(vals + base + lane) : T(0);
    const uint64_t pol = policy_evict_last();
    T *sm = prod[warp];

    T acc = T(0);  // m = ((+0 + q_0) + q_1) + ..., carried across r-tiles
    for (int64_t r0 = 0; r0 < R; r0 += RT) {
        const int64_t col = r0 + (int64_t)sub * VEC;
        const bool col_ok = col < R;  // VEC divides R on the vector path: a pack is all in or all out
        MPack<T, VEC> p[kSteps];
        // q = ((U_0 * U_1) * U_2) * ... over the modes in ascending order, each product rounded
#pragma unroll
        for (int m = 0; m < kMaxOrder; ++m) {
            if (m < order) {
                const T *fm = (const T *)md.fac[m] + col;
                const int64_t ldm = md.ld[m];
                MPack<T, VEC> f[kSteps];
#pragma unroll
                for (int s = 0; s < kSteps; ++s) {
                    const int e = s * kEntriesPerStep + grp;
                    const I ix = __shfl_sync(FULL, c[m], e);
                    if (e < cnt && col_ok) f[s] = m_load<T, VEC>(fm + (int64_t)ix * ldm, pol);
                    else {
#pragma unroll
                        for (int k = 0; k < VEC; ++k) f[s].v[k] = T(0);
                    }
                }
#pragma unroll
                for (int s = 0; s < kSteps; ++s)
#pragma unroll
                    for (int k = 0; k < VEC; ++k) p[s].v[k] = m == 0 ? f[s].v[k] : mul_rn(p[s].v[k], f[s].v[k]);
            }
        }
#pragma unroll
        for (int s = 0; s < kSteps; ++s) {
            const int e = s * kEntriesPerStep + grp;
#pragma unroll
            for (int k = 0; k < VEC; ++k) sm[e * LDS + sub * VEC + k] = p[s].v[k];
        }
        __syncwarp();
        const int64_t left = R - r0;
        const int n = left < RT ? (int)left : RT;
        if (n == RT) {
#pragma unroll
            for (int k = 0; k < RT; ++k) acc = add_rn(acc, sm[lane * LDS + k]);
        } else {
            for (int k = 0; k < n; ++k) acc = add_rn(acc, sm[lane * LDS + k]);
        }
        __syncwarp();  // the next r-tile overwrites the products
    }
    if (own) out[base + lane] = mul_rn(v, acc);
}

template <typename T, typename I, int VEC>
static void launch_tttp(const TttpModes<I> &md, int order, const T *vals, int64_t nnz, int64_t R, T *out,
                        cudaStream_t s) {
    const int64_t per_block = kWarps * 32;
    const unsigned blocks = (unsigned)((nnz + per_block - 1) / per_block);
    tttp_kernel<T, I, VEC><<<blocks, kWarps * 32, 0, s>>>(md, order, vals, nnz, R, out);
}

template <typename T, typename I>
static int tttp_impl(int order, int64_t nnz, int64_t R, const void *const *coords, const void *vals,
                     const void *const *factors, const int64_t *ld, void *out, cudaStream_t s) {
    constexpr int VEC = 16 / sizeof(T);
    TttpModes<I> md{};
    bool aligned = R % VEC == 0;
    for (int m = 0; m < order; ++m) {
        md.coord[m] = (const I *)coords[m];
        md.fac[m] = factors[m];
        md.ld[m] = ld[m];
        aligned = aligned && ((uintptr_t)factors[m] & 15) == 0 && ld[m] % VEC == 0;
    }
    if (aligned) launch_tttp<T, I, VEC>(md, order, (const T *)vals, nnz, R, (T *)out, s);
    else launch_tttp<T, I, 1>(md, order, (const T *)vals, nnz, R, (T *)out, s);
    const cudaError_t e = cudaGetLastError();
    count_launch();
    B2S_REQUIRE(e == cudaSuccess, B2S_ERR_CUDA, "tttp: kernel launch failed: %s", cudaGetErrorString(e));
    return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_tttp(int dtype, int idx_bytes, int order, int64_t nnz, int64_t R, const void *const *coords_host,
             const void *vals_dev, const void *const *factors_host, const int64_t *ld_host, void *out_vals_dev,
             void *stream) {
    const char *op = "tttp";
    int rc = check_tensor(op, dtype, idx_bytes, order);
    if (rc) return rc;
    B2S_REQUIRE(nnz >= 0 && R >= 0, B2S_ERR_INVALID, "%s: negative size", op);
    B2S_REQUIRE(nnz / 256 < INT32_MAX, B2S_ERR_INVALID, "%s: nnz %lld exceeds one grid", op, (long long)nnz);
    if (nnz == 0) return B2S_OK;
    rc = check_factors(op, order, -1, coords_host, factors_host, ld_host, R, nullptr);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    return dispatch_tensor(dtype, idx_bytes, [&](auto t, auto i) {
        return tttp_impl<decltype(t), decltype(i)>(order, nnz, R, coords_host, vals_dev, factors_host, ld_host,
                                                   out_vals_dev, s);
    });
}

}  // extern "C"
