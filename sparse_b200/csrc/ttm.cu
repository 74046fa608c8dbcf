// ttm.cu -- K14: mode-n tensor times matrix (TTM) of a sparse tensor of order 2..8, with a sparse result.
//
//   Y[i_0, ..., r, ..., i_{N-1}] = sum_{i_n} X[i_0, ..., i_n, ..., i_{N-1}] * U[i_n, r]
//
// The input is the fiber stream of `mode` (built on the host, _fused._fiber_stream): the entries sorted by the key over
// the axes (other modes ascending, then `mode`), cut into fibers (runs that share every coordinate but `mode`), and the
// fibers cut into groups (runs that share the coordinates before `mode`).  A fiber of at most long_min entries is owned
// by a group of LPF lanes (a power of two, the smallest that covers R in packs of VEC columns, at most 32) that walks
// its entries in stream order, i.e. ascending i_mode, gathering one VEC-column pack of U's row per entry and lane
// (16-byte loads with an L2 evict_last hint: U is the reused operand); R wider than 32 packs is walked in column tiles.
// A longer fiber gets whole CTAs, one per column tile of 32 packs, that gather a chunk of its entries at once and stage
// the products in shared memory, so a skewed fiber length costs one serial add per entry and column instead of one
// gather latency per four entries; those CTAs come first in the grid and run beside the short-fiber ones.  Each
// (fiber, column) sum is carried by one thread from +0 to the end of the fiber, so the order of include/sparse_b200.h
// holds whatever the grid or the role, and the vector (VEC = 16 B / itemsize) and scalar (VEC = 1) forms are
// bit-identical.  No fiber is split into partial sums.
//
// Every (fiber f, r) value goes straight to its slot of the result's C order, before pruning:
//   slot = R * g0 + r * s_g + (f - g0),   key = (P * R + r) * Q_ext + Q
// with g0 / s_g the first fiber / size of f's group, P / Q the linear coordinates before / after `mode`, and Q_ext the
// product of the extents after `mode`.  The kernel writes the value, its key and a keep flag (value != 0); the caller
// compacts with the scan + compact primitives.  No atomics, no scratch memory, no stream synchronisation.
#include "tensor_modes.cuh"

namespace b2s {

constexpr int kTtmWarps = 8;                  // warps per CTA
constexpr int kTtmThreads = kTtmWarps * 32;
constexpr int kTtmUnroll = 4;                 // entries whose U packs are in flight at once (short-fiber role)
constexpr int kLongLoads = 4;                 // U packs in flight per thread (long-fiber role)
constexpr int kLongRow = kTtmThreads * kLongLoads;  // elements of a staged chunk, in packs

// slot, key and keep flag of (fiber, column r) -- see the header comment
template <typename T>
__device__ __forceinline__ void ttm_put(T y, int64_t slot, int64_t key, T *out, int64_t *okeys, uint8_t *oflags) {
    out[slot] = y;
    okeys[slot] = key;
    oflags[slot] = y != T(0);
}

// Long-fiber role: the whole CTA works on fiber f, columns [c_lo, c_lo + 32 * VEC).  Per chunk of E entries every
// thread gathers kLongLoads U packs and multiplies them by their entries' values (the products are independent, so
// this is parallel), stages them in shared memory, and one thread per column adds the chunk's products in stream order
// onto its running sum while the next chunk's gathers are in flight (double buffer).  Same bits as the short role.
template <typename T, typename I, int VEC>
__device__ __forceinline__ void ttm_long_fiber(T (*buf)[kLongRow * VEC], const I *__restrict__ kc,
                                               const T *__restrict__ vals, int64_t e0, int64_t e1,
                                               const T *__restrict__ U, int64_t ldu, int64_t R, int64_t c_lo,
                                               uint64_t pol, int64_t slot0, int64_t sg, int64_t key0, int64_t q_ext,
                                               T *out, int64_t *okeys, uint8_t *oflags) {
    const int tid = threadIdx.x;
    const int64_t left = (R - c_lo + VEC - 1) / VEC;  // packs of this column tile
    int pt_log2 = 0;
    while (pt_log2 < 5 && ((int64_t)1 << pt_log2) < left) ++pt_log2;
    const int W = VEC << pt_log2;                    // staged columns per entry
    const int E = kLongRow >> pt_log2;               // entries per chunk
    const int rstep = kTtmThreads >> pt_log2;        // entries gathered per load round
    const int row = tid >> pt_log2;
    const int sub = tid & ((1 << pt_log2) - 1);
    const int64_t col = c_lo + (int64_t)sub * VEC;
    const bool col_ok = col < R;                     // VEC divides R on the vector path
    const int ncols = (int)(R - c_lo < W ? R - c_lo : W);

    MPack<T, VEC> p[kLongLoads];
    auto gather = [&](int64_t base) {
#pragma unroll
        for (int j = 0; j < kLongLoads; ++j) {
            const int64_t e = base + row + j * rstep;
            if (e < e1 && col_ok) {
                const T v = __ldg(vals + e);
                p[j] = m_load<T, VEC>(U + (int64_t)__ldg(kc + e) * ldu + col, pol);
#pragma unroll
                for (int c = 0; c < VEC; ++c) p[j].v[c] = mul_rn(v, p[j].v[c]);
            } else {
#pragma unroll
                for (int c = 0; c < VEC; ++c) p[j].v[c] = T(0);  // staged, never summed
            }
        }
    };
    auto stage = [&](int b) {
#pragma unroll
        for (int j = 0; j < kLongLoads; ++j)
#pragma unroll
            for (int c = 0; c < VEC; ++c) buf[b][(row + j * rstep) * W + sub * VEC + c] = p[j].v[c];
    };

    T acc = T(0);
    gather(e0);
    stage(0);
    __syncthreads();
    int b = 0;
    for (int64_t base = e0; base < e1; base += E) {  // block-uniform trip count
        const int64_t next = base + E;
        if (next < e1) gather(next);
        if (tid < ncols) {
            const int n = e1 - base < E ? (int)(e1 - base) : E;
            const T *src = buf[b] + tid;
            for (int e = 0; e < n; ++e) acc = add_rn(acc, src[e * W]);
        }
        if (next < e1) stage(b ^ 1);
        __syncthreads();
        b ^= 1;
    }
    if (tid < ncols) {
        const int64_t r = c_lo + tid;
        ttm_put(acc, slot0 + r * sg, key0 + r * q_ext, out, okeys, oflags);
    }
}

// Blocks [0, n_long * tiles) take the long fibers (fptr[f + 1] - fptr[f] > long_min, listed in long_ids), one column
// tile of 32 * VEC columns each, so they start first and run beside the rest; the other blocks take consecutive fibers
// in the short-fiber role and skip the long ones.
template <typename T, typename I, int VEC>
__global__ void __launch_bounds__(kTtmThreads)
ttm_mode_kernel(const I *__restrict__ kc, const T *__restrict__ vals, const I *__restrict__ fptr,
                const I *__restrict__ fgroup, const I *__restrict__ gptr, const int64_t *__restrict__ fkey,
                const int64_t *__restrict__ pkey, const int64_t n_fibers, const int64_t *__restrict__ long_ids,
                const int64_t n_long, const int64_t long_min, const T *__restrict__ U, const int64_t ldu,
                const int64_t R, const int64_t q_ext, const int lpf_log2, T *__restrict__ out,
                int64_t *__restrict__ okeys, uint8_t *__restrict__ oflags) {
    __shared__ T buf[2][kLongRow * VEC];
    const int64_t tiles = (R + 32 * VEC - 1) / (32 * VEC);
    const int64_t long_blocks = n_long * tiles;
    const uint64_t pol = policy_evict_last();
    if ((int64_t)blockIdx.x < long_blocks) {
        const int64_t f = long_ids[blockIdx.x / tiles];
        const int64_t c_lo = (blockIdx.x % tiles) * 32 * VEC;
        const int64_t g = fgroup[f];
        const int64_t g0 = gptr[g], sg = gptr[g + 1] - g0;
        const int64_t P = pkey[f];
        ttm_long_fiber<T, I, VEC>(buf, kc, vals, fptr[f], fptr[f + 1], U, ldu, R, c_lo, pol, R * g0 + (f - g0), sg,
                                  P * R * q_ext + (fkey[f] - P * q_ext), q_ext, out, okeys, oflags);
        return;
    }
    const int lane = threadIdx.x & 31;
    const int lpf = 1 << lpf_log2;
    const int sub = lane & (lpf - 1);  // which pack of the column tile
    const int64_t f = (((int64_t)blockIdx.x - long_blocks) * kTtmWarps + (threadIdx.x >> 5)) * (32 >> lpf_log2) +
                      (lane >> lpf_log2);
    if (f >= n_fibers) return;  // no collectives below

    const int64_t e0 = fptr[f], e1 = fptr[f + 1];
    if (e1 - e0 > long_min) return;  // a long-fiber block owns it
    const int64_t g = fgroup[f];
    const int64_t g0 = gptr[g], sg = gptr[g + 1] - g0;
    const int64_t P = pkey[f];
    const int64_t Q = fkey[f] - P * q_ext;
    const int64_t slot0 = R * g0 + (f - g0);

    for (int64_t c0 = (int64_t)sub * VEC; c0 < R; c0 += (int64_t)lpf * VEC) {
        // VEC divides R on the vector path: a pack is all in or all out
        T acc[VEC];
#pragma unroll
        for (int c = 0; c < VEC; ++c) acc[c] = T(0);
        const T *u0 = U + c0;
        int64_t e = e0;
        // y_r = ((+0 + v_1 * U[k_1, r]) + v_2 * U[k_2, r]) + ... in stream order, each product and sum rounded
        for (; e + kTtmUnroll <= e1; e += kTtmUnroll) {
            I k[kTtmUnroll];
            T v[kTtmUnroll];
            MPack<T, VEC> u[kTtmUnroll];
#pragma unroll
            for (int j = 0; j < kTtmUnroll; ++j) {
                k[j] = __ldg(kc + e + j);
                v[j] = __ldg(vals + e + j);
            }
#pragma unroll
            for (int j = 0; j < kTtmUnroll; ++j) u[j] = m_load<T, VEC>(u0 + (int64_t)k[j] * ldu, pol);
#pragma unroll
            for (int j = 0; j < kTtmUnroll; ++j)
#pragma unroll
                for (int c = 0; c < VEC; ++c) acc[c] = add_rn(acc[c], mul_rn(v[j], u[j].v[c]));
        }
        for (; e < e1; ++e) {
            const MPack<T, VEC> u = m_load<T, VEC>(u0 + (int64_t)__ldg(kc + e) * ldu, pol);
            const T v = __ldg(vals + e);
#pragma unroll
            for (int c = 0; c < VEC; ++c) acc[c] = add_rn(acc[c], mul_rn(v, u.v[c]));
        }
        const int64_t key0 = (P * R + c0) * q_ext + Q;
        if constexpr (VEC > 1) {
            if (sg == 1) {
                // a group of one fiber (always at mode N-1): the pack's VEC slots and keys are contiguous and aligned
                const int64_t s = slot0 + c0;
                MPack<T, VEC> p;
                uint8_t fl[VEC];
#pragma unroll
                for (int c = 0; c < VEC; ++c) {
                    p.v[c] = acc[c];
                    fl[c] = acc[c] != T(0);
                }
                uint4 w;
                memcpy(&w, &p, 16);
                stg_cs_v4(out + s, w);
#pragma unroll
                for (int c = 0; c < VEC; c += 2) {
                    const longlong2 kk = make_longlong2(key0 + c * q_ext, key0 + (c + 1) * q_ext);
                    memcpy(&w, &kk, 16);
                    stg_cs_v4(okeys + s + c, w);
                }
                if constexpr (VEC == 4) {
                    uint32_t fw;
                    memcpy(&fw, fl, 4);
                    *reinterpret_cast<uint32_t *>(oflags + s) = fw;
                } else {
                    uint16_t fw;
                    memcpy(&fw, fl, 2);
                    *reinterpret_cast<uint16_t *>(oflags + s) = fw;
                }
                continue;
            }
        }
#pragma unroll
        for (int c = 0; c < VEC; ++c)
            ttm_put(acc[c], slot0 + (c0 + c) * sg, key0 + c * q_ext, out, okeys, oflags);
    }
}

// flags[f] = 1 iff fiber f has more than long_min entries
template <typename I>
__global__ void ttm_long_flags_kernel(const I *__restrict__ fptr, int64_t n_fibers, int64_t long_min,
                                      uint8_t *__restrict__ flags) {
    for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f < n_fibers;
         f += (int64_t)gridDim.x * blockDim.x)
        flags[f] = (int64_t)fptr[f + 1] - (int64_t)fptr[f] > long_min;
}

template <typename T, typename I, int VEC>
static void launch_ttm(const I *kc, const T *vals, const I *fptr, const I *fgroup, const I *gptr, const int64_t *fkey,
                       const int64_t *pkey, int64_t n_fibers, const int64_t *long_ids, int64_t n_long, int64_t long_min,
                       const T *U, int64_t ldu, int64_t R, int64_t q_ext, int lpf_log2, T *out, int64_t *okeys,
                       uint8_t *oflags, unsigned blocks, cudaStream_t s) {
    ttm_mode_kernel<T, I, VEC><<<blocks, kTtmThreads, 0, s>>>(kc, vals, fptr, fgroup, gptr, fkey, pkey, n_fibers,
                                                              long_ids, n_long, long_min, U, ldu, R, q_ext, lpf_log2,
                                                              out, okeys, oflags);
}

template <typename T, typename I>
static int ttm_impl(int64_t n_fibers, int64_t R, int64_t q_ext, const void *kc, const void *vals, const void *fptr,
                    const void *fgroup, const void *gptr, const int64_t *fkey, const int64_t *pkey,
                    const int64_t *long_ids, int64_t n_long, int64_t long_min, const void *U, int64_t ldu, void *out,
                    int64_t *okeys, uint8_t *oflags, cudaStream_t s) {
    constexpr int VEC = 16 / sizeof(T);
    const bool aligned = R % VEC == 0 && ldu % VEC == 0 && ((uintptr_t)U & 15) == 0;
    const int vec = aligned ? VEC : 1;
    const int64_t packs = (R + vec - 1) / vec;
    int lpf_log2 = 0;
    while (lpf_log2 < 5 && ((int64_t)1 << lpf_log2) < packs) ++lpf_log2;
    const int64_t per_block = (int64_t)kTtmWarps * (32 >> lpf_log2);
    const int64_t tiles = (R + 32 * vec - 1) / (32 * vec);
    const int64_t blocks = n_long * tiles + (n_fibers + per_block - 1) / per_block;
    B2S_REQUIRE(blocks <= INT32_MAX, B2S_ERR_INVALID, "ttm_mode: %lld fibers exceed one grid", (long long)n_fibers);
    if (aligned)
        launch_ttm<T, I, VEC>((const I *)kc, (const T *)vals, (const I *)fptr, (const I *)fgroup, (const I *)gptr, fkey,
                              pkey, n_fibers, long_ids, n_long, long_min, (const T *)U, ldu, R, q_ext, lpf_log2,
                              (T *)out, okeys, oflags, (unsigned)blocks, s);
    else
        launch_ttm<T, I, 1>((const I *)kc, (const T *)vals, (const I *)fptr, (const I *)fgroup, (const I *)gptr, fkey,
                            pkey, n_fibers, long_ids, n_long, long_min, (const T *)U, ldu, R, q_ext, lpf_log2,
                            (T *)out, okeys, oflags, (unsigned)blocks, s);
    const cudaError_t e = cudaGetLastError();
    count_launch();
    B2S_REQUIRE(e == cudaSuccess, B2S_ERR_CUDA, "ttm_mode: kernel launch failed: %s", cudaGetErrorString(e));
    return B2S_OK;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_ttm_mode_long_flags(int idx_bytes, int64_t n_fibers, const void *fptr_dev, int64_t long_min,
                            uint8_t *flags_out_dev, void *stream) {
    B2S_REQUIRE(idx_bytes == 4 || idx_bytes == 8, B2S_ERR_INVALID, "ttm_mode_long_flags: idx_bytes");
    B2S_REQUIRE(n_fibers >= 0 && long_min >= 0, B2S_ERR_INVALID, "ttm_mode_long_flags: negative size");
    if (n_fibers == 0) return B2S_OK;
    B2S_REQUIRE(fptr_dev && flags_out_dev, B2S_ERR_INVALID, "ttm_mode_long_flags: NULL pointer");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t want = (n_fibers + 255) / 256;
    const unsigned blocks = (unsigned)(want < 65535 ? want : 65535);
    if (idx_bytes == 4)
        ttm_long_flags_kernel<int32_t><<<blocks, 256, 0, s>>>((const int32_t *)fptr_dev, n_fibers, long_min,
                                                              flags_out_dev);
    else
        ttm_long_flags_kernel<int64_t><<<blocks, 256, 0, s>>>((const int64_t *)fptr_dev, n_fibers, long_min,
                                                              flags_out_dev);
    B2S_CHECK_LAUNCH();
    return B2S_OK;
}

int b2s_ttm_mode(int dtype, int idx_bytes, int64_t n_fibers, int64_t R, int64_t q_ext, const void *kcoord_dev,
                 const void *vals_dev, const void *fptr_dev, const void *fgroup_dev, const void *gptr_dev,
                 const int64_t *fkey_dev, const int64_t *pkey_dev, const int64_t *long_ids_dev, int64_t n_long,
                 int64_t long_min, const void *u_dev, int64_t ldu, void *out_vals_dev, int64_t *out_keys_dev,
                 uint8_t *out_flags_dev, void *stream) {
    const char *op = "ttm_mode";
    B2S_REQUIRE(dtype == B2S_F32 || dtype == B2S_F64, B2S_ERR_UNSUPPORTED, "%s: dtype %d (f32/f64 only)", op, dtype);
    B2S_REQUIRE(idx_bytes == 4 || idx_bytes == 8, B2S_ERR_INVALID, "%s: idx_bytes", op);
    B2S_REQUIRE(n_fibers >= 0 && R >= 0 && q_ext >= 1 && n_long >= 0 && n_long <= n_fibers && long_min >= 0,
                B2S_ERR_INVALID, "%s: negative size", op);
    if (n_fibers == 0 || R == 0) return B2S_OK;
    B2S_REQUIRE(ldu >= R, B2S_ERR_INVALID, "%s: ldu %lld < R %lld", op, (long long)ldu, (long long)R);
    B2S_REQUIRE(kcoord_dev && vals_dev && fptr_dev && fgroup_dev && gptr_dev && fkey_dev && pkey_dev && u_dev &&
                    out_vals_dev && out_keys_dev && out_flags_dev && (n_long == 0 || long_ids_dev),
                B2S_ERR_INVALID, "%s: NULL pointer", op);
    cudaStream_t s = (cudaStream_t)stream;
    return dispatch_tensor(dtype, idx_bytes, [&](auto t, auto i) {
        return ttm_impl<decltype(t), decltype(i)>(n_fibers, R, q_ext, kcoord_dev, vals_dev, fptr_dev, fgroup_dev,
                                                  gptr_dev, fkey_dev, pkey_dev, long_ids_dev, n_long, long_min, u_dev,
                                                  ldu, out_vals_dev, out_keys_dev, out_flags_dev, s);
    });
}

}  // extern "C"
