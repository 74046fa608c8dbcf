// tensor_modes.cuh -- what the sparse-tensor kernels K10 / K12 (mttkrp.cu) and K13 (tttp.cu) share: the per-mode
// pointer arrays, the factor-row pack and its load, and the argument checks and dtype x index-width dispatch of their
// C entry points.
#pragma once
#include "common.cuh"

namespace b2s {

// coordinate array, factor and factor row stride of up to N modes, passed to a kernel by value
template <typename I, int N>
struct ModeArrays {
    const I *coord[N];
    const void *fac[N];
    int64_t ld[N];
};

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
