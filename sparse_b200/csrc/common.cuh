// common.cuh -- shared helpers for the sm_90a kernels of libsparse_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "sparse_b200.h"

namespace b2s {

// ---------------------------------------------------------------------------
// error plumbing (thread-local message, no exceptions across the ABI)
// ---------------------------------------------------------------------------
void set_error(const char *fmt, ...);
void count_launch(int n = 1);

#define B2S_CUDA(expr)                                                                          \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess) {                                                                \
            b2s::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,                 \
                           cudaGetErrorString(_e));                                             \
            return B2S_ERR_CUDA;                                                                \
        }                                                                                       \
    } while (0)

#define B2S_CHECK_LAUNCH()                                                                      \
    do {                                                                                        \
        b2s::count_launch();                                                                    \
        cudaError_t _e = cudaGetLastError();                                                    \
        if (_e != cudaSuccess) {                                                                \
            b2s::set_error("kernel launch failed at %s:%d: %s", __FILE__, __LINE__,             \
                           cudaGetErrorString(_e));                                             \
            return B2S_ERR_CUDA;                                                                \
        }                                                                                       \
    } while (0)

#define B2S_REQUIRE(cond, code, ...)                                                            \
    do {                                                                                        \
        if (!(cond)) {                                                                          \
            b2s::set_error(__VA_ARGS__);                                                        \
            return (code);                                                                      \
        }                                                                                       \
    } while (0)

inline size_t dtype_size(int dt) {
    switch (dt) {
        case B2S_F32: return 4;
        case B2S_F64: return 8;
        case B2S_I32: return 4;
        case B2S_I64: return 8;
        case B2S_BOOL: return 1;
        default: return 0;
    }
}

constexpr int kNumSMsH100 = 132;  // H100 SXM; used only if the device query fails

// number of SMs of the current device (cached)
int num_sms();

// Stream-ordered scratch memory (cudaMallocAsync pool); freed with scratch_free.
int scratch_alloc(void **p, size_t nbytes, cudaStream_t s);
int scratch_free(void *p, cudaStream_t s);

// K1 internals shared with the host-buffer pipeline (spmm_host.cu)
int spmm_csr_dense_impl(int dtype, int idx_bytes, int64_t M, int64_t K, int64_t N, const void *ad, const void *ai,
                        const void *ap, const void *b, int64_t ldb, void *out, int64_t ldc, cudaStream_t s);
int narrow_i64_i32(const int64_t *in, int32_t *out, int64_t n, cudaStream_t s);
void set_call_skew(int v);  // per-call override of the long-row path (-1 = process default)
// per-call guard of the one-pass kernel: it returns at entry while *guard == 0 (nullptr = always runs)
void set_call_guard(const int *guard);
extern int g_tile_hint;  // spmm_panel.cu: L2 evict_last hint on the B loads of the tiled passes (tuning)

// ---------------------------------------------------------------------------
// exact (non-contracted) arithmetic: the reference rounds a*b and (+) separately
// ---------------------------------------------------------------------------
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ int32_t mul_rn(int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); }
__device__ __forceinline__ int64_t mul_rn(int64_t a, int64_t b) { return (int64_t)((uint64_t)a * (uint64_t)b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ int32_t add_rn(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
__device__ __forceinline__ int64_t add_rn(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }

// ---------------------------------------------------------------------------
// cache-policy helpers (sm_80+: createpolicy; used for L2 evict_first / evict_last)
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint64_t policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}

// 16-byte gather load: read-only path, no L1 allocation, L2 policy hint.
__device__ __forceinline__ uint4 ldg_nc_v4_hint(const void *p, uint64_t pol) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ uint4 ldg_nc_v4(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
// streaming 16-byte store (written once, never re-read by this kernel)
__device__ __forceinline__ void stg_cs_v4(void *p, uint4 v) {
    asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}
// streaming scalar loads of the A stream (read exactly once)
template <typename T>
__device__ __forceinline__ T ldg_stream(const T *p) {
    return __ldcs(p);
}

}  // namespace b2s
