// sptc.cu -- K17: the two steps that sparse x sparse tensor contraction (sptc) adds around K4 (spgemm.cu).
//
// Both operands reach K4 as doubly-compressed CSR (DCSR, built on the host by _fused._sptc_stream): only the rows that
// hold entries exist, each with its linear key (xrows[nF] over X's free axes, yrows[nC] over the contracted axes), and
// Y's columns are ranks among its distinct free keys ycols[nG].  Nothing is sized by an extent.
//
//   b2s_sptc_join  out[q] = the index of query[q] in the ascending, duplicate-free int64 array set[0..ns), or ns when
//                  it is absent.  With set = yrows and query = the contracted key of every X entry it gives K4's A
//                  column ids (ns = nC is a B row without entries); with set = ycols and query = Y's free keys, all
//                  present, it gives Y's column ranks.  Each thread takes kJoinPer consecutive queries (two 16-byte
//                  streaming loads) and bisects the set through the read-only path with an L2 evict_last hint: the set
//                  is read again and again, the queries once.  The kJoinPer bisections of a thread are independent, so
//                  their loads overlap; starting a query from its left neighbour's answer (queries ascend inside a row
//                  of X) chains them and measured 1.3-1.6x slower (DESIGN K17).  Any query order is allowed.
//   b2s_sptc_keys  keys[i] = xrows[rows[i]] * g_ext + ycols[cols[i]] for K4's (rows, cols) output: the result's
//                  linear keys, ascending because K4's SORTED order is (row, column rank) order.  Two entries per
//                  thread, one 16-byte streaming store.
//
// No atomics, no scratch memory, no stream synchronisation.
#include "common.cuh"

namespace b2s {

constexpr int kJoinThreads = 256;
constexpr int kJoinPer = 4;  // consecutive queries per thread

__device__ __forceinline__ int64_t ld_set(const int64_t *p, uint64_t pol) {
    int64_t v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.b64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
    return v;
}

// first position in [lo, hi) whose element is >= q (hi when none)
__device__ __forceinline__ int64_t lower_bound(const int64_t *__restrict__ set, int64_t lo, int64_t hi, int64_t q,
                                               uint64_t pol) {
    while (lo < hi) {
        const int64_t mid = lo + ((hi - lo) >> 1);
        if (ld_set(set + mid, pol) < q) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

template <typename I>
__global__ void __launch_bounds__(kJoinThreads)
sptc_join_kernel(const int64_t *__restrict__ query, const int64_t nq, const int64_t *__restrict__ set,
                 const int64_t ns, I *__restrict__ out) {
    const uint64_t pol = policy_evict_last();
    const int64_t base = ((int64_t)blockIdx.x * kJoinThreads + threadIdx.x) * kJoinPer;
    if (base >= nq) return;
    int64_t q[kJoinPer];
    const bool whole = base + kJoinPer <= nq;
    if (whole) {
#pragma unroll
        for (int j = 0; j < kJoinPer; j += 2) {
            const longlong2 v = __ldcs(reinterpret_cast<const longlong2 *>(query + base + j));
            q[j] = v.x;
            q[j + 1] = v.y;
        }
    } else {
#pragma unroll
        for (int j = 0; j < kJoinPer; ++j) q[j] = base + j < nq ? __ldcs(query + base + j) : 0;
    }
    int64_t lb[kJoinPer];
    I r[kJoinPer];
#pragma unroll
    for (int j = 0; j < kJoinPer; ++j) {
        lb[j] = lower_bound(set, 0, ns, q[j], pol);
    }
#pragma unroll
    for (int j = 0; j < kJoinPer; ++j) r[j] = (I)(lb[j] < ns && ld_set(set + lb[j], pol) == q[j] ? lb[j] : ns);
    if (whole) {
        // base is a multiple of kJoinPer: 16-byte aligned for either index width
        if constexpr (sizeof(I) == 4) {
            stg_cs_v4(out + base, make_uint4((uint32_t)r[0], (uint32_t)r[1], (uint32_t)r[2], (uint32_t)r[3]));
        } else {
#pragma unroll
            for (int j = 0; j < kJoinPer; j += 2) {
                const longlong2 p = make_longlong2(r[j], r[j + 1]);
                uint4 w;
                memcpy(&w, &p, 16);
                stg_cs_v4(out + base + j, w);
            }
        }
    } else {
#pragma unroll
        for (int j = 0; j < kJoinPer; ++j)
            if (base + j < nq) out[base + j] = r[j];
    }
}

__global__ void __launch_bounds__(256)
sptc_keys_kernel(const int64_t n, const int64_t *__restrict__ rows, const int64_t *__restrict__ cols,
                 const int64_t *__restrict__ xrows, const int64_t *__restrict__ ycols, const int64_t g_ext,
                 int64_t *__restrict__ keys) {
    const uint64_t pol = policy_evict_last();
    const int64_t i = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 2;
    if (i >= n) return;
    if (i + 1 < n) {
        const longlong2 r = __ldcs(reinterpret_cast<const longlong2 *>(rows + i));
        const longlong2 c = __ldcs(reinterpret_cast<const longlong2 *>(cols + i));
        const longlong2 k = make_longlong2(ld_set(xrows + r.x, pol) * g_ext + ld_set(ycols + c.x, pol),
                                           ld_set(xrows + r.y, pol) * g_ext + ld_set(ycols + c.y, pol));
        uint4 w;
        memcpy(&w, &k, 16);
        stg_cs_v4(keys + i, w);
    } else {
        keys[i] = ld_set(xrows + __ldcs(rows + i), pol) * g_ext + ld_set(ycols + __ldcs(cols + i), pol);
    }
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_sptc_join(int idx_bytes, int64_t nq, const int64_t *query_dev, int64_t ns, const int64_t *set_dev,
                  void *out_dev, void *stream) {
    const char *op = "sptc_join";
    B2S_REQUIRE(idx_bytes == 4 || idx_bytes == 8, B2S_ERR_INVALID, "%s: idx_bytes %d (4 or 8)", op, idx_bytes);
    B2S_REQUIRE(nq >= 0 && ns >= 0, B2S_ERR_INVALID, "%s: negative size", op);
    B2S_REQUIRE(idx_bytes == 8 || ns < 2147483647LL, B2S_ERR_INVALID, "%s: a set of %lld does not fit 4-byte indices",
                op, (long long)ns);
    if (nq == 0) return B2S_OK;
    B2S_REQUIRE(query_dev && out_dev && (ns == 0 || set_dev), B2S_ERR_INVALID, "%s: NULL pointer", op);
    B2S_REQUIRE(((uintptr_t)query_dev & 15) == 0 && ((uintptr_t)out_dev & 15) == 0, B2S_ERR_INVALID,
                "%s: query and out must be 16-byte aligned", op);
    const int64_t per_block = (int64_t)kJoinThreads * kJoinPer;
    const int64_t blocks = (nq + per_block - 1) / per_block;
    B2S_REQUIRE(blocks <= INT32_MAX, B2S_ERR_INVALID, "%s: %lld queries exceed one grid", op, (long long)nq);
    cudaStream_t s = (cudaStream_t)stream;
    if (idx_bytes == 4)
        sptc_join_kernel<int32_t><<<(unsigned)blocks, kJoinThreads, 0, s>>>(query_dev, nq, set_dev, ns,
                                                                            (int32_t *)out_dev);
    else
        sptc_join_kernel<int64_t><<<(unsigned)blocks, kJoinThreads, 0, s>>>(query_dev, nq, set_dev, ns,
                                                                            (int64_t *)out_dev);
    B2S_CHECK_LAUNCH();
    return B2S_OK;
}

int b2s_sptc_keys(int64_t n, const int64_t *rows_dev, const int64_t *cols_dev, const int64_t *xrows_dev,
                  const int64_t *ycols_dev, int64_t g_ext, int64_t *keys_out_dev, void *stream) {
    const char *op = "sptc_keys";
    B2S_REQUIRE(n >= 0 && g_ext >= 1, B2S_ERR_INVALID, "%s: n %lld, g_ext %lld", op, (long long)n, (long long)g_ext);
    if (n == 0) return B2S_OK;
    B2S_REQUIRE(rows_dev && cols_dev && xrows_dev && ycols_dev && keys_out_dev, B2S_ERR_INVALID, "%s: NULL pointer",
                op);
    B2S_REQUIRE((((uintptr_t)rows_dev | (uintptr_t)cols_dev | (uintptr_t)keys_out_dev) & 15) == 0, B2S_ERR_INVALID,
                "%s: rows, cols and keys must be 16-byte aligned", op);
    const int64_t blocks = (n + 511) / 512;
    B2S_REQUIRE(blocks <= INT32_MAX, B2S_ERR_INVALID, "%s: %lld entries exceed one grid", op, (long long)n);
    sptc_keys_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n, rows_dev, cols_dev, xrows_dev, ycols_dev,
                                                                        g_ext, keys_out_dev);
    B2S_CHECK_LAUNCH();
    return B2S_OK;
}

}  // extern "C"
