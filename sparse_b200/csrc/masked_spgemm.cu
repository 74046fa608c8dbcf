// masked_spgemm.cu -- K11: masked sparse x sparse product, out = mask * (A @ B) at the mask's stored positions only.
//
// examples/triangles_example.py computes sum(a @ a * a) / 6: the unfused path builds every product of A @ B
// (sum_k |A_i,:| * |B_k,:| of them, about n d^2 for a graph of degree d) and throws nearly all of them away in the
// multiply with the mask (n d entries).  Here each stored mask entry (i, j) is the sparse dot product of row i of A
// with column j of B (row j of B^T), so memory and work scale with nnz(mask), not with the product count.
//
// Decomposition:
//   * the mask's entries (CSR order) are cut into chunks of CHUNK entries; warps take chunks from a ticket counter, so
//     power-law rows cannot unbalance the grid.  A chunk may span several short rows or be a piece of a long one.
//   * per (row, chunk) the warp stages A_i (k, a) in shared memory, in ascending-k segments of at most `cap` entries;
//     each mask entry's running sum c' lives in a shared-memory slot between segments, so the fold continues in order.
//   * lane groups of G lanes (G from the average length of a B^T row) take one mask entry each.  Normally the lanes
//     read B^T_j's indices coalesced and binary-search them in the staged segment; for a hub column (B^T_j much longer
//     than the segment) they walk the staged segment instead and binary-search B^T_j in global memory.  Either way the
//     matches of one step are in ascending k across the lanes and are folded into c' in lane order (ballot + shuffles),
//     so the sum order of include/sparse_b200.h holds.  b_kj is gathered only on a match.
//   * after the last segment, out[p] = m_p * T(c'); the caller drops bitwise +0 results with the prune compaction.
#include "common.cuh"

namespace b2s {

constexpr int MS_WARPS = 4;
constexpr int MS_CHUNK = 128;       // mask entries per work item
constexpr int MS_CAP_DEFAULT = 512; // staged A entries per segment
constexpr int MS_HUB = 32;          // B^T row longer than MS_HUB x segment: search B instead of A

static int g_ms_cap = MS_CAP_DEFAULT;  // test hook (b2s_masked_spgemm_set_stage)

template <typename I>
__device__ __forceinline__ int ms_find_smem(const I *keys, int n, I k) {  // index of k in keys[0..n) or -1
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (keys[mid] < k) lo = mid + 1;
        else hi = mid;
    }
    return (lo < n && keys[lo] == k) ? lo : -1;
}

template <typename I>
__device__ __forceinline__ int64_t ms_find_global(const I *__restrict__ keys, int64_t lo, int64_t hi, I k) {
    const int64_t end = hi;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(keys + mid) < k) lo = mid + 1;
        else hi = mid;
    }
    return (lo < end && __ldg(keys + lo) == k) ? lo : -1;
}

// Fold the products of one step into c in lane order of the group: c = ((c + p_l0) + p_l1) + ... over the hit lanes.
template <typename Tc>
__device__ __forceinline__ Tc ms_fold(Tc c, Tc prod, bool hit, unsigned gmask) {
    unsigned bal = __ballot_sync(gmask, hit) & gmask;
    while (bal) {
        const int src = __ffs(bal) - 1;
        c = add_rn(c, __shfl_sync(gmask, prod, src));
        bal &= bal - 1;
    }
    return c;
}

template <typename Tc, typename T, typename I, int G>
__global__ void __launch_bounds__(MS_WARPS * 32, 8)
masked_spgemm_kernel(int64_t M, int64_t nnz_m, const I *__restrict__ m_ptr, const I *__restrict__ m_cols,
                     const T *__restrict__ m_vals, const I *__restrict__ a_ptr, const I *__restrict__ a_cols,
                     const Tc *__restrict__ a_vals, const I *__restrict__ b_ptr, const I *__restrict__ b_cols,
                     const Tc *__restrict__ b_vals, int cap, unsigned long long *__restrict__ ticket,
                     T *__restrict__ out) {
    constexpr int NG = 32 / G;
    extern __shared__ __align__(16) unsigned char ms_smem[];
    const int lane = threadIdx.x & 31;
    const int w = threadIdx.x >> 5;
    const int g = lane / G, gl = lane % G;
    const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (g * G));
    const size_t warp_bytes = ((size_t)cap * (sizeof(Tc) + sizeof(I)) + MS_CHUNK * sizeof(Tc) + 15) & ~(size_t)15;
    Tc *s_av = reinterpret_cast<Tc *>(ms_smem + w * warp_bytes);
    Tc *s_acc = s_av + cap;
    I *s_ak = reinterpret_cast<I *>(s_acc + MS_CHUNK);
    const int64_t nchunks = (nnz_m + MS_CHUNK - 1) / MS_CHUNK;

    for (;;) {
        unsigned long long tk = 0;
        if (lane == 0) tk = atomicAdd(ticket, 1ull);
        const int64_t c = (int64_t)__shfl_sync(0xffffffffu, tk, 0);
        if (c >= nchunks) break;
        const int64_t p0 = c * MS_CHUNK;
        const int64_t p1 = p0 + MS_CHUNK < nnz_m ? p0 + MS_CHUNK : nnz_m;
        // row of entry p0: the last i with m_ptr[i] <= p0
        int64_t lo = 0, hi = M;
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if ((int64_t)__ldg(m_ptr + mid) <= p0) lo = mid;
            else hi = mid;
        }
        for (int64_t i = lo; i < M; ++i) {
            const int64_t mr0 = (int64_t)__ldg(m_ptr + i), mr1 = (int64_t)__ldg(m_ptr + i + 1);
            if (mr0 >= p1) break;
            const int64_t rs = mr0 > p0 ? mr0 : p0, re = mr1 < p1 ? mr1 : p1;
            if (rs >= re) continue;
            const int n = (int)(re - rs);
            for (int e = lane; e < n; e += 32) s_acc[e] = Tc(0);
            const int64_t a0 = (int64_t)__ldg(a_ptr + i), a1 = (int64_t)__ldg(a_ptr + i + 1);
            for (int64_t sb = a0; sb < a1; sb += cap) {
                const int slen = (int)(a1 - sb < cap ? a1 - sb : cap);
                __syncwarp();
                for (int q = lane; q < slen; q += 32) {
                    s_ak[q] = __ldg(a_cols + sb + q);
                    s_av[q] = __ldg(a_vals + sb + q);
                }
                __syncwarp();
                const I khi = s_ak[slen - 1];
                for (int r0 = 0; r0 < n; r0 += 32) {
                    // the next (up to) 32 entries: lane l loads entry r0 + l's column and B^T row extent
                    I jl = 0;
                    int64_t b0l = 0, b1l = 0;
                    if (r0 + lane < n) {
                        jl = __ldg(m_cols + rs + r0 + lane);
                        b0l = (int64_t)__ldg(b_ptr + jl);
                        b1l = (int64_t)__ldg(b_ptr + jl + 1);
                    }
                    const int cnt = n - r0 < 32 ? n - r0 : 32;
                    for (int t = 0; t < cnt; t += NG) {
                        const int le = t + g;  // this group's entry, relative to r0
                        const bool valid = le < cnt;
                        const int64_t b0 = __shfl_sync(0xffffffffu, b0l, valid ? le : 0);
                        const int64_t b1 = __shfl_sync(0xffffffffu, b1l, valid ? le : 0);
                        Tc acc = valid ? s_acc[r0 + le] : Tc(0);
                        if (valid) {
                            if (b1 - b0 > (int64_t)MS_HUB * slen) {
                                // hub: walk the staged segment, search B^T_j in global memory
                                for (int q = 0; q < slen; q += G) {
                                    const int qa = q + gl;
                                    bool hit = false;
                                    Tc prod = Tc(0);
                                    if (qa < slen) {
                                        const int64_t pb = ms_find_global(b_cols, b0, b1, s_ak[qa]);
                                        if (pb >= 0) {
                                            hit = true;
                                            prod = mul_rn(s_av[qa], __ldg(b_vals + pb));
                                        }
                                    }
                                    acc = ms_fold<Tc>(acc, prod, hit, gmask);
                                }
                            } else {
                                // walk B^T_j coalesced, search each k in the staged segment
                                for (int64_t q = b0; q < b1; q += G) {
                                    const int64_t qb = q + gl;
                                    bool hit = false, past = false;
                                    Tc prod = Tc(0);
                                    if (qb < b1) {
                                        const I kb = __ldg(b_cols + qb);
                                        past = kb > khi;
                                        const int pa = past ? -1 : ms_find_smem(s_ak, slen, kb);
                                        if (pa >= 0) {
                                            hit = true;
                                            prod = mul_rn(s_av[pa], __ldg(b_vals + qb));
                                        }
                                    }
                                    acc = ms_fold<Tc>(acc, prod, hit, gmask);
                                    if (__ballot_sync(gmask, past) & gmask) break;  // the rest of B^T_j is above khi
                                }
                            }
                            if (gl == 0) s_acc[r0 + le] = acc;
                        }
                    }
                }
            }
            __syncwarp();
            for (int e = lane; e < n; e += 32) out[rs + e] = mul_rn(__ldg(m_vals + rs + e), (T)s_acc[e]);
            __syncwarp();
        }
    }
}

// strictly increasing indices within every row (the precondition of the kernel's searches)
template <typename I>
__global__ void ms_rows_sorted_kernel(int64_t M, const I *__restrict__ indptr, const I *__restrict__ indices,
                                      int *__restrict__ flag) {
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    bool bad = false;
    for (int64_t row = warp; row < M; row += nwarps) {
        const int64_t s = (int64_t)indptr[row], e = (int64_t)indptr[row + 1];
        for (int64_t p = s + lane; p + 1 < e; p += 32) bad |= indices[p + 1] <= indices[p];
    }
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(flag, 1);
}

// flags[q] = 1 iff query[q] occurs in the ascending array set[0..ns)
__global__ void keys_member_kernel(const int64_t *__restrict__ query, int64_t nq, const int64_t *__restrict__ set,
                                   int64_t ns, uint8_t *__restrict__ flags) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += (int64_t)gridDim.x * blockDim.x)
        flags[q] = ms_find_global(set, (int64_t)0, ns, query[q]) >= 0 ? 1 : 0;
}

template <typename Tc, typename T, typename I, int G>
static void ms_launch(unsigned blocks, size_t smem, cudaStream_t s, int64_t M, int64_t nnz_m, const void *mp,
                      const void *mc, const void *mv, const void *ap, const void *ac, const void *av, const void *bp,
                      const void *bc, const void *bv, int cap, unsigned long long *ticket, void *out) {
    masked_spgemm_kernel<Tc, T, I, G><<<blocks, MS_WARPS * 32, smem, s>>>(
        M, nnz_m, (const I *)mp, (const I *)mc, (const T *)mv, (const I *)ap, (const I *)ac, (const Tc *)av,
        (const I *)bp, (const I *)bc, (const Tc *)bv, cap, ticket, (T *)out);
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_masked_spgemm_set_stage(int cap) {
    B2S_REQUIRE(cap >= 0 && cap <= MS_CAP_DEFAULT, B2S_ERR_INVALID, "masked_spgemm_set_stage: cap %d", cap);
    g_ms_cap = cap ? cap : MS_CAP_DEFAULT;
    return B2S_OK;
}

int b2s_masked_spgemm(int dtype_c, int dtype_out, int idx_bytes, int64_t M, int64_t N, int64_t K, int64_t nnz_m,
                      const void *m_indptr_dev, const void *m_cols_dev, const void *m_vals_dev,
                      const void *a_indptr_dev, const void *a_cols_dev, const void *a_vals_dev, int64_t nnz_bt,
                      const void *bt_indptr_dev, const void *bt_cols_dev, const void *bt_vals_dev, void *out_vals_dev,
                      void *stream) {
    B2S_REQUIRE(idx_bytes == 4 || idx_bytes == 8, B2S_ERR_INVALID, "masked_spgemm: idx_bytes");
    B2S_REQUIRE(M >= 0 && N >= 0 && K >= 0 && nnz_m >= 0 && nnz_bt >= 0, B2S_ERR_INVALID, "masked_spgemm: sizes");
    if (nnz_m == 0) return B2S_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const int cap = g_ms_cap;
    const int G = (N > 0 && nnz_bt >= 16 * N) ? 32 : 8;  // lanes per mask entry, from the average B^T row length
    const size_t warp_bytes = ((size_t)cap * (dtype_size(dtype_c) + idx_bytes) + MS_CHUNK * dtype_size(dtype_c) + 15) &
                              ~(size_t)15;
    const size_t smem = warp_bytes * MS_WARPS;
    const int64_t nchunks = (nnz_m + MS_CHUNK - 1) / MS_CHUNK;
    int64_t blocks = (nchunks + MS_WARPS - 1) / MS_WARPS;
    const int64_t full = (int64_t)num_sms() * 8;
    if (blocks > full) blocks = full;
    unsigned long long *ticket = nullptr;
    int rc = scratch_alloc((void **)&ticket, 8, s);
    if (rc) return rc;
    B2S_CUDA(cudaMemsetAsync(ticket, 0, 8, s));
    bool ok = true;
#define B2S_MS(TC, TO, I, GG)                                                                                        \
    ms_launch<TC, TO, I, GG>((unsigned)blocks, smem, s, M, nnz_m, m_indptr_dev, m_cols_dev, m_vals_dev,              \
                             a_indptr_dev, a_cols_dev, a_vals_dev, bt_indptr_dev, bt_cols_dev, bt_vals_dev, cap,     \
                             ticket, out_vals_dev)
#define B2S_MSG(TC, TO, I) \
    if (G == 32) B2S_MS(TC, TO, I, 32); else B2S_MS(TC, TO, I, 8);
#define B2S_MSI(TC, TO) \
    if (idx_bytes == 4) { B2S_MSG(TC, TO, int32_t) } else { B2S_MSG(TC, TO, int64_t) }
    if (dtype_c == B2S_F32 && dtype_out == B2S_F32) { B2S_MSI(float, float) }
    else if (dtype_c == B2S_F32 && dtype_out == B2S_F64) { B2S_MSI(float, double) }
    else if (dtype_c == B2S_F64 && dtype_out == B2S_F64) { B2S_MSI(double, double) }
    else if (dtype_c == B2S_I32 && dtype_out == B2S_I32) { B2S_MSI(int32_t, int32_t) }
    else if (dtype_c == B2S_I32 && dtype_out == B2S_I64) { B2S_MSI(int32_t, int64_t) }
    else if (dtype_c == B2S_I32 && dtype_out == B2S_F64) { B2S_MSI(int32_t, double) }
    else if (dtype_c == B2S_I64 && dtype_out == B2S_I64) { B2S_MSI(int64_t, int64_t) }
    else if (dtype_c == B2S_I64 && dtype_out == B2S_F64) { B2S_MSI(int64_t, double) }
    else ok = false;
#undef B2S_MSI
#undef B2S_MSG
#undef B2S_MS
    if (!ok) {
        scratch_free(ticket, s);
        B2S_REQUIRE(false, B2S_ERR_UNSUPPORTED, "masked_spgemm: dtype pair (%d, %d)", dtype_c, dtype_out);
    }
    B2S_CHECK_LAUNCH();
    return scratch_free(ticket, s);
}

int b2s_masked_spgemm_sorted(int idx_bytes, int64_t M, const void *a_indptr_dev, const void *a_cols_dev, int64_t N,
                             const void *bt_indptr_dev, const void *bt_cols_dev, int *sorted_host, void *stream) {
    B2S_REQUIRE(sorted_host != nullptr, B2S_ERR_INVALID, "masked_spgemm_sorted: NULL output");
    B2S_REQUIRE(idx_bytes == 4 || idx_bytes == 8, B2S_ERR_INVALID, "masked_spgemm_sorted: idx_bytes");
    *sorted_host = 1;
    const bool do_a = a_indptr_dev && M > 0, do_b = bt_indptr_dev && N > 0;
    if (!do_a && !do_b) return B2S_OK;
    cudaStream_t s = (cudaStream_t)stream;
    int *flag = nullptr;
    int rc = scratch_alloc((void **)&flag, 4, s);
    if (rc) return rc;
    B2S_CUDA(cudaMemsetAsync(flag, 0, 4, s));
    const int64_t cap = (int64_t)num_sms() * 16;
    for (int which = 0; which < 2; ++which) {
        const int64_t rows = which ? N : M;
        const void *ptr = which ? bt_indptr_dev : a_indptr_dev;
        const void *idx = which ? bt_cols_dev : a_cols_dev;
        if (!(which ? do_b : do_a)) continue;
        int64_t blocks = (rows * 32 + 255) / 256;
        if (blocks > cap) blocks = cap;
        if (idx_bytes == 4)
            ms_rows_sorted_kernel<int32_t><<<(unsigned)blocks, 256, 0, s>>>(rows, (const int32_t *)ptr, (const int32_t *)idx, flag);
        else
            ms_rows_sorted_kernel<int64_t><<<(unsigned)blocks, 256, 0, s>>>(rows, (const int64_t *)ptr, (const int64_t *)idx, flag);
        B2S_CHECK_LAUNCH();
    }
    int h = 0;
    B2S_CUDA(cudaMemcpyAsync(&h, flag, 4, cudaMemcpyDeviceToHost, s));
    B2S_CUDA(cudaStreamSynchronize(s));
    scratch_free(flag, s);
    *sorted_host = h ? 0 : 1;
    return B2S_OK;
}

int b2s_keys_member(const int64_t *query_dev, int64_t nq, const int64_t *set_dev, int64_t ns, uint8_t *flags_dev,
                    void *stream) {
    if (nq == 0) return B2S_OK;
    int64_t blocks = (nq + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    keys_member_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(query_dev, nq, set_dev, ns, flags_dev);
    B2S_CHECK_LAUNCH();
    return B2S_OK;
}

}  // extern "C"
