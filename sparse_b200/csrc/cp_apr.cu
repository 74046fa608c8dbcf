// cp_apr.cu -- K16: the fused ratio MTTKRP of Poisson CP (CP-APR), mode n of a sparse tensor of order 2..8, in a fixed
// order.
//
//   m_e       = sum_r  U_0[i_0(e), r] * U_1[i_1(e), r] * ... * U_{N-1}[i_{N-1}(e), r]   the model at e (B = U_n too)
//   w_e       = v_e / max(m_e, eps)                                                       (a NaN m_e stays NaN)
//   out[i, r] = sum over stored e with i_n(e) = i of  ((w_e * U_a[i_a, r]) * U_b[i_b, r]) * ...   (a < b < ... != n)
//
// Input is K10's mode stream S_n, cut into the same chunks of B2S_MTTKRP_CHUNK entries.  A group of G lanes owns one
// chunk and all R columns, VEC columns (one 16-byte pack) per lane; G is the packs per row rounded up to a power of
// two, so a narrow R puts several chunks in one warp, as K10 does.  The group reads the stream G entries at a time,
// one per lane, and takes them U at a time: every lane gathers its pack of all N factor rows of the U entries (L2
// evict_last: the factors are the reused operand), forms q = ((U_0 * U_1) * U_2) * ... and writes it to the entry's
// padded row in shared memory.  The lane that read the entry adds that row in ascending r from +0 (K13's order) to get
// m, then d = max(m, eps) and w = v / d; w goes back to the group by shuffles, and each lane forms
// p = ((w * U_a) * U_b) * ... from the packs still in its registers and adds it to its row accumulators.  So each
// factor row is gathered once per entry.  Row flushes, the rows that cross chunks (K10's combine kernel, from
// tensor_modes.cuh) and the zeroing of rows without entries are K10's, so the sums are b2s_mttkrp_mode's steps 4-5.
//
// Factors that are not 16-byte aligned with a row stride that is a multiple of VEC, or an R that is not a multiple of
// VEC, are first copied to aligned rows of R' = ceil(R / VEC) * VEC columns with +0 in the pad.  That is exact: a
// padded column's q is +0, and m is never -0 (it starts at +0), so m + (+0) = m; and only columns < R are written.  So
// there is one kernel form.  No atomics: the result is the order of include/sparse_b200.h whatever the grid, index
// width or factor layout.
#include <cmath>

#include "tensor_modes.cuh"

namespace b2s {

constexpr int kAprMaxOrder = 8;
constexpr int kAprWarps = 8;  // warps per CTA

template <typename I>
using AprModes = ModeArrays<I, kAprMaxOrder>;

template <typename T, typename I, int VEC, int G, int U, int NM>
__global__ void __launch_bounds__(kAprWarps * 32)
cp_apr_phi_kernel(const AprModes<I> md, const int order, const int mode, const I *__restrict__ rowc,
                  const T *__restrict__ vals, const int64_t nnz, const int64_t rows, const int R, const T eps,
                  T *__restrict__ out, const int64_t ldo, T *__restrict__ pieces, const int64_t ldp) {
    static_assert(G >= 1 && G <= 32 && (G & (G - 1)) == 0, "G must be a power of two <= 32");
    static_assert(U <= G && G % U == 0, "U must divide G");
    static_assert(NM <= kAprMaxOrder, "NM: the largest order of the instantiation");
    constexpr int NG = 32 / G;         // chunks per warp
    constexpr int LDS = G * VEC + 1;   // padded shared row: the owners' column reads are conflict-free
    constexpr unsigned FULL = 0xffffffffu;
    __shared__ T qs[kAprWarps][NG * U * LDS];

    const int lane = threadIdx.x & 31;
    const int sub = lane & (G - 1);
    const int64_t chunk = ((int64_t)blockIdx.x * kAprWarps + (threadIdx.x >> 5)) * NG + lane / G;
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    const int col0 = sub * VEC;
    const bool col_ok = col0 < R;  // the factors hold whole packs (R' columns): a pack is all in or all out
    T *sq = qs[threadIdx.x >> 5] + (lane / G) * U * LDS;
    const uint64_t pol = policy_evict_last();

    // this lane's columns < R of one row
    auto store = [&](T *row, const T (&v)[VEC]) {
#pragma unroll
        for (int k = 0; k < VEC; ++k)
            if (col0 + k < R) row[col0 + k] = v[k];
    };
    auto zero_rows = [&](int64_t from, int64_t to) {
        T z[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) z[k] = T(0);
        for (int64_t r = from; r < to; ++r) store(out + r * ldo, z);
    };
    auto any = [&](bool p) -> bool {
        if constexpr (G == 32) return p;  // one chunk per warp: already uniform
        else return __any_sync(FULL, p);
    };

    ChunkSpan sp(chunk);  // lanes past the last chunk walk an empty span, but still join the shuffles
    if (chunk < nchunks) {
        sp = ChunkSpan(rowc, nnz, chunk);
        zero_rows(sp.prev + 1, sp.row_first);
        if (sp.end == nnz) zero_rows(sp.row_last + 1, rows);
    }
    int64_t base = sp.base;
    const int64_t end = sp.end;

    T acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = T(0);
    int64_t cur = sp.row_first;
    // a row complete in the chunk goes to `out`, a crossing one to its piece row
    auto flush = [&](int64_t r) { store(sp.dest(pieces, ldp, r, out, ldo), acc); };

    // prefetch the first G entries of the stream: every mode's coordinate (the row is coordinate `mode`) and the value
    I c_n[NM];
    T v_n = T(0);
#pragma unroll
    for (int m = 0; m < NM; ++m) c_n[m] = 0;
    if (base + sub < end) {
        v_n = ldg_stream(vals + base + sub);
#pragma unroll
        for (int m = 0; m < NM; ++m)
            if (m < order) c_n[m] = ldg_stream(md.coord[m] + base + sub);
    }

    while (any(base < end)) {
        I c[NM];
#pragma unroll
        for (int m = 0; m < NM; ++m) c[m] = c_n[m];
        const T v = v_n;
        const int64_t rem = end - base;
        const int cnt = rem > G ? G : (rem > 0 ? (int)rem : 0);
        const int64_t nb = base + G;
        if (nb + sub < end) {  // next G entries while these are consumed
            v_n = ldg_stream(vals + nb + sub);
#pragma unroll
            for (int m = 0; m < NM; ++m)
                if (m < order) c_n[m] = ldg_stream(md.coord[m] + nb + sub);
        }
#pragma unroll 1
        for (int j = 0; j < G; j += U) {
            if (!any(j < cnt)) break;
            // this lane's pack of every factor row of entries j .. j + U - 1
            MPack<T, VEC> f[U][NM];
            int64_t rr[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                rr[u] = 0;
#pragma unroll
                for (int m = 0; m < NM; ++m) {
                    if (m < order) {
                        const I ix = __shfl_sync(FULL, c[m], j + u, G);
                        if (m == mode) rr[u] = (int64_t)ix;
                        if (j + u < cnt && col_ok)
                            f[u][m] = m_load<T, VEC>((const T *)md.fac[m] + (int64_t)ix * md.ld[m] + col0, pol);
                        else {
#pragma unroll
                            for (int k = 0; k < VEC; ++k) f[u][m].v[k] = T(0);
                        }
                    }
                }
            }
            // q = ((U_0 * U_1) * U_2) * ... over every mode in ascending order, each product rounded, to the entry's row
#pragma unroll
            for (int u = 0; u < U; ++u) {
                T q[VEC];
#pragma unroll
                for (int m = 0; m < NM; ++m) {
                    if (m < order) {
#pragma unroll
                        for (int k = 0; k < VEC; ++k) q[k] = m == 0 ? f[u][m].v[k] : mul_rn(q[k], f[u][m].v[k]);
                    }
                }
#pragma unroll
                for (int k = 0; k < VEC; ++k) sq[u * LDS + col0 + k] = q[k];
            }
            __syncwarp();
            // the lane that read entry j + u: m = ((+0 + q_0) + q_1) + ... in ascending r, d = eps if m < eps else m
            // (NaN stays NaN), w = v / d correctly rounded
            T w = T(0);
            const int own = sub - j;
            if (own >= 0 && own < U && sub < cnt) {
                const T *qr = sq + own * LDS;
                T mv = T(0);
#pragma unroll 4
                for (int k = 0; k < R; ++k) mv = add_rn(mv, qr[k]);
                w = div_rn(v, mv < eps ? eps : mv);
            }
            __syncwarp();  // the rows are read before the next U entries overwrite them
            // p = ((w * U_a) * U_b) * ... over the modes other than `mode`, ascending, added to the row in stream order
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const T wu = __shfl_sync(FULL, w, j + u, G);
                if (j + u < cnt) {
                    if (rr[u] != cur) {
                        flush(cur);
                        zero_rows(cur + 1, rr[u]);
                        cur = rr[u];
#pragma unroll
                        for (int k = 0; k < VEC; ++k) acc[k] = T(0);
                    }
                    T p[VEC];
#pragma unroll
                    for (int k = 0; k < VEC; ++k) p[k] = wu;
#pragma unroll
                    for (int m = 0; m < NM; ++m) {
                        if (m < order && m != mode) {
#pragma unroll
                            for (int k = 0; k < VEC; ++k) p[k] = mul_rn(p[k], f[u][m].v[k]);
                        }
                    }
#pragma unroll
                    for (int k = 0; k < VEC; ++k) acc[k] = add_rn(acc[k], p[k]);
                }
            }
        }
        base = nb;
    }
    if (chunk < nchunks) flush(cur);
}

// the arguments of one K16 launch
template <typename T, typename I>
struct PhiArgs {
    AprModes<I> md;  // every mode, B's included; the factors hold whole 16-byte packs
    int order, mode, R;
    const I *rowc;
    const T *vals;
    int64_t nnz, rows;
    T eps;
    T *out;
    int64_t ldo;
    T *pieces;
    int64_t ldp;
};

template <typename T, typename I, int VEC, int G, int U>
static int launch_phi(const PhiArgs<T, I> &a, cudaStream_t s) {
    constexpr int chunks_per_block = kAprWarps * (32 / G);
    const int64_t nchunks = (a.nnz + kChunk - 1) / kChunk;
    const int64_t blocks = (nchunks + chunks_per_block - 1) / chunks_per_block;
    B2S_REQUIRE(blocks <= INT32_MAX, B2S_ERR_INVALID, "cp_apr_phi_mode: nnz %lld exceeds one grid", (long long)a.nnz);
    // orders up to 4 (the common case) hold packs of 4 factor rows per entry, which leaves room for more warps
    auto kern = a.order <= 4 ? cp_apr_phi_kernel<T, I, VEC, G, U, 4> : cp_apr_phi_kernel<T, I, VEC, G, U, 8>;
    kern<<<(unsigned)blocks, kAprWarps * 32, 0, s>>>(a.md, a.order, a.mode, a.rowc, a.vals, a.nnz, a.rows, a.R, a.eps,
                                                     a.out, a.ldo, a.pieces, a.ldp);
    return B2S_OK;
}

// group width from the packs per row, as K10's dispatch_mode; up to 4 entries' gathers in flight per lane (2 for the
// 32-lane float64 groups, which spill with 4)
template <typename T, typename I>
static int dispatch_phi(const PhiArgs<T, I> &a, cudaStream_t s) {
    constexpr int VEC = 16 / sizeof(T);
    const int packs = (a.R + VEC - 1) / VEC;
    if constexpr (VEC == 2) {  // R <= 64: only float64 needs more than 16 packs
        if (packs > 16) return launch_phi<T, I, VEC, 32, 2>(a, s);
    }
    if (packs > 8) return launch_phi<T, I, VEC, 16, 4>(a, s);
    if (packs > 4) return launch_phi<T, I, VEC, 8, 4>(a, s);
    if (packs > 2) return launch_phi<T, I, VEC, 4, 4>(a, s);
    if (packs > 1) return launch_phi<T, I, VEC, 2, 2>(a, s);
    return launch_phi<T, I, VEC, 1, 1>(a, s);
}

template <typename T, typename I>
static int cp_apr_phi_impl(int order, int mode, int64_t nnz, int64_t rows, int R, T eps, const void *const *coords,
                           const void *vals, const void *const *factors, const int64_t *ld, const int64_t *extents,
                           void *out, int64_t ldo, cudaStream_t s) {
    constexpr int VEC = 16 / sizeof(T);
    const int64_t Rp = (R + VEC - 1) / VEC * VEC;
    PhiArgs<T, I> a{};
    // the factors the kernel cannot gather as aligned packs get an aligned copy of Rp columns, +0 in the pad
    bool pad[kAprMaxOrder];
    int64_t pad_elems = 0;
    for (int m = 0; m < order; ++m) {
        pad[m] = Rp != R || ((uintptr_t)factors[m] & 15) != 0 || ld[m] % VEC != 0;
        if (pad[m]) pad_elems += extents[m] * Rp;
    }
    T *padded = nullptr;
    if (pad_elems > 0) {
        const int rc = scratch_alloc((void **)&padded, (size_t)pad_elems * sizeof(T), s);
        if (rc) return rc;
    }
    cudaError_t e = cudaSuccess;
    T *next = padded;
    for (int m = 0; m < order; ++m) {
        a.md.coord[m] = (const I *)coords[m];
        a.md.fac[m] = factors[m];
        a.md.ld[m] = ld[m];
        if (!pad[m]) continue;
        a.md.fac[m] = next;
        a.md.ld[m] = Rp;
        if (extents[m] > 0 && e == cudaSuccess) {
            const size_t pitch = (size_t)Rp * sizeof(T);
            if (Rp > R) e = cudaMemset2DAsync(next + R, pitch, 0, (size_t)(Rp - R) * sizeof(T), (size_t)extents[m], s);
            if (e == cudaSuccess)
                e = cudaMemcpy2DAsync(next, pitch, factors[m], (size_t)ld[m] * sizeof(T), (size_t)R * sizeof(T),
                                      (size_t)extents[m], cudaMemcpyDeviceToDevice, s);
        }
        next += extents[m] * Rp;
    }
    int rc = B2S_OK;
    if (e != cudaSuccess) {
        set_error("cp_apr_phi_mode: padding the factors failed: %s", cudaGetErrorString(e));
        rc = B2S_ERR_CUDA;
    } else {
        a.order = order;
        a.mode = mode;
        a.R = R;
        a.rowc = (const I *)coords[mode];
        a.vals = (const T *)vals;
        a.nnz = nnz;
        a.rows = rows;
        a.eps = eps;
        a.out = (T *)out;
        a.ldo = ldo;
        auto main = [&](T *pieces, int64_t ldp) {
            a.pieces = pieces;
            a.ldp = ldp;
            return dispatch_phi<T, I>(a, s);
        };
        auto combine = [&](T *pieces, int64_t ldp, int64_t nchunks) {
            return launch_mttkrp_combine<T, I>(a.rowc, nnz, R, pieces, ldp, nchunks, a.out, ldo, s);
        };
        rc = chunked_launches<T>("cp_apr_phi_mode", nnz, R, s, main, combine);
    }
    const int frc = padded ? scratch_free(padded, s) : B2S_OK;  // stream-ordered: after the kernels that read it
    return rc ? rc : frc;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_cp_apr_phi_max_rank(void) { return B2S_CP_APR_PHI_MAX_RANK; }

int b2s_cp_apr_phi_mode(int dtype, int idx_bytes, int order, int mode, int64_t nnz, int64_t rows, int64_t R,
                        double eps, const void *const *coords_host, const void *vals_dev,
                        const void *const *factors_host, const int64_t *ld_host, const int64_t *extents_host,
                        void *out_dev, int64_t ldo, void *stream) {
    const char *op = "cp_apr_phi_mode";
    int rc = check_tensor(op, dtype, idx_bytes, order);
    if (rc) return rc;
    B2S_REQUIRE(mode >= 0 && mode < order, B2S_ERR_INVALID, "%s: mode %d of an order-%d tensor", op, mode, order);
    B2S_REQUIRE(nnz >= 0 && rows >= 0 && R >= 0, B2S_ERR_INVALID, "%s: negative size", op);
    B2S_REQUIRE(R <= B2S_CP_APR_PHI_MAX_RANK, B2S_ERR_INVALID, "%s: R %lld above B2S_CP_APR_PHI_MAX_RANK = %d", op,
                (long long)R, B2S_CP_APR_PHI_MAX_RANK);
    const bool eps_ok = dtype == B2S_F32 ? eps >= 0 && std::isfinite((float)eps) : eps >= 0 && std::isfinite(eps);
    B2S_REQUIRE(eps_ok, B2S_ERR_INVALID, "%s: eps must be finite and >= 0 in the value type", op);
    B2S_REQUIRE(ldo >= R, B2S_ERR_INVALID, "%s: ldo < R", op);
    if (rows == 0 || R == 0) return B2S_OK;
    rc = check_factors(op, order, -1, coords_host, factors_host, ld_host, R, nullptr);
    if (rc) return rc;
    B2S_REQUIRE(extents_host != nullptr, B2S_ERR_INVALID, "%s: NULL extents", op);
    for (int m = 0; m < order; ++m)
        B2S_REQUIRE(extents_host[m] >= 0, B2S_ERR_INVALID, "%s: negative extent of mode %d", op, m);
    cudaStream_t s = (cudaStream_t)stream;
    if (nnz == 0) {
        const size_t es = dtype_size(dtype);
        B2S_CUDA(cudaMemset2DAsync(out_dev, (size_t)ldo * es, 0, (size_t)R * es, (size_t)rows, s));
        return B2S_OK;
    }
    return dispatch_tensor(dtype, idx_bytes, [&](auto t, auto i) {
        using T = decltype(t);
        return cp_apr_phi_impl<T, decltype(i)>(order, mode, nnz, rows, (int)R, (T)eps, coords_host, vals_dev,
                                               factors_host, ld_host, extents_host, out_dev, ldo, s);
    });
}

}  // extern "C"
