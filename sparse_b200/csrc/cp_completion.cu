// cp_completion.cu -- K15: the row-wise regularised least-squares update of CP tensor completion (ALS), mode n of a
// sparse tensor of order 2..8, in a fixed order.
//
//   h_e[r] = prod_{m != n} U_m[i_m(e), r]                    the Khatri-Rao row of entry e
//   G_i = sum_{e in row i} h_e h_e^T,   b_i = sum_{e in row i} v_e h_e  (b_i is K10's mttkrp_mode row, bit for bit)
//   out[i, :] = x,  (G_i + reg I) x = b_i  by Cholesky factorisation and two triangular solves
//
// Input is K10's mode stream S_n, cut into the same chunks of B2S_MTTKRP_CHUNK entries.  One CTA owns one chunk and
// walks it in stream order, kBatch entries at a time: the CTA gathers the other modes' factor rows of the batch (16-byte
// packs under an L2 evict_last policy, or scalars when a factor is not 16-byte aligned) and forms h_e and
// p_e = ((v_e * U_a) * U_b) * ... in shared memory.  The NS = R(R+1)/2 + R accumulators of a row -- the upper triangle
// of G (h_e[r] * h_e[s], r <= s) and b (p_e[r] * 1, exact) -- are spread over the CTA's threads, KS fixed slots each,
// and added in registers in stream order.
//
// A row that starts and ends inside the chunk is solved there: its A = G + reg I and b go to shared memory and the
// CTA factorises A (right-looking, the columns' elements in parallel) and runs the two substitutions.  The first and
// the last row of a chunk may continue into the neighbouring chunk: their accumulators go to two scratch slots per
// chunk (K10's scheme, from tensor_modes.cuh), and a second kernel adds each crossing row's slots in chunk order and
// solves it.  Rows without entries are filled beforehand with the solution of reg I x = 0: +0 for reg > 0, NaN for
// reg = 0.  No atomics: the result is the order of include/sparse_b200.h, whatever the grid, and the vector and scalar
// gathers give the same bits.
#include "tensor_modes.cuh"

namespace b2s {

constexpr int kThreads = 256;
constexpr int kBatch = 32;  // entries gathered into shared memory at a time
constexpr int kMaxRank = B2S_CP_COMPLETION_MAX_RANK;

__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float sqrt_rn(float a) { return __fsqrt_rn(a); }
__device__ __forceinline__ double sqrt_rn(double a) { return __dsqrt_rn(a); }

template <typename T>
__device__ __forceinline__ T quiet_nan();
template <>
__device__ __forceinline__ float quiet_nan<float>() { return __int_as_float(0x7fffffff); }
template <>
__device__ __forceinline__ double quiet_nan<double>() { return __longlong_as_double(0x7fffffffffffffffll); }

// The shared-memory layout of one CTA (T-aligned regions first).
template <typename T, typename I>
struct Smem {
    T *hp;        // kBatch rows of 2R + 1: h_e[0..R), p_e[0..R), 1
    T *A;         // R x (R + 1): A, then L in its lower triangle
    T *b;         // R: b, then the forward-substitution partials
    T *y;         // R: y, then x
    int64_t *row; // kBatch: the batch's row indices
    I *coord;     // kMaxOther x kBatch: the batch's other-mode coordinates
    uint16_t *tab;  // NS: the hp offsets of each accumulator's two factors, lo | hi << 8

    // every region stays aligned: the T count before `row` is even, so it ends on 8 bytes for float too
    __device__ Smem(unsigned char *base, int R) {
        hp = (T *)base;
        A = hp + kBatch * (2 * R + 1);
        b = A + R * (R + 1);
        y = b + R;
        row = (int64_t *)(y + R);
        coord = (I *)(row + kBatch);
        tab = (uint16_t *)(coord + kMaxOther * kBatch);
    }
    static size_t bytes(int R) {
        const int ns = R * (R + 1) / 2 + R;
        return sizeof(T) * ((size_t)kBatch * (2 * R + 1) + (size_t)R * (R + 1) + 2 * R) + sizeof(int64_t) * kBatch +
               sizeof(I) * kMaxOther * kBatch + sizeof(uint16_t) * ns;
    }
};

// Accumulator slot t < R(R+1)/2 is G[r][s] (r <= s, the upper triangle row by row), slot R(R+1)/2 + r is b[r].  Its
// two factors in an hp row: h[r] and h[s] for G, p[r] and the 1 at 2R for b.
__device__ __forceinline__ void build_table(uint16_t *tab, int R) {
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
        int t = r * R - r * (r - 1) / 2;
        for (int s = r; s < R; ++s) tab[t++] = (uint16_t)(r | (s << 8));
        tab[R * (R + 1) / 2 + r] = (uint16_t)((R + r) | ((2 * R) << 8));
    }
}

// A (lower triangle, diagonal included) and b already in shared memory: factorise A = L L^T and solve, the order of
// include/sparse_b200.h steps 5-7; out_row[0..R) = x, or NaN when a pivot is not positive.  Every thread of the CTA
// calls it.
template <typename T>
__device__ void solve_row(T *A, T *b, T *y, const int R, T *out_row) {
    const int ld = R + 1;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    bool ok = true;
    for (int j = 0; j < R; ++j) {
        __syncthreads();
        // d = ((A_jj - L_j0 L_j0) - L_j1 L_j1) - ... was left in A[j][j] by the trailing updates, k ascending
        const T d = A[j * ld + j];
        if (!(d > T(0))) {
            ok = false;
            break;
        }
        const T ljj = sqrt_rn(d);
        for (int i = j + 1 + tid; i < R; i += blockDim.x) A[i * ld + j] = div_rn(A[i * ld + j], ljj);
        __syncthreads();
        if (tid == 0) A[j * ld + j] = ljj;
        // trailing update of the lower triangle, one subtraction per element and step: k = j ascending
        for (int i = j + 1 + warp; i < R; i += nwarps) {
            const T lij = A[i * ld + j];
            for (int l = j + 1 + lane; l <= i; l += 32) A[i * ld + l] = sub_rn(A[i * ld + l], mul_rn(lij, A[l * ld + j]));
        }
    }
    __syncthreads();
    if (!ok) {
        for (int r = tid; r < R; r += blockDim.x) out_row[r] = quiet_nan<T>();
        return;
    }
    // forward: y_j = ((b_j - L_j0 y_0) - L_j1 y_1 - ...) / L_jj; each b_i takes its subtractions in ascending j
    if (warp == 0) {
        for (int j = 0; j < R; ++j) {
            const T yj = div_rn(b[j], A[j * ld + j]);
            for (int i = j + 1 + lane; i < R; i += 32) b[i] = sub_rn(b[i], mul_rn(A[i * ld + j], yj));
            if (lane == 0) y[j] = yj;
            __syncwarp();
        }
        // backward: x_j = ((y_j - L_{j+1,j} x_{j+1}) - L_{j+2,j} x_{j+2} - ...) / L_jj, j descending, k ascending
        if (lane == 0) {
            for (int j = R - 1; j >= 0; --j) {
                T t = y[j];
                for (int k = j + 1; k < R; ++k) t = sub_rn(t, mul_rn(A[k * ld + j], y[k]));
                y[j] = div_rn(t, A[j * ld + j]);
            }
        }
        __syncwarp();
        for (int r = lane; r < R; r += 32) out_row[r] = y[r];
    }
}

// this thread's accumulators of one row into A (both triangles' lower copy: A[s][r] for slot (r, s)) and b, with
// reg added to the diagonal
template <typename T, int KS>
__device__ __forceinline__ void stage_row(const T (&acc)[KS], const uint16_t (&tb)[KS], const int ns, const int ng,
                                          const int R, const T reg, T *A, T *b) {
#pragma unroll
    for (int k = 0; k < KS; ++k) {
        const int t = threadIdx.x + k * kThreads;
        if (t < ns) {
            const int lo = tb[k] & 0xff, hi = tb[k] >> 8;
            if (t < ng) A[hi * (R + 1) + lo] = lo == hi ? add_rn(acc[k], reg) : acc[k];
            else b[lo - R] = acc[k];
        }
    }
}

// K15 main kernel: one CTA per chunk
template <typename T, typename I, int VEC, int KS>
__global__ void __launch_bounds__(kThreads, 1)
cp_completion_kernel(const OtherModes<I> om, const int n_other, const I *__restrict__ rowc, const T *__restrict__ vals,
                     const int64_t nnz, const int R, const T reg, T *__restrict__ out, const int64_t ldo,
                     T *__restrict__ pieces, const int64_t ldp) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem<T, I> sm(smem_raw, R);
    const int tid = threadIdx.x;
    const int ng = R * (R + 1) / 2, ns = ng + R, hw = 2 * R + 1;
    const ChunkSpan sp(rowc, nnz, blockIdx.x);
    const uint64_t pol = policy_evict_last();

    build_table(sm.tab, R);
    for (int e = tid; e < kBatch; e += kThreads) sm.hp[e * hw + 2 * R] = T(1);
    __syncthreads();
    uint16_t tb[KS];
    T acc[KS];
#pragma unroll
    for (int k = 0; k < KS; ++k) {
        const int t = tid + k * kThreads;
        tb[k] = t < ns ? sm.tab[t] : 0;
        acc[k] = T(0);
    }
    int64_t cur = sp.row_first;

    // a complete row is solved here, a crossing one goes to its piece row (CTA-uniform)
    auto flush = [&](int64_t r) {
        if (T *dst = sp.dest(pieces, ldp, r, (T *)nullptr, 0)) {  // nullptr: solved here
#pragma unroll
            for (int k = 0; k < KS; ++k)
                if (tid + k * kThreads < ns) dst[tid + k * kThreads] = acc[k];
            return;
        }
        __syncthreads();  // the previous row's solve has released A and b
        stage_row<T, KS>(acc, tb, ns, ng, R, reg, sm.A, sm.b);
        solve_row<T>(sm.A, sm.b, sm.y, R, out + r * ldo);
    };

    const int npk = R / VEC;  // packs per factor row
    for (int64_t b0 = sp.base; b0 < sp.end; b0 += kBatch) {
        const int n = sp.end - b0 < kBatch ? (int)(sp.end - b0) : kBatch;
        if (tid < n) {
            sm.row[tid] = (int64_t)ldg_stream(rowc + b0 + tid);
#pragma unroll
            for (int m = 0; m < kMaxOther; ++m)
                if (m < n_other) sm.coord[m * kBatch + tid] = ldg_stream(om.coord[m] + b0 + tid);
        }
        __syncthreads();
        // h_e = (U_a * U_b) * ..., p_e = ((v_e * U_a) * U_b) * ..., other modes ascending, each product rounded
        for (int t = tid; t < n * npk; t += kThreads) {
            const int e = t / npk, c0 = (t - e * npk) * VEC;
            const T v = __ldg(vals + b0 + e);
            T h[VEC], p[VEC];
#pragma unroll
            for (int m = 0; m < kMaxOther; ++m) {
                if (m < n_other) {
                    const MPack<T, VEC> f = m_load<T, VEC>(
                        (const T *)om.fac[m] + (int64_t)sm.coord[m * kBatch + e] * om.ld[m] + c0, pol);
#pragma unroll
                    for (int q = 0; q < VEC; ++q) {
                        h[q] = m == 0 ? f.v[q] : mul_rn(h[q], f.v[q]);
                        p[q] = mul_rn(m == 0 ? v : p[q], f.v[q]);
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < VEC; ++q) {
                sm.hp[e * hw + c0 + q] = h[q];
                sm.hp[e * hw + R + c0 + q] = p[q];
            }
        }
        __syncthreads();
        for (int e = 0; e < n; ++e) {
            const int64_t r = sm.row[e];
            if (r != cur) {
                flush(cur);
                cur = r;
#pragma unroll
                for (int k = 0; k < KS; ++k) acc[k] = T(0);
            }
            const T *he = sm.hp + e * hw;
#pragma unroll
            for (int k = 0; k < KS; ++k) acc[k] = add_rn(acc[k], mul_rn(he[tb[k] & 0xff], he[tb[k] >> 8]));
        }
        __syncthreads();  // the batch's shared rows are consumed
    }
    flush(cur);
}

// One CTA per chunk boundary b: the row that b owns (crossing_row) adds its NS slots into A and b, then it is solved
template <typename T, typename I>
__global__ void __launch_bounds__(kThreads, 1)
cp_completion_combine_kernel(const I *__restrict__ rowc, const int64_t nnz, const int R, const T reg,
                             const T *__restrict__ pieces, const int64_t ldp, T *__restrict__ out, const int64_t ldo) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem<T, I> sm(smem_raw, R);
    const int64_t b = (int64_t)blockIdx.x + 1;
    int64_t row, first, last;
    if (!crossing_row(rowc, nnz, b, row, first, last)) return;
    const int ng = R * (R + 1) / 2, ns = ng + R;
    build_table(sm.tab, R);
    __syncthreads();
    for (int t = threadIdx.x; t < ns; t += kThreads) {
        T acc = T(0);
        acc = add_rn(acc, pieces[first * ldp + t]);
        for (int64_t c = b; c <= last; ++c) acc = add_rn(acc, pieces[(2 * c) * ldp + t]);
        const int l = sm.tab[t] & 0xff, h = sm.tab[t] >> 8;
        if (t < ng) sm.A[h * (R + 1) + l] = l == h ? add_rn(acc, reg) : acc;
        else sm.b[l - R] = acc;
    }
    solve_row<T>(sm.A, sm.b, sm.y, R, out + row * ldo);
}

// every row of `out` (rows x R, stride ldo) = v
template <typename T>
__global__ void __launch_bounds__(kThreads) fill_rows_kernel(T *out, const int64_t rows, const int R,
                                                             const int64_t ldo, const T v) {
    const int64_t n = rows * R;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = t / R;
        out[i * ldo + (t - i * R)] = v;
    }
}

template <typename T, typename I, int VEC, int KS>
static int launch_main(const OtherModes<I> &om, int n_other, const I *rowc, const T *vals, int64_t nnz, int R, T reg,
                       T *out, int64_t ldo, T *pieces, int64_t ldp, size_t shm, cudaStream_t s) {
    auto kern = cp_completion_kernel<T, I, VEC, KS>;
    if (shm > 48 * 1024) B2S_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    kern<<<(unsigned)nchunks, kThreads, shm, s>>>(om, n_other, rowc, vals, nnz, R, reg, out, ldo, pieces, ldp);
    return B2S_OK;
}

// accumulator slots per thread from NS = R(R+1)/2 + R
template <typename T, typename I, int VEC>
static int dispatch_ks(const OtherModes<I> &om, int n_other, const I *rowc, const T *vals, int64_t nnz, int R, T reg,
                       T *out, int64_t ldo, T *pieces, int64_t ldp, size_t shm, cudaStream_t s) {
    const int ns = R * (R + 1) / 2 + R;
    if (ns <= kThreads)
        return launch_main<T, I, VEC, 1>(om, n_other, rowc, vals, nnz, R, reg, out, ldo, pieces, ldp, shm, s);
    if (ns <= 4 * kThreads)
        return launch_main<T, I, VEC, 4>(om, n_other, rowc, vals, nnz, R, reg, out, ldo, pieces, ldp, shm, s);
    static_assert((kMaxRank * (kMaxRank + 1) / 2 + kMaxRank + kThreads - 1) / kThreads <= 9, "KS 9 covers R <= 64");
    return launch_main<T, I, VEC, 9>(om, n_other, rowc, vals, nnz, R, reg, out, ldo, pieces, ldp, shm, s);
}

template <typename T, typename I>
static int cp_completion_impl(int order, int mode, int64_t nnz, int64_t rows, int R, double reg_d,
                              const void *const *coords, const void *vals_, const void *const *factors,
                              const int64_t *ld, void *out_, int64_t ldo, cudaStream_t s) {
    constexpr int VEC = 16 / sizeof(T);
    const T reg = (T)reg_d;
    T *out = (T *)out_;
    const T *vals = (const T *)vals_;
    // rows without entries: the solution of reg I x = 0
    {
        const T empty = reg > T(0) ? T(0) : (T)NAN;
        const int64_t n = rows * R;
        const int64_t blocks = (n + kThreads - 1) / kThreads;
        fill_rows_kernel<T><<<(unsigned)(blocks < 4096 ? blocks : 4096), kThreads, 0, s>>>(out, rows, R, ldo, empty);
        B2S_CHECK_LAUNCH();
    }
    if (nnz == 0) return B2S_OK;
    OtherModes<I> om{};
    int n_other = 0;
    bool aligned = R % VEC == 0;
    for (int m = 0; m < order; ++m) {
        if (m == mode) continue;
        aligned = aligned && ((uintptr_t)factors[m] & 15) == 0 && ld[m] % VEC == 0;
        om.coord[n_other] = (const I *)coords[m];
        om.fac[n_other] = factors[m];
        om.ld[n_other] = ld[m];
        ++n_other;
    }
    const I *rowc = (const I *)coords[mode];
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    B2S_REQUIRE(nchunks <= INT32_MAX, B2S_ERR_INVALID, "cp_completion_mode: nnz %lld exceeds one grid",
                (long long)nnz);
    const size_t shm = Smem<T, I>::bytes(R);
    auto main = [&](T *pieces, int64_t ldp) {
        return aligned ? dispatch_ks<T, I, VEC>(om, n_other, rowc, vals, nnz, R, reg, out, ldo, pieces, ldp, shm, s)
                       : dispatch_ks<T, I, 1>(om, n_other, rowc, vals, nnz, R, reg, out, ldo, pieces, ldp, shm, s);
    };
    auto combine = [&](T *pieces, int64_t ldp, int64_t) -> int {
        auto kern = cp_completion_combine_kernel<T, I>;
        if (shm > 48 * 1024) B2S_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
        kern<<<(unsigned)(nchunks - 1), kThreads, shm, s>>>(rowc, nnz, R, reg, pieces, ldp, out, ldo);
        return B2S_OK;
    };
    return chunked_launches<T>("cp_completion_mode", nnz, (int64_t)R * (R + 1) / 2 + R, s, main, combine);
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_cp_completion_max_rank(void) { return B2S_CP_COMPLETION_MAX_RANK; }

int b2s_cp_completion_mode(int dtype, int idx_bytes, int order, int mode, int64_t nnz, int64_t rows, int64_t R,
                           double reg, const void *const *coords_host, const void *vals_dev,
                           const void *const *factors_host, const int64_t *ld_host, void *out_dev, int64_t ldo,
                           void *stream) {
    const char *op = "cp_completion_mode";
    int rc = check_tensor(op, dtype, idx_bytes, order);
    if (rc) return rc;
    B2S_REQUIRE(mode >= 0 && mode < order, B2S_ERR_INVALID, "%s: mode %d of an order-%d tensor", op, mode, order);
    B2S_REQUIRE(nnz >= 0 && rows >= 0 && R >= 0, B2S_ERR_INVALID, "%s: negative size", op);
    B2S_REQUIRE(R <= B2S_CP_COMPLETION_MAX_RANK, B2S_ERR_INVALID, "%s: R %lld above B2S_CP_COMPLETION_MAX_RANK = %d",
                op, (long long)R, B2S_CP_COMPLETION_MAX_RANK);
    B2S_REQUIRE(reg >= 0 && reg <= 1.7976931348623157e308, B2S_ERR_INVALID, "%s: reg must be finite and >= 0", op);
    B2S_REQUIRE(ldo >= R, B2S_ERR_INVALID, "%s: ldo < R", op);
    if (rows == 0 || R == 0) return B2S_OK;
    rc = check_factors(op, order, mode, coords_host, factors_host, ld_host, R, nullptr);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    return dispatch_tensor(dtype, idx_bytes, [&](auto t, auto i) {
        return cp_completion_impl<decltype(t), decltype(i)>(order, mode, nnz, rows, (int)R, reg, coords_host, vals_dev,
                                                            factors_host, ld_host, out_dev, ldo, s);
    });
}

}  // extern "C"
