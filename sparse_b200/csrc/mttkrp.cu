// mttkrp.cu -- K10: mode-n MTTKRP and K12: mode-n TTMc of a sparse tensor of order 2..8, nnz-balanced and in a fixed
// order.
//
//   K10  out[i, r]   = sum over stored e with i_n(e) = i of  v_e * prod_{m != n} U_m[i_m(e), r]
//   K12  out[i, col] = sum over stored e with i_n(e) = i of  v_e * U_a[i_a, r_a] * U_b[i_b, r_b] * ... * U_z[i_z, r_z]
//        col = ((r_a * R_b + r_b) * R_c + r_c) ... (C order over the other modes a < b < ... < z)
//
// Input is the mode stream S_n: the tensor's entries ordered by coordinate n (stable in C order), as N coordinate
// arrays plus the values.  The stream is cut into chunks of B2S_MTTKRP_CHUNK consecutive entries; a group of G lanes
// owns one (chunk, column tile) and walks its chunk in stream order, so the work per group is the same whatever the
// slice lengths are (a 100-slice mode of a 1e8-entry tensor is as balanced as a 1e6-slice one).  Lane l of a group
// owns VEC consecutive columns; the (coordinates, value) stream is read G entries at a time and broadcast by shuffles
// (as K1 does), and the factor rows of U entries are gathered at once under an L2 evict_last policy (the factors are
// the reused operand).  Per entry a lane multiplies (((v * U_a) * U_b) * ...) * U_z over the other modes in ascending
// order, the association of the order contract.  K10 and K12 share that walk (mode_stream_walk) and differ only in
// their gathers and grid mapping:
//   K10 (Khatri-Rao): every other mode is a 16-byte pack at the lane's columns; column tiles on blockIdx.y.
//   K12 (Kronecker): the lane's VEC columns (VEC dividing R_z) share the digits r_a .. r_y, so each leading mode is one
//   scalar (the group reads the same factor rows), the prefix ((v * U_a) * ...) * U_y is formed once and multiplied by
//   one VEC pack of U_z; a flat grid with the column tiles of a chunk range adjacent.
//
// A row that starts and ends inside a chunk is written straight to `out`.  The first and the last row of a chunk may
// continue into the neighbouring chunk: their partials go to a scratch array (two slots per chunk), and a second
// kernel adds each crossing row's partials in chunk order (the chunk scheme of tensor_modes.cuh, shared with K15).
// Rows without entries are zeroed by the chunk that follows them in the stream (the last chunk zeroes the rows after
// it).  No atomics: the result is the order of include/sparse_b200.h, independent of grid size and scheduling, and
// the vector and scalar forms are bit-identical.
#include <type_traits>

#include "tensor_modes.cuh"

namespace b2s {

// K12: ranks of the leading other modes, ascending
struct TtmcRanks {
    int r[kMaxOther];
};

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

template <typename T>
__device__ __forceinline__ T stream_load(const T *p, bool reread) {
    return reread ? __ldg(p) : ldg_stream(p);  // several column tiles read the stream: keep it in L2 for the others
}

// The walk of chunk `chunk` by one G-lane group (`sub` the lane in it) for the lane's columns col0 .. col0 + VEC - 1:
// zero the empty rows before the chunk's first row (and, in the last chunk, after its last row), gather and multiply
// each entry's factor rows, add the products of a row in stream order and flush each row to `out` or to the chunk's
// two piece slots.  The n_om modes of `om` are gathered LV = KRON ? 1 : VEC columns wide at column lcol[m] of their
// factor and multiplied in ascending order.  K10 (Khatri-Rao): `om` holds every other mode, the last one included, as
// packs at col0.  K12 (Kronecker): `om` holds the leading modes, each a scalar at the lane's digit, and each add takes
// that prefix times one VEC pack of the last mode (coordinates `lastc`, factor `flast` already at the lane's columns).
// Both compute (((v * U_a) * U_b) * ...) * U_z, each product rounded.
template <typename T, typename I, int VEC, bool KRON, int G, int U, typename C>
__device__ __forceinline__ void mode_stream_walk(const OtherModes<I> &om, const C (&lcol)[kMaxOther], const int n_om,
                                                 const I *__restrict__ lastc, const T *__restrict__ flast,
                                                 const int64_t ld_last, const I *__restrict__ rowc,
                                                 const T *__restrict__ vals, const int64_t nnz, const int64_t rows,
                                                 const int64_t chunk, const int64_t nchunks, const int sub,
                                                 const int64_t col0, const bool col_ok, const bool reread,
                                                 T *__restrict__ out, const int64_t ldo, T *__restrict__ pieces,
                                                 const int64_t ldp) {
    static_assert(G >= 1 && G <= 32 && (G & (G - 1)) == 0, "G must be a power of two <= 32");
    static_assert(U <= G && G % U == 0, "U must divide G");
    constexpr int LV = KRON ? 1 : VEC;
    using Row = std::conditional_t<KRON, I, int64_t>;  // the type of a shuffled row index (K10 widens it once)
    constexpr unsigned FULL = 0xffffffffu;

    ChunkSpan sp(chunk);  // lanes past the last chunk walk an empty span, but still join the shuffles
    if (chunk < nchunks) {
        sp = ChunkSpan(rowc, nnz, chunk);
        if (col_ok) {
            m_zero_rows<T, VEC>(out, ldo, sp.prev + 1, sp.row_first, col0);
            if (sp.end == nnz) m_zero_rows<T, VEC>(out, ldo, sp.row_last + 1, rows, col0);
        }
    }
    int64_t base = sp.base;
    const int64_t end = sp.end;
    const uint64_t pol = policy_evict_last();

    T acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = T(0);
    int64_t cur = sp.row_first;

    // a row complete in the chunk goes to `out`, a crossing one to its piece row
    auto flush = [&](int64_t r) {
        if (!col_ok) return;
        m_store<T, VEC>(sp.dest(pieces + col0, ldp, r, out + col0, ldo), acc);
    };

    auto any = [&](bool p) -> bool {
        if constexpr (G == 32) return p;  // one chunk per warp: already uniform
        else return __any_sync(FULL, p);
    };

    // prefetch the first G entries of the stream
    I rc_n = 0, cz_n = 0;
    I c_n[kMaxOther];
    T v_n = T(0);
#pragma unroll
    for (int m = 0; m < kMaxOther; ++m) c_n[m] = 0;
    if (base + sub < end) {
        rc_n = stream_load(rowc + base + sub, reread);
        v_n = stream_load(vals + base + sub, reread);
        if constexpr (KRON) cz_n = stream_load(lastc + base + sub, reread);
#pragma unroll
        for (int m = 0; m < kMaxOther; ++m)
            if (m < n_om) c_n[m] = stream_load(om.coord[m] + base + sub, reread);
    }

    while (any(base < end)) {
        const I rc = rc_n, cz = cz_n;
        const T v = v_n;
        I c[kMaxOther];
#pragma unroll
        for (int m = 0; m < kMaxOther; ++m) c[m] = c_n[m];
        const int64_t rem = end - base;
        const int cnt = rem > G ? G : (rem > 0 ? (int)rem : 0);
        const int64_t nb = base + G;
        if (nb + sub < end) {  // next G entries while these are consumed
            rc_n = stream_load(rowc + nb + sub, reread);
            v_n = stream_load(vals + nb + sub, reread);
            if constexpr (KRON) cz_n = stream_load(lastc + nb + sub, reread);
#pragma unroll
            for (int m = 0; m < kMaxOther; ++m)
                if (m < n_om) c_n[m] = stream_load(om.coord[m] + nb + sub, reread);
        }
#pragma unroll 1
        for (int j = 0; j < G; j += U) {
            if (!any(j < cnt)) break;
            T p[U][LV];
            Row rr[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const T vu = __shfl_sync(FULL, v, j + u, G);
                rr[u] = (Row)__shfl_sync(FULL, rc, j + u, G);
#pragma unroll
                for (int k = 0; k < LV; ++k) p[u][k] = vu;
            }
            // (((v * U_a) * U_b) * ...) over the modes of `om` in ascending order, each product rounded
#pragma unroll
            for (int m = 0; m < kMaxOther; ++m) {
                if (m < n_om) {
                    const T *fm = (const T *)om.fac[m] + lcol[m];
                    const int64_t ldm = om.ld[m];
                    MPack<T, LV> f[U];
#pragma unroll
                    for (int u = 0; u < U; ++u) {
                        const I ix = __shfl_sync(FULL, c[m], j + u, G);
                        if (j + u < cnt && col_ok) f[u] = m_load<T, LV>(fm + (int64_t)ix * ldm, pol);
                        else {
#pragma unroll
                            for (int k = 0; k < LV; ++k) f[u].v[k] = T(0);
                        }
                    }
#pragma unroll
                    for (int u = 0; u < U; ++u)
#pragma unroll
                        for (int k = 0; k < LV; ++k) p[u][k] = mul_rn(p[u][k], f[u].v[k]);
                }
            }
            MPack<T, VEC> fz[U];  // K12: the last mode's packs
            if constexpr (KRON) {
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const I ix = __shfl_sync(FULL, cz, j + u, G);
                    if (j + u < cnt && col_ok) fz[u] = m_load<T, VEC>(flast + (int64_t)ix * ld_last, pol);
                    else {
#pragma unroll
                        for (int k = 0; k < VEC; ++k) fz[u].v[k] = T(0);
                    }
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
                    for (int k = 0; k < VEC; ++k)
                        acc[k] = add_rn(acc[k], KRON ? mul_rn(p[u][0], fz[u].v[k]) : p[u][k % LV]);
                }
            }
        }
        base = nb;
    }
    if (chunk < nchunks) flush(cur);
}

// K10: column tiles on blockIdx.y; the stream is read once, with streaming loads
template <typename T, typename I, int VEC, int G, int U>
__global__ void __launch_bounds__(256)
mttkrp_mode_kernel(const OtherModes<I> om, const int n_other, const I *__restrict__ rowc, const T *__restrict__ vals,
                   const int64_t nnz, const int64_t rows, const int64_t R, T *__restrict__ out, const int64_t ldo,
                   T *__restrict__ pieces, const int64_t ldp) {
    const int lane = threadIdx.x & 31;
    const int sub = lane & (G - 1);
    const int64_t chunk = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * (32 / G) + lane / G;
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    const int64_t col0 = ((int64_t)blockIdx.y * G + sub) * VEC;
    int64_t lcol[kMaxOther];
#pragma unroll
    for (int m = 0; m < kMaxOther; ++m) lcol[m] = col0;
    mode_stream_walk<T, I, VEC, false, G, U>(om, lcol, n_other, nullptr, nullptr, 0, rowc, vals, nnz, rows, chunk, nchunks,
                                             sub, col0, col0 < R, false, out, ldo, pieces, ldp);
}

// K12: a flat grid with the column tiles of one chunk range adjacent, so the tiles that re-read a chunk's stream
// entries run together and mostly find them in L2
template <typename T, typename I, int VEC, int G, int U>
__global__ void __launch_bounds__(256)
ttmc_mode_kernel(const OtherModes<I> lead, const TtmcRanks rk, const int n_lead, const I *__restrict__ lastc,
                 const T *__restrict__ fac_last, const int64_t ld_last, const int64_t R_last,
                 const I *__restrict__ rowc, const T *__restrict__ vals, const int64_t nnz, const int64_t rows,
                 const int64_t W, const int64_t ntiles, T *__restrict__ out, const int64_t ldo, T *__restrict__ pieces,
                 const int64_t ldp) {
    const int lane = threadIdx.x & 31;
    const int sub = lane & (G - 1);
    const int64_t tile = (int64_t)blockIdx.x % ntiles;
    const int64_t cblock = (int64_t)blockIdx.x / ntiles;
    const int64_t chunk = (cblock * (blockDim.x >> 5) + (threadIdx.x >> 5)) * (32 / G) + lane / G;
    const int64_t nchunks = (nnz + kChunk - 1) / kChunk;
    const int64_t col0 = (tile * G + sub) * VEC;
    const bool col_ok = col0 < W;

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
    mode_stream_walk<T, I, VEC, true, G, U>(lead, dig, n_lead, lastc, fac_last + rz0, ld_last, rowc, vals, nnz, rows,
                                            chunk, nchunks, sub, col0, col_ok, ntiles > 1, out, ldo, pieces,
                                            ldp);
}

// the arguments of one K10 or K12 launch
template <typename T, typename I>
struct StreamArgs {
    OtherModes<I> om;  // K10: every other mode; K12: the leading ones
    TtmcRanks rk;      // K12 only
    int n_om;
    const I *lastc;  // K12 only: the last other mode
    const T *fac_last;
    int64_t ld_last, R_last;
    const I *rowc;
    const T *vals;
    int64_t nnz, rows, W;  // W output columns: R for K10
    T *out;
    int64_t ldo;
    T *pieces;
    int64_t ldp;
};

template <typename T, typename I, int VEC, int G, int U>
static int launch_mode(const StreamArgs<T, I> &a, cudaStream_t s) {
    constexpr int chunks_per_block = 8 * (32 / G);
    const int64_t nchunks = (a.nnz + kChunk - 1) / kChunk;
    dim3 grid((unsigned)((nchunks + chunks_per_block - 1) / chunks_per_block),
              (unsigned)((a.W + (int64_t)G * VEC - 1) / ((int64_t)G * VEC)));
    mttkrp_mode_kernel<T, I, VEC, G, U><<<grid, 256, 0, s>>>(a.om, a.n_om, a.rowc, a.vals, a.nnz, a.rows, a.W, a.out,
                                                            a.ldo, a.pieces, a.ldp);
    return B2S_OK;
}

// group width from the column packs per row, as K1's dispatch_g: a narrow R puts several chunks in one warp
template <typename T, typename I, int VEC>
static int dispatch_mode(const StreamArgs<T, I> &a, cudaStream_t s) {
    const int64_t packs = (a.W + VEC - 1) / VEC;
    if (packs > 16) return launch_mode<T, I, VEC, 32, 8>(a, s);
    if (packs > 8) return launch_mode<T, I, VEC, 16, 8>(a, s);
    if (packs > 4) return launch_mode<T, I, VEC, 8, 8>(a, s);
    if (packs > 2) return launch_mode<T, I, VEC, 4, 4>(a, s);
    if (packs > 1) return launch_mode<T, I, VEC, 2, 2>(a, s);
    return launch_mode<T, I, VEC, 1, 1>(a, s);
}

template <typename T, typename I, int VEC, int G, int U>
static int launch_ttmc(const StreamArgs<T, I> &a, cudaStream_t s) {
    constexpr int chunks_per_block = 8 * (32 / G);
    const int64_t nchunks = (a.nnz + kChunk - 1) / kChunk;
    const int64_t ntiles = (a.W + (int64_t)G * VEC - 1) / ((int64_t)G * VEC);
    const int64_t blocks = (nchunks + chunks_per_block - 1) / chunks_per_block * ntiles;
    B2S_REQUIRE(blocks <= INT32_MAX, B2S_ERR_INVALID, "ttmc_mode: %lld chunks x %lld column tiles exceed one grid",
                (long long)nchunks, (long long)ntiles);
    ttmc_mode_kernel<T, I, VEC, G, U><<<(unsigned)blocks, 256, 0, s>>>(a.om, a.rk, a.n_om, a.lastc, a.fac_last,
                                                                       a.ld_last, a.R_last, a.rowc, a.vals, a.nnz,
                                                                       a.rows, a.W, ntiles, a.out, a.ldo, a.pieces,
                                                                       a.ldp);
    return B2S_OK;
}

template <typename T, typename I, int VEC>
static int dispatch_ttmc(const StreamArgs<T, I> &a, cudaStream_t s) {
    const int64_t packs = (a.W + VEC - 1) / VEC;
    // at most 16 lanes per group (two chunks per warp, 16 entries' gathers in flight): against 32 lanes, W = 256 and
    // 1024 in f32 ran 20 % faster on the H100, more than paying for twice the column tiles
    if (packs > 8) return launch_ttmc<T, I, VEC, 16, 8>(a, s);
    if (packs > 4) return launch_ttmc<T, I, VEC, 8, 8>(a, s);
    if (packs > 2) return launch_ttmc<T, I, VEC, 4, 4>(a, s);
    if (packs > 1) return launch_ttmc<T, I, VEC, 2, 2>(a, s);
    return launch_ttmc<T, I, VEC, 1, 1>(a, s);
}

// K10 (ranks NULL, W = R) or K12 (W = the product of the other modes' ranks): the mode-stream kernel, then the
// combine of the rows that cross chunks
template <typename T, typename I>
static int mode_stream_impl(const char *op, int order, int mode, int64_t nnz, int64_t rows, const int64_t *ranks,
                            int64_t W, const void *const *coords, const void *vals, const void *const *factors,
                            const int64_t *ld, void *out, int64_t ldo, cudaStream_t s) {
    constexpr int VEC = 16 / sizeof(T);
    const bool kron = ranks != nullptr;
    const int last = mode == order - 1 ? order - 2 : order - 1;  // the last other mode
    StreamArgs<T, I> a{};
    a.R_last = kron ? ranks[last] : W;
    // the vector path needs every factor gathered as VEC packs 16-byte aligned: K10 all, K12 the last one
    bool aligned = a.R_last % VEC == 0 && ldo % VEC == 0 && ((uintptr_t)out & 15) == 0;
    for (int m = 0; m < order; ++m) {
        if (m == mode) continue;
        if (!kron || m == last) aligned = aligned && ((uintptr_t)factors[m] & 15) == 0 && ld[m] % VEC == 0;
        if (kron && m == last) continue;
        a.om.coord[a.n_om] = (const I *)coords[m];
        a.om.fac[a.n_om] = factors[m];
        a.om.ld[a.n_om] = ld[m];
        if (kron) a.rk.r[a.n_om] = (int)ranks[m];
        ++a.n_om;
    }
    a.lastc = (const I *)coords[last];
    a.fac_last = (const T *)factors[last];
    a.ld_last = ld[last];
    a.rowc = (const I *)coords[mode];
    a.vals = (const T *)vals;
    a.nnz = nnz;
    a.rows = rows;
    a.W = W;
    a.out = (T *)out;
    a.ldo = ldo;
    auto main = [&](T *pieces, int64_t ldp) {
        a.pieces = pieces;
        a.ldp = ldp;
        if (kron) return aligned ? dispatch_ttmc<T, I, VEC>(a, s) : dispatch_ttmc<T, I, 1>(a, s);
        return aligned ? dispatch_mode<T, I, VEC>(a, s) : dispatch_mode<T, I, 1>(a, s);
    };
    auto combine = [&](T *pieces, int64_t ldp, int64_t nchunks) {
        return launch_mttkrp_combine<T, I>(a.rowc, nnz, W, pieces, ldp, nchunks, a.out, ldo, s);
    };
    return chunked_launches<T>(op, nnz, W, s, main, combine);
}

// what b2s_mttkrp_mode and b2s_ttmc_mode do after their own checks
static int mode_stream_entry(const char *op, int dtype, int idx_bytes, int order, int mode, int64_t nnz, int64_t rows,
                             const int64_t *ranks, int64_t W, const void *const *coords, const void *vals,
                             const void *const *factors, const int64_t *ld, void *out, int64_t ldo, void *stream) {
    if (rows == 0 || W == 0) return B2S_OK;
    const int rc = check_factors(op, order, mode, coords, factors, ld, W, ranks);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const size_t es = dtype_size(dtype);
    if (nnz == 0) {
        B2S_CUDA(cudaMemset2DAsync(out, (size_t)ldo * es, 0, (size_t)W * es, (size_t)rows, s));
        return B2S_OK;
    }
    return dispatch_tensor(dtype, idx_bytes, [&](auto t, auto i) {
        return mode_stream_impl<decltype(t), decltype(i)>(op, order, mode, nnz, rows, ranks, W, coords, vals, factors,
                                                          ld, out, ldo, s);
    });
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_mttkrp_mode_chunk(void) { return B2S_MTTKRP_CHUNK; }

int b2s_mttkrp_mode(int dtype, int idx_bytes, int order, int mode, int64_t nnz, int64_t rows, int64_t R,
                    const void *const *coords_host, const void *vals_dev, const void *const *factors_host,
                    const int64_t *ld_host, void *out_dev, int64_t ldo, void *stream) {
    const char *op = "mttkrp_mode";
    const int rc = check_tensor(op, dtype, idx_bytes, order);
    if (rc) return rc;
    B2S_REQUIRE(mode >= 0 && mode < order, B2S_ERR_INVALID, "%s: mode %d of an order-%d tensor", op, mode, order);
    B2S_REQUIRE(nnz >= 0 && rows >= 0 && R >= 0, B2S_ERR_INVALID, "%s: negative size", op);
    B2S_REQUIRE(ldo >= R, B2S_ERR_INVALID, "%s: ldo < R", op);
    return mode_stream_entry(op, dtype, idx_bytes, order, mode, nnz, rows, nullptr, R, coords_host, vals_dev,
                             factors_host, ld_host, out_dev, ldo, stream);
}

int b2s_ttmc_mode_max_width(void) { return B2S_TTMC_MAX_W; }

int b2s_ttmc_mode(int dtype, int idx_bytes, int order, int mode, int64_t nnz, int64_t rows, const int64_t *ranks_host,
                  const void *const *coords_host, const void *vals_dev, const void *const *factors_host,
                  const int64_t *ld_host, void *out_dev, int64_t ldo, void *stream) {
    const char *op = "ttmc_mode";
    const int rc = check_tensor(op, dtype, idx_bytes, order);
    if (rc) return rc;
    B2S_REQUIRE(mode >= 0 && mode < order, B2S_ERR_INVALID, "%s: mode %d of an order-%d tensor", op, mode, order);
    B2S_REQUIRE(nnz >= 0 && rows >= 0, B2S_ERR_INVALID, "%s: negative size", op);
    B2S_REQUIRE(ranks_host != nullptr, B2S_ERR_INVALID, "%s: NULL ranks", op);
    int64_t W = 1;
    for (int m = 0; m < order; ++m) {
        if (m == mode) continue;
        B2S_REQUIRE(ranks_host[m] >= 0, B2S_ERR_INVALID, "%s: negative rank of mode %d", op, m);
        if (ranks_host[m] == 0) W = 0;
        else if (W > 0) W = W > B2S_TTMC_MAX_W / ranks_host[m] ? B2S_TTMC_MAX_W + 1 : W * ranks_host[m];
    }
    B2S_REQUIRE(W <= B2S_TTMC_MAX_W, B2S_ERR_INVALID, "%s: width above B2S_TTMC_MAX_W = %d", op, B2S_TTMC_MAX_W);
    B2S_REQUIRE(ldo >= W, B2S_ERR_INVALID, "%s: ldo < W", op);
    return mode_stream_entry(op, dtype, idx_bytes, order, mode, nnz, rows, ranks_host, W, coords_host, vals_dev,
                             factors_host, ld_host, out_dev, ldo, stream);
}

}  // extern "C"
