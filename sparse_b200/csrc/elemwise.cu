// elemwise.cu -- K5: broadcasting element-wise coiteration over sorted COO key streams.
//
// Replaces the mask enumeration of _Elemwise.get_result / _get_func_coords_data / _match_coo and the
// sort-merge join _match_arrays (sparse/numba_backend/_umath.py:457-503, 576-654, 656-751, 53-92) with ONE
// merge-path pass: both operands are streams of (linear key, value) sorted by the C-order linear index of the
// broadcast result shape; an operand that is broadcast along TRAILING axes is expanded virtually (key = k*R + r,
// r < R) so the C3 case (a:(512,512,512,64) + b:(512,512,512,1)) never materialises b's 64x expansion.
// Every position of the union gets f(a or fill_a, b or fill_b); results bitwise-equal to the output fill value
// are flagged for removal (`equivalent`, _utils.py:448-452).  Because both streams are consumed in key order the
// output is already canonical: no final sort (the reference's COO(...) -> _sort_indices, _coo/core.py:1310-1317).
//
// Also here: COO (x) scalar / unary maps and COO (x) dense-ndarray gathers (mask (True, None), _umath.py:606-608),
// and the broadcast expansion kernel for non-trailing broadcast axes (_get_expanded_coords_data, :220-277).
#include <cub/cub.cuh>
#include <limits>
#include <type_traits>

#include "common.cuh"
#include "fastdiv.cuh"

namespace b2s {

// ---- operator tables (numpy ufunc semantics) -------------------------------------------------
enum BinOp {
    OP_ADD = 0, OP_SUB = 1, OP_MUL = 2, OP_DIV = 3, OP_MAXIMUM = 4, OP_MINIMUM = 5, OP_FMAX = 6, OP_FMIN = 7,
    OP_POW = 8, OP_FLOORDIV = 9, OP_MOD = 10, OP_BAND = 11, OP_BOR = 12, OP_BXOR = 13,
    OP_NANREPLACE = 14,  // where(isnan(a), b, a): _replace_nan of the nan-reductions (_coo/common.py:293-310)
    // three-operand where(c, x, y) (_coo/common.py:533-579) as two selections and an OR of the raw bit patterns
    OP_SEL_X = 15,   // a != 0 ? b : +0
    OP_SEL_Y = 16,   // a != 0 ? +0 : b
    OP_BITOR_RAW = 17,
    // integer shifts with NumPy's out-of-range rule: a count outside [0, bits) gives 0 (or -1 for a negative a >> n)
    OP_LSHIFT = 18, OP_RSHIFT = 19,
    // predicates (bool output)
    OP_GT = 32, OP_GE = 33, OP_LT = 34, OP_LE = 35, OP_EQ = 36, OP_NE = 37, OP_LAND = 38, OP_LOR = 39, OP_LXOR = 40
};
enum UnOp {
    U_NEG = 0, U_ABS = 1, U_SQRT = 2, U_SQUARE = 3, U_SIGN = 4, U_EXP = 5, U_EXPM1 = 6, U_LOG = 7, U_LOG1P = 8,
    U_SIN = 9, U_COS = 10, U_TAN = 11, U_TANH = 12, U_SINH = 13, U_COSH = 14, U_ARCSIN = 15, U_ARCTAN = 16,
    U_FLOOR = 17, U_CEIL = 18, U_TRUNC = 19, U_RINT = 20, U_RECIP = 21, U_POS = 22, U_INVERT = 23, U_ARCSINH = 24,
    U_ARCTANH = 25, U_DEG2RAD = 26, U_RAD2DEG = 27, U_EXP2 = 28, U_LOG2 = 29, U_LOG10 = 30, U_CBRT = 31,
    // predicates
    U_ISNAN = 64, U_ISINF = 65, U_ISFINITE = 66, U_LNOT = 67, U_SIGNBIT = 68
};

template <typename T>
__device__ __forceinline__ bool is_nan(T x) {
    if constexpr (std::is_floating_point<T>::value) return x != x;
    else return false;
}

template <typename T>
__device__ __forceinline__ T raw_or(T a, T b) {
    if constexpr (sizeof(T) == 4) {
        uint32_t x, y;
        memcpy(&x, &a, 4);
        memcpy(&y, &b, 4);
        x |= y;
        T r;
        memcpy(&r, &x, 4);
        return r;
    } else {
        uint64_t x, y;
        memcpy(&x, &a, 8);
        memcpy(&y, &b, 8);
        x |= y;
        T r;
        memcpy(&r, &x, 8);
        return r;
    }
}

// Integer power by squaring with wrapping products: multiplication modulo 2^bits is associative, so this equals
// NumPy's loop bit for bit (0 ** 0 = 1).  b >= 0: the host refuses negative exponents.  Not inlined: a copy of the loop
// in each of the merge kernel's 7 unrolled items would add register spills to every integer instantiation.
template <typename T>
__device__ __noinline__ T int_pow(T a, T b) {
    T r = T(1), base = a;
    for (auto e = (typename std::make_unsigned<T>::type)b; e != 0; e >>= 1) {
        if (e & 1) r = mul_rn(r, base);
        base = mul_rn(base, base);
    }
    return r;
}

template <typename T>
__device__ __forceinline__ T bin_apply(int op, T a, T b) {
    if (op >= OP_SEL_X && op <= OP_BITOR_RAW) {
        if (op == OP_SEL_X) return a != T(0) ? b : T(0);
        if (op == OP_SEL_Y) return a != T(0) ? T(0) : b;
        return raw_or<T>(a, b);
    }
    if constexpr (std::is_floating_point<T>::value) {
        switch (op) {
            case OP_ADD: return add_rn(a, b);
            case OP_SUB: return add_rn(a, -b);
            case OP_MUL: return mul_rn(a, b);
            case OP_DIV: return a / b;
            // NaN propagates; ties (+0 vs -0) return the SECOND operand, like NumPy's x86 SIMD loops (maxpd/minpd)
            case OP_MAXIMUM: return (is_nan(a) || is_nan(b)) ? (is_nan(a) ? a : b) : (a > b ? a : b);
            case OP_MINIMUM: return (is_nan(a) || is_nan(b)) ? (is_nan(a) ? a : b) : (a < b ? a : b);
            // a NaN operand loses; of two NaNs the FIRST is returned, bits kept (NumPy: a >= b || isnan(b) ? a : b)
            case OP_FMAX: return is_nan(b) ? a : (is_nan(a) ? b : (a > b ? a : b));
            case OP_FMIN: return is_nan(b) ? a : (is_nan(a) ? b : (a < b ? a : b));
            case OP_NANREPLACE: return is_nan(a) ? b : a;
            case OP_POW: return pow(a, b);
            case OP_FLOORDIV: {
                if (b == T(0)) return a / b;
                T mod = fmod(a, b);
                T div = (a - mod) / b;
                if (mod != T(0) && ((b < T(0)) != (mod < T(0)))) div -= T(1);
                if (div != T(0)) {
                    T fl = floor(div);
                    if (div - fl > T(0.5)) fl += T(1);
                    return fl;
                }
                return copysign(T(0), a / b);
            }
            case OP_MOD: {
                if (b == T(0)) return fmod(a, b);
                T mod = fmod(a, b);
                if (mod != T(0)) {
                    if ((b < T(0)) != (mod < T(0))) mod += b;
                } else {
                    mod = copysign(T(0), b);
                }
                return mod;
            }
            default: return T(0);
        }
    } else {
        switch (op) {
            case OP_ADD: return add_rn(a, b);
            case OP_SUB: return (T)((typename std::make_unsigned<T>::type)a - (typename std::make_unsigned<T>::type)b);
            case OP_MUL: return mul_rn(a, b);
            case OP_POW: return int_pow(a, b);
            case OP_MAXIMUM: case OP_FMAX: return a >= b ? a : b;
            case OP_MINIMUM: case OP_FMIN: return a <= b ? a : b;
            case OP_FLOORDIV: {
                if (b == 0) return 0;
                T q = a / b;
                if ((a % b != 0) && ((a < 0) != (b < 0))) --q;
                return q;
            }
            case OP_MOD: {
                if (b == 0) return 0;
                T r = a % b;
                if (r != 0 && ((r < 0) != (b < 0))) r += b;
                return r;
            }
            case OP_BAND: return a & b;
            case OP_BOR: return a | b;
            case OP_BXOR: return a ^ b;
            case OP_LSHIFT: {
                using U = typename std::make_unsigned<T>::type;
                return ((U)b < (U)(8 * sizeof(T))) ? (T)((U)a << (U)b) : T(0);
            }
            case OP_RSHIFT: {
                using U = typename std::make_unsigned<T>::type;
                return ((U)b < (U)(8 * sizeof(T))) ? (T)(a >> b) : (a < 0 ? T(-1) : T(0));
            }
            case OP_NANREPLACE: return a;
            default: return T(0);
        }
    }
}

template <typename T>
__device__ __forceinline__ bool bin_pred(int op, T a, T b) {
    switch (op) {
        case OP_GT: return a > b;
        case OP_GE: return a >= b;
        case OP_LT: return a < b;
        case OP_LE: return a <= b;
        case OP_EQ: return a == b;
        case OP_NE: return a != b;
        case OP_LAND: return (a != T(0)) && (b != T(0));
        case OP_LOR: return (a != T(0)) || (b != T(0));
        case OP_LXOR: return (a != T(0)) != (b != T(0));
        default: return false;
    }
}

template <typename T>
__device__ __forceinline__ T un_apply(int op, T a) {
    if constexpr (std::is_floating_point<T>::value) {
        switch (op) {
            case U_NEG: return -a;
            case U_POS: return a;
            case U_ABS: return fabs(a);
            case U_SQRT: return sqrt(a);
            case U_SQUARE: return mul_rn(a, a);
            case U_SIGN: return is_nan(a) ? a : (a > T(0) ? T(1) : (a < T(0) ? T(-1) : T(0)));
            case U_EXP: return exp(a);
            case U_EXPM1: return expm1(a);
            case U_EXP2: return exp2(a);
            case U_LOG: return log(a);
            case U_LOG1P: return log1p(a);
            case U_LOG2: return log2(a);
            case U_LOG10: return log10(a);
            case U_SIN: return sin(a);
            case U_COS: return cos(a);
            case U_TAN: return tan(a);
            case U_TANH: return tanh(a);
            case U_SINH: return sinh(a);
            case U_COSH: return cosh(a);
            case U_ARCSIN: return asin(a);
            case U_ARCTAN: return atan(a);
            case U_ARCSINH: return asinh(a);
            case U_ARCTANH: return atanh(a);
            case U_FLOOR: return floor(a);
            case U_CEIL: return ceil(a);
            case U_TRUNC: return trunc(a);
            case U_RINT: return rint(a);
            case U_RECIP: return T(1) / a;
            case U_CBRT: return cbrt(a);
            // NumPy's constants: pi / 180 and 180 / pi rounded in T (180 / pi in float is 57.295776f, not the float
            // nearest to 180 / pi in double, 57.29578f)
            case U_DEG2RAD: { constexpr T k = T(3.14159265358979323846) / T(180); return a * k; }
            case U_RAD2DEG: { constexpr T k = T(180) / T(3.14159265358979323846); return a * k; }
            default: return T(0);
        }
    } else {
        switch (op) {
            case U_NEG: return (T)(0 - (typename std::make_unsigned<T>::type)a);
            case U_POS: return a;
            case U_ABS: return a < 0 ? (T)(0 - (typename std::make_unsigned<T>::type)a) : a;
            case U_SQUARE: return mul_rn(a, a);
            case U_SIGN: return a > 0 ? T(1) : (a < 0 ? T(-1) : T(0));
            case U_INVERT: return ~a;
            case U_FLOOR: case U_CEIL: case U_TRUNC: return a;  // NumPy >= 2 keeps the integer dtype: the identity
            // NumPy computes (T)(1.0 / a): 1 -> 1, -1 -> -1, 0 -> (T)inf, which is the minimum on x86-64, else 0
            case U_RECIP: return (a == T(1) || a == T(-1)) ? a : (a == T(0) ? std::numeric_limits<T>::min() : T(0));
            default: return T(0);
        }
    }
}

template <typename T>
__device__ __forceinline__ bool un_pred(int op, T a) {
    if constexpr (std::is_floating_point<T>::value) {
        switch (op) {
            case U_ISNAN: return a != a;
            case U_ISINF: return isinf(a);
            case U_ISFINITE: return isfinite(a);
            case U_LNOT: return a == T(0);
            case U_SIGNBIT: return signbit(a);
            default: return false;
        }
    } else {
        switch (op) {
            case U_ISFINITE: return true;
            case U_LNOT: return a == T(0);
            case U_SIGNBIT: return a < 0;
            default: return false;
        }
    }
}

template <typename O>
__device__ __forceinline__ bool bits_differ(O v, O fill) {
    if constexpr (sizeof(O) == 1) {
        uint8_t x, y;
        memcpy(&x, &v, 1);
        memcpy(&y, &fill, 1);
        return x != y;
    } else if constexpr (sizeof(O) == 4) {
        uint32_t x, y;
        memcpy(&x, &v, 4);
        memcpy(&y, &fill, 4);
        return x != y;
    } else {
        uint64_t x, y;
        memcpy(&x, &v, 8);
        memcpy(&y, &fill, 8);
        return x != y;
    }
}

// ---- virtual (trailing-broadcast) key streams ------------------------------------------------
struct Stream {
    const int64_t *keys;  // prefix keys, sorted, unique
    int64_t n;            // stored entries
    int64_t R;            // trailing expansion factor (>= 1)
    FastDiv fR;           // division by R without the 64-bit divide sequence
    __device__ __forceinline__ int64_t len() const { return n * R; }
    __device__ __forceinline__ int64_t key(int64_t p) const {
        if (R == 1) return keys[p];
        const int64_t q = (int64_t)fR.div((uint64_t)p);
        return keys[q] * R + (p - q * R);
    }
    __device__ __forceinline__ int64_t src(int64_t p) const { return R == 1 ? p : (int64_t)fR.div((uint64_t)p); }
};
static inline Stream make_stream(const int64_t *keys, int64_t n, int64_t R) {
    Stream s;
    s.keys = keys;
    s.n = n;
    s.R = R;
    s.fR = make_fastdiv((uint64_t)R);
    return s;
}

constexpr int EW_THREADS = 256;
constexpr int EW_ITEMS = 7;  // odd: per-thread merge ranges start 7 keys (56 B) apart -> no shared-memory bank conflicts
constexpr int EW_TILE = EW_THREADS * EW_ITEMS;

// merge-path split of diagonal d: number of a-items among the first d merged items (ties: a first)
__device__ __forceinline__ int64_t merge_split(const Stream &A, const Stream &B, int64_t d) {
    const int64_t la = A.len(), lb = B.len();
    int64_t lo = d > lb ? d - lb : 0;
    int64_t hi = d < la ? d : la;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (A.key(mid) <= B.key(d - 1 - mid)) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__global__ void ew_partition_kernel(Stream A, Stream B, int64_t ntiles, int64_t *__restrict__ split_a) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t > ntiles) return;
    const int64_t total = A.len() + B.len();
    int64_t d = t * EW_TILE;
    if (d > total) d = total;
    split_a[t] = merge_split(A, B, d);
}

// ---------------------------------------------------------------------------------------------------------
// Fused SINGLE-pass merge (the production path for COO (x) COO): every 1792-position tile of the merge path is
// merged, the operator applied and the kept (key, value) pairs compacted in shared memory; the tile's offset in the
// output comes from a decoupled look-back over the (status | count) words of its predecessors (Merrill & Garland,
// "Single-pass parallel prefix scan with decoupled look-back").  Tiles are taken in TICKET order (atomic counter),
// every tile publishes its own count before it waits for anything, and it only ever waits on tiles with smaller
// tickets, i.e. on CTAs that are already running -- so the wait cannot deadlock.  No (key, value, flag) temporaries
// of union size ever touch HBM and the merge runs once; coordinates are derived lazily from the keys by the caller.
// ---------------------------------------------------------------------------------------------------------
constexpr int kEwMaxDims = 16;
constexpr uint64_t LB_AGG = 1ull << 62, LB_PREFIX = 2ull << 62, LB_VALUE = (1ull << 62) - 1;
__device__ __forceinline__ uint64_t lb_load(const uint64_t *p) { return *(const volatile uint64_t *)p; }
__device__ __forceinline__ void lb_store(uint64_t *p, uint64_t v) { *(volatile uint64_t *)p = v; }

template <typename T, typename O, bool PRED>
__global__ void __launch_bounds__(EW_THREADS, 1536 / EW_THREADS)
ew_merge_fused_kernel(Stream A, Stream B, const T *__restrict__ da, const T *__restrict__ db, T fill_a, T fill_b,
                      O out_fill, int op, const int64_t *__restrict__ split_a, O *__restrict__ vals_out,
                      int64_t *__restrict__ keys_out, uint64_t *__restrict__ lb_status,
                      unsigned int *__restrict__ lb_ticket, int64_t *__restrict__ total_out) {
    __shared__ int64_t sa[EW_TILE + 2];
    __shared__ int64_t sb[EW_TILE + 2];
    __shared__ int s_warp[EW_THREADS / 32];
    __shared__ int64_t s_tile, s_base;
    const int64_t la = A.len(), lb = B.len();
    const int64_t total = la + lb;
    if (threadIdx.x == 0) s_tile = (int64_t)atomicAdd(lb_ticket, 1u);
    __syncthreads();
    const int64_t tile = s_tile;
    const int64_t d0 = tile * EW_TILE;
    const int64_t d1 = (d0 + EW_TILE < total) ? d0 + EW_TILE : total;
    const int64_t a0 = split_a[tile], a1 = split_a[tile + 1];
    const int64_t b0 = d0 - a0, b1 = d1 - a1;
    const int na = (int)(a1 - a0), nb = (int)(b1 - b0);
    constexpr int64_t NEG = INT64_MIN, POS = INT64_MAX;
    // stage both key ranges (+ one sentinel on each side); all global loads of a thread are issued before the first
    // shared-memory store so that up to 2 x EW_LD of them are in flight per thread
    constexpr int EW_LD = (EW_TILE + 2 + EW_THREADS - 1) / EW_THREADS;
    {
        int64_t ra[EW_LD], rb[EW_LD];
#pragma unroll
        for (int k = 0; k < EW_LD; ++k) {
            const int i = threadIdx.x + k * EW_THREADS;
            const int64_t pa = a0 - 1 + i, pb = b0 - 1 + i;
            ra[k] = (i < na + 2) ? ((pa < 0) ? NEG : (pa < la ? A.key(pa) : POS)) : POS;
            rb[k] = (i < nb + 2) ? ((pb < 0) ? NEG : (pb < lb ? B.key(pb) : POS)) : POS;
        }
#pragma unroll
        for (int k = 0; k < EW_LD; ++k) {
            const int i = threadIdx.x + k * EW_THREADS;
            if (i < na + 2) sa[i] = ra[k];
            if (i < nb + 2) sb[i] = rb[k];
        }
    }
    __syncthreads();
    const int64_t *ka = sa + 1, *kb = sb + 1;
    const int dloc = threadIdx.x * EW_ITEMS;
    const int dn = (int)(d1 - d0);
    int64_t rkey[EW_ITEMS];
    O rval[EW_ITEMS];
    unsigned keepmask = 0;
    if (dloc < dn) {
        int lo = dloc > nb ? dloc - nb : 0;
        int hi = dloc < na ? dloc : na;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ka[mid] <= kb[dloc - 1 - mid]) lo = mid + 1;
            else hi = mid;
        }
        int i = lo, j = dloc - lo;
#pragma unroll
        for (int it = 0; it < EW_ITEMS; ++it) {
            const int d = dloc + it;
            rkey[it] = 0;
            rval[it] = O(0);
            if (d < dn) {
                const bool take_a = (j >= nb) || (i < na && ka[i] <= kb[j]);
                int64_t key;
                T va, vb;
                bool emit = true;
                if (take_a) {
                    key = ka[i];
                    va = da[A.src(a0 + i)];
                    vb = (kb[j] == key) ? db[B.src(b0 + j)] : fill_b;
                    ++i;
                } else {
                    key = kb[j];
                    emit = (ka[i - 1] != key);
                    va = fill_a;
                    vb = db[B.src(b0 + j)];
                    ++j;
                }
                O r;
                if constexpr (PRED) r = (O)bin_pred<T>(op, va, vb);
                else r = (O)bin_apply<T>(op, va, vb);
                rkey[it] = key;
                rval[it] = r;
                if (emit && bits_differ<O>(r, out_fill)) keepmask |= 1u << it;
            }
        }
    }
    // block-wide exclusive scan of the per-thread keep counts
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int mine = __popc(keepmask);
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s_warp[w] = incl;
    __syncthreads();  // also: every thread is done reading sa / sb
    int woff = 0, tile_total = 0;
#pragma unroll
    for (int q = 0; q < EW_THREADS / 32; ++q) {
        const int c = s_warp[q];
        if (q < w) woff += c;
        tile_total += c;
    }
    // publish this tile's count as early as possible: successors can start summing while we compact
    if (threadIdx.x == 0) lb_store(&lb_status[tile], ((tile == 0 ? 2ull : 1ull) << 62) | (uint64_t)tile_total);
    // compact into shared memory (reusing the key staging arrays), then coalesced write-out
    int64_t *sk = sa;
    O *sv = reinterpret_cast<O *>(sb);
    int pos = woff + incl - mine;
#pragma unroll
    for (int it = 0; it < EW_ITEMS; ++it) {
        if (keepmask & (1u << it)) {
            sk[pos] = rkey[it];
            sv[pos] = rval[it];
            ++pos;
        }
    }
    __syncthreads();
    if (w == 0) {  // decoupled look-back: 64 predecessors per step (two per lane), nearest in lane 0
        int64_t excl = 0;
        if (tile != 0) {
            int64_t p = tile - 1;
            for (;;) {
                const int64_t i0 = p - lane, i1 = p - 32 - lane;
                uint64_t v0 = i0 >= 0 ? lb_load(&lb_status[i0]) : LB_PREFIX;  // virtual prefix 0 before tile 0
                uint64_t v1 = i1 >= 0 ? lb_load(&lb_status[i1]) : LB_PREFIX;
                while (__any_sync(0xffffffffu, (v0 >> 62) == 0)) {
                    __nanosleep(64);  // leave the issue slots to the warps that are still merging
                    if ((v0 >> 62) == 0) v0 = lb_load(&lb_status[i0]);
                }
                const unsigned pm0 = __ballot_sync(0xffffffffu, (v0 >> 62) == 2);
                int64_t c;
                unsigned done = pm0;
                if (pm0) {
                    c = lane <= __ffs(pm0) - 1 ? (int64_t)(v0 & LB_VALUE) : 0;  // up to the nearest full prefix
                } else {
                    while (__any_sync(0xffffffffu, (v1 >> 62) == 0)) {
                        __nanosleep(64);
                        if ((v1 >> 62) == 0) v1 = lb_load(&lb_status[i1]);
                    }
                    const unsigned pm1 = __ballot_sync(0xffffffffu, (v1 >> 62) == 2);
                    const int first1 = pm1 ? __ffs(pm1) - 1 : 31;
                    c = (int64_t)(v0 & LB_VALUE) + (lane <= first1 ? (int64_t)(v1 & LB_VALUE) : 0);
                    done = pm1;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
                excl += __shfl_sync(0xffffffffu, c, 0);
                if (done) break;
                p -= 64;
            }
            if (lane == 0) lb_store(&lb_status[tile], LB_PREFIX | (uint64_t)(excl + tile_total));
        }
        if (lane == 0) {
            s_base = excl;
            if (tile == (int64_t)gridDim.x - 1) *total_out = excl + tile_total;
        }
    }
    __syncthreads();
    const int64_t base = s_base;
    for (int t = threadIdx.x; t < tile_total; t += EW_THREADS) {
        vals_out[base + t] = sv[t];
        keys_out[base + t] = sk[t];
    }
}

// ---- COO (x) scalar, scalar (x) COO, unary ---------------------------------------------------
// mode: 0 = f(x, s), 1 = f(s, x), 2 = unary f(x)
template <typename T, typename O, bool PRED>
__global__ void ew_map_kernel(const T *__restrict__ x, int64_t n, T scalar, int mode, int op, O out_fill,
                              O *__restrict__ out, uint8_t *__restrict__ flags) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const T v = x[i];
        O r;
        if (mode == 2) {
            if constexpr (PRED) r = (O)un_pred<T>(op, v);
            else r = (O)un_apply<T>(op, v);
        } else {
            const T a = mode == 0 ? v : scalar, b = mode == 0 ? scalar : v;
            if constexpr (PRED) r = (O)bin_pred<T>(op, a, b);
            else r = (O)bin_apply<T>(op, a, b);
        }
        out[i] = r;
        flags[i] = bits_differ<O>(r, out_fill) ? 1 : 0;
    }
}

// ---- COO (x) dense ndarray: gather the dense operand at the (virtually expanded) coordinates ----
struct DenseIdx {
    int ndim;
    FastDiv extent[kEwMaxDims];   // result shape
    int64_t dstride[kEwMaxDims];  // element strides of the dense operand broadcast to the result shape (0 on broadcast axes)
};

template <typename T, typename O, bool PRED>
__global__ void ew_dense_kernel(Stream A, const T *__restrict__ da, const T *__restrict__ dense, DenseIdx di,
                                int swap, int op, O out_fill, int64_t *__restrict__ out_keys, O *__restrict__ out_vals,
                                uint8_t *__restrict__ flags) {
    const int64_t L = A.len();
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < L; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t key = A.key(p);
        uint64_t k = (uint64_t)key;
        int64_t off = 0;
        for (int d = di.ndim - 1; d >= 0; --d) {
            uint64_t q, r;
            di.extent[d].divmod(k, q, r);
            off += (int64_t)r * di.dstride[d];
            k = q;
        }
        const T sv = da[A.src(p)];
        const T dv = dense[off];
        const T a = swap ? dv : sv, b = swap ? sv : dv;
        O r;
        if constexpr (PRED) r = (O)bin_pred<T>(op, a, b);
        else r = (O)bin_apply<T>(op, a, b);
        out_keys[p] = key;
        out_vals[p] = r;
        flags[p] = bits_differ<O>(r, out_fill) ? 1 : 0;
    }
}

// ---- broadcast expansion for arbitrary (non-trailing) broadcast axes ---------------------------
// Every stored element is replicated over all combinations of the broadcast axes; entry e*R + r gets the key
// built from e's own coordinates on its real axes and the mixed-radix digits of r on the broadcast axes.
struct ExpandDims {
    int ndim;                       // result ndim
    int64_t stride[kEwMaxDims];     // C-order stride of the result shape
    int64_t bextent[kEwMaxDims];    // extent of broadcast axes (1 elsewhere)
    int is_bcast[kEwMaxDims];
    int src_row[kEwMaxDims];        // row of the operand's coords for real axes (-1 for axes it lacks)
};

template <typename I>
__global__ void ew_expand_kernel(const I *__restrict__ coords, int64_t row_stride, int64_t n, int64_t R,
                                 ExpandDims ed, int64_t *__restrict__ out_keys, int64_t *__restrict__ out_src) {
    const int64_t L = n * R;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < L; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e = p / R;
        int64_t r = p - e * R;
        int64_t key = 0;
        for (int d = ed.ndim - 1; d >= 0; --d) {
            int64_t c;
            if (ed.is_bcast[d]) {
                const int64_t ext = ed.bextent[d];
                const int64_t q = r / ext;
                c = r - q * ext;
                r = q;
            } else {
                c = (int64_t)coords[(int64_t)ed.src_row[d] * row_stride + e];
            }
            key += c * ed.stride[d];
        }
        out_keys[p] = key;
        out_src[p] = e;
    }
}

static unsigned ew_grid(int64_t n) {
    int64_t b = (n + 255) / 256;
    const int64_t cap = (int64_t)num_sms() * 16;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (unsigned)b;
}

template <typename T>
static T scalar_from(const void *p) {
    T v;
    memcpy(&v, p, sizeof(T));
    return v;
}

}  // namespace b2s

using namespace b2s;

#define B2S_EW_DISPATCH(dtype, pred, CALL)                                              \
    do {                                                                                \
        if (pred) {                                                                     \
            switch (dtype) {                                                            \
                case B2S_F32: { using T = float; using O = uint8_t; constexpr bool P = true; CALL; } break;   \
                case B2S_F64: { using T = double; using O = uint8_t; constexpr bool P = true; CALL; } break;  \
                case B2S_I32: { using T = int32_t; using O = uint8_t; constexpr bool P = true; CALL; } break; \
                case B2S_I64: { using T = int64_t; using O = uint8_t; constexpr bool P = true; CALL; } break; \
                default: set_error("elemwise: dtype %d", dtype); return B2S_ERR_UNSUPPORTED;                    \
            }                                                                           \
        } else {                                                                        \
            switch (dtype) {                                                            \
                case B2S_F32: { using T = float; using O = float; constexpr bool P = false; CALL; } break;     \
                case B2S_F64: { using T = double; using O = double; constexpr bool P = false; CALL; } break;   \
                case B2S_I32: { using T = int32_t; using O = int32_t; constexpr bool P = false; CALL; } break; \
                case B2S_I64: { using T = int64_t; using O = int64_t; constexpr bool P = false; CALL; } break; \
                default: set_error("elemwise: dtype %d", dtype); return B2S_ERR_UNSUPPORTED;                    \
            }                                                                           \
        }                                                                               \
    } while (0)

extern "C" {

/*
 * Single-pass form: the caller provides output buffers of `capacity` >= na*Ra + nb*Rb entries (the union can never be
 * larger); one merge kernel with a decoupled look-back writes the kept (key, value) pairs densely from offset 0 and
 * the output nnz comes back through nnz_out (one host sync).  No second merge, no scan kernel.
 */
int b2s_ew_merge_single(int dtype, int op, const int64_t *keys_a_dev, const void *data_a_dev, int64_t na, int64_t Ra,
                        const int64_t *keys_b_dev, const void *data_b_dev, int64_t nb, int64_t Rb,
                        const void *fill_a_host, const void *fill_b_host, const void *out_fill_host, int64_t capacity,
                        void *vals_out_dev, int64_t *keys_out_dev, int64_t *nnz_out, void *stream) {
    B2S_REQUIRE(nnz_out != nullptr, B2S_ERR_INVALID, "ew_merge_single: NULL nnz_out");
    B2S_REQUIRE(Ra >= 1 && Rb >= 1 && na >= 0 && nb >= 0, B2S_ERR_INVALID, "ew_merge_single: bad sizes");
    *nnz_out = 0;
    const int64_t total = na * Ra + nb * Rb;
    if (total == 0) return B2S_OK;
    B2S_REQUIRE(keys_out_dev && vals_out_dev, B2S_ERR_INVALID, "ew_merge_single: NULL output");
    B2S_REQUIRE(capacity >= total, B2S_ERR_INVALID, "ew_merge_single: capacity %lld < %lld candidates",
                (long long)capacity, (long long)total);
    const int64_t ntiles = (total + EW_TILE - 1) / EW_TILE;
    B2S_REQUIRE(ntiles < 2147483647LL, B2S_ERR_OVERFLOW, "ew_merge: too many tiles");
    cudaStream_t s = (cudaStream_t)stream;
    const Stream A = make_stream(keys_a_dev, na, Ra), B = make_stream(keys_b_dev, nb, Rb);
    int64_t *split = nullptr;
    uint64_t *status = nullptr;  // [ntiles] status words, then the ticket counter and the total
    int rc;
    if ((rc = scratch_alloc((void **)&split, (size_t)(ntiles + 1) * 8, s))) return rc;
    if ((rc = scratch_alloc((void **)&status, (size_t)(ntiles + 2) * 8, s))) return rc;
    B2S_CUDA(cudaMemsetAsync(status, 0, (size_t)(ntiles + 2) * 8, s));
    unsigned int *ticket = (unsigned int *)(status + ntiles);
    int64_t *total_dev = (int64_t *)(status + ntiles + 1);
    ew_partition_kernel<<<(unsigned)((ntiles + 1 + 127) / 128), 128, 0, s>>>(A, B, ntiles, split);
    B2S_CHECK_LAUNCH();
    const bool pred = op >= 32;
    B2S_EW_DISPATCH(dtype, pred,
                    (ew_merge_fused_kernel<T, O, P><<<(unsigned)ntiles, EW_THREADS, 0, s>>>(
                        A, B, (const T *)data_a_dev, (const T *)data_b_dev, scalar_from<T>(fill_a_host),
                        scalar_from<T>(fill_b_host), scalar_from<O>(out_fill_host), op, split, (O *)vals_out_dev,
                        keys_out_dev, status, ticket, total_dev)));
    B2S_CHECK_LAUNCH();
    int64_t total_out = 0;
    B2S_CUDA(cudaMemcpyAsync(&total_out, total_dev, 8, cudaMemcpyDeviceToHost, s));
    B2S_CUDA(cudaStreamSynchronize(s));
    scratch_free(split, s);
    scratch_free(status, s);
    *nnz_out = total_out;
    return B2S_OK;
}

/* mode 0: f(x, scalar); 1: f(scalar, x); 2: unary f(x).  op >= 32 (binary) / >= 64 (unary) -> bool output. */
int b2s_ew_map(int dtype, int op, int mode, const void *x_dev, int64_t n, const void *scalar_host,
               const void *out_fill_host, void *out_vals_dev, uint8_t *out_flags_dev, void *stream) {
    if (n == 0) return B2S_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const bool pred = (mode == 2) ? (op >= 64) : (op >= 32);
    B2S_EW_DISPATCH(dtype, pred,
                    (ew_map_kernel<T, O, P><<<ew_grid(n), 256, 0, s>>>((const T *)x_dev, n, scalar_from<T>(scalar_host),
                                                                      mode, op, scalar_from<O>(out_fill_host),
                                                                      (O *)out_vals_dev, out_flags_dev)));
    B2S_CHECK_LAUNCH();
    return B2S_OK;
}

/* COO (x) dense: dense operand addressed through element strides over the result shape (0 on broadcast axes). */
int b2s_ew_dense(int dtype, int op, int swap, const int64_t *keys_a_dev, const void *data_a_dev, int64_t na,
                 int64_t Ra, const void *dense_dev, int ndim, const int64_t *shape_host,
                 const int64_t *dense_strides_host, const void *out_fill_host, int64_t *out_keys_dev,
                 void *out_vals_dev, uint8_t *out_flags_dev, void *stream) {
    B2S_REQUIRE(ndim >= 0 && ndim <= kEwMaxDims, B2S_ERR_UNSUPPORTED, "ew_dense: ndim %d", ndim);
    const int64_t L = na * Ra;
    if (L == 0) return B2S_OK;
    cudaStream_t s = (cudaStream_t)stream;
    Stream A = make_stream(keys_a_dev, na, Ra);
    DenseIdx di{};
    di.ndim = ndim;
    for (int d = 0; d < ndim; ++d) {
        di.extent[d] = make_fastdiv((uint64_t)shape_host[d]);
        di.dstride[d] = dense_strides_host[d];
    }
    const bool pred = op >= 32;
    B2S_EW_DISPATCH(dtype, pred,
                    (ew_dense_kernel<T, O, P><<<ew_grid(L), 256, 0, s>>>(A, (const T *)data_a_dev, (const T *)dense_dev,
                                                                        di, swap, op, scalar_from<O>(out_fill_host),
                                                                        out_keys_dev, (O *)out_vals_dev,
                                                                        out_flags_dev)));
    B2S_CHECK_LAUNCH();
    return B2S_OK;
}

/* Broadcast expansion to `ndim` result axes; outputs n*R (key, source index) pairs (unsorted in general). */
int b2s_ew_expand(int idx_bytes, const void *coords_dev, int64_t row_stride, int64_t n, int ndim,
                  const int64_t *result_shape_host, const int32_t *is_bcast_host, const int32_t *src_row_host,
                  int64_t *out_keys_dev, int64_t *out_src_dev, void *stream) {
    B2S_REQUIRE(ndim >= 0 && ndim <= kEwMaxDims, B2S_ERR_UNSUPPORTED, "ew_expand: ndim %d", ndim);
    ExpandDims ed{};
    ed.ndim = ndim;
    int64_t R = 1, st = 1;
    for (int d = ndim - 1; d >= 0; --d) {
        ed.stride[d] = st;
        st *= result_shape_host[d];
        ed.is_bcast[d] = is_bcast_host[d];
        ed.src_row[d] = src_row_host[d];
        ed.bextent[d] = is_bcast_host[d] ? result_shape_host[d] : 1;
        if (is_bcast_host[d]) R *= result_shape_host[d];
    }
    const int64_t L = n * R;
    if (L == 0) return B2S_OK;
    cudaStream_t s = (cudaStream_t)stream;
    if (idx_bytes == 4)
        ew_expand_kernel<int32_t><<<ew_grid(L), 256, 0, s>>>((const int32_t *)coords_dev, row_stride, n, R, ed, out_keys_dev, out_src_dev);
    else
        ew_expand_kernel<int64_t><<<ew_grid(L), 256, 0, s>>>((const int64_t *)coords_dev, row_stride, n, R, ed, out_keys_dev, out_src_dev);
    B2S_CHECK_LAUNCH();
    return B2S_OK;
}

}  // extern "C"
