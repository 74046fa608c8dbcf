// reduce_fused.cu -- K7 production path: hand-written segmented-scan reduction over sorted COO keys.
//
// Replaces _calc_counts_invidx + ufunc.reduceat + the fill-value correction + the result's coordinate build
// (sparse/numba_backend/_coo/core.py:1601-1661, 693-723; _sparse_array.py:405-422) with ONE streaming pass:
//
//   per 2048-element tile: head flags (group id = key / n_cols changes), a segmented reduction inside every thread's
//   8 consecutive elements and a block-level segmented scan -> tile aggregate (number of heads, "contains a head",
//   value and count of the run that is still open at the tile end); the tile's carry-in comes from a decoupled
//   look-back over its predecessors' descriptors; then the thread that owns the LAST element of every run writes its
//   group id and its value with the fill-value contribution already applied (add: + fill*n_fill, multiply:
//   * fill**n_fill, others: op(v, fill) when the group is incomplete).  Results equal to the result fill value are
//   counted so the (rare) prune compaction only runs when needed.  Coordinates are derived lazily from the group ids.
//
// Traffic: n x (8 + sizeof(T)) bytes read, n_groups x (8 + sizeof(T)) written.
// Association order differs from NumPy's reduceat (itself unspecified) -> tolerance parity for float add/multiply.
#include <cub/cub.cuh>
#include <type_traits>

#include "common.cuh"
#include "fastdiv.cuh"

namespace b2s {

enum RedOp2 { RF_ADD = 0, RF_MUL = 1, RF_MAX = 2, RF_MIN = 3, RF_AND = 4, RF_OR = 5, RF_BAND = 6, RF_BOR = 7, RF_BXOR = 8,
              RF_FMAX = 9, RF_FMIN = 10 };  // NaN-ignoring (np.fmax / np.fmin: nanmax / nanmin)

constexpr int RD_THREADS = 256;
constexpr int RD_ITEMS = 8;
constexpr int RD_TILE = RD_THREADS * RD_ITEMS;

template <typename T>
__device__ __forceinline__ T red_apply(int op, T a, T b) {
    if constexpr (std::is_floating_point<T>::value) {
        switch (op) {
            case RF_ADD: return add_rn(a, b);
            case RF_MUL: return mul_rn(a, b);
            case RF_MAX: return (a != a) ? a : ((b != b) ? b : (a >= b ? a : b));  // NaN propagates (np.maximum)
            case RF_MIN: return (a != a) ? a : ((b != b) ? b : (a <= b ? a : b));
            case RF_FMAX: return (a >= b || b != b) ? a : b;  // the other operand when one is NaN
            case RF_FMIN: return (a <= b || b != b) ? a : b;
            default: return a;
        }
    } else {
        switch (op) {
            case RF_ADD: return (T)(a + b);
            case RF_MUL: return (T)(a * b);
            case RF_MAX: case RF_FMAX: return a >= b ? a : b;
            case RF_MIN: case RF_FMIN: return a <= b ? a : b;
            case RF_AND: return (T)((a != T(0)) && (b != T(0)));
            case RF_OR: return (T)((a != T(0)) || (b != T(0)));
            case RF_BAND: return (T)(a & b);
            case RF_BOR: return (T)(a | b);
            case RF_BXOR: return (T)(a ^ b);
            default: return a;
        }
    }
}

// fill-value contribution of SparseArray.reduce (_sparse_array.py:405-422).  NumPy computes fill (T) * n_fill (int64)
// and fill ** n_fill in float64 and combines them with v in float64 too, rounding to T once: for float32 the whole step
// runs in double here, unfused, so that add is bit-identical to it (and a contribution that overflows or underflows
// float32 on its own, such as 3e38 * 2 or 0.5 ** 150, still reaches the result correctly).
// b ** n for n > 0.  CUDA's pow may be an ulp or two off even where the result is exact, so a power of two base
// (fill 0.5, 2, -4, ...) is raised exactly by its exponent; that keeps results such as 0.5 * 0.5 ** 6 equal to the
// result fill 0.5 ** 7, and so pruned, as NumPy's correctly rounded pow does.
__device__ __forceinline__ double fill_pow(double b, int64_t n) {
    int e;
    const double m = frexp(b, &e);
    if (fabs(m) == 0.5) {
        // |e - 1| <= 1074, and any |k| >= 4096 already gives inf or 0: clamp n first so that k cannot overflow
        const int k = (e - 1) * (int)(n > 4096 ? 4096 : n);
        const double r = ldexp(1.0, k);
        // the sign follows NumPy's float64 exponent: from 2^53 on, (double)n is even
        return (m < 0 && n < (1ll << 53) && (n & 1)) ? -r : r;
    }
    return pow(b, (double)n);
}

template <typename T>
__device__ __forceinline__ T fill_fix(int op, T v, int64_t count, int64_t ncols, T fill) {
    const int64_t nf = ncols - count;
    if constexpr (std::is_same<T, float>::value) {
        if (op == RF_ADD) return (float)__dadd_rn((double)v, nf != 0 ? __dmul_rn((double)fill, (double)nf) : 0.0);
        if (op == RF_MUL) return (float)__dmul_rn((double)v, nf != 0 ? fill_pow((double)fill, nf) : 1.0);
    }
    if (op == RF_ADD) {
        T contrib = T(0);
        if (nf != 0) {
            if constexpr (std::is_floating_point<T>::value) contrib = mul_rn(fill, (T)nf);
            else contrib = (T)(fill * (T)nf);
        }
        return red_apply<T>(RF_ADD, v, contrib);
    }
    if (op == RF_MUL) {
        T contrib = T(1);
        if (nf != 0) {
            if constexpr (std::is_floating_point<T>::value) contrib = (T)fill_pow((double)fill, nf);
            else {
                T b = fill, r = T(1);
                int64_t e = nf;
                while (e > 0) {
                    if (e & 1) r = (T)(r * b);
                    b = (T)(b * b);
                    e >>= 1;
                }
                contrib = r;
            }
        }
        return red_apply<T>(RF_MUL, v, contrib);
    }
    return nf != 0 ? red_apply<T>(op, v, fill) : v;
}

template <typename T>
struct Run {  // state of the run that is open at some position
    int flag;     // 1 if a head lies at or before this position (within the scanned range)
    T val;
    int64_t cnt;
};

template <typename T>
__device__ __forceinline__ Run<T> run_combine(int op, const Run<T> &a, const Run<T> &b) {
    // b comes after a
    Run<T> r;
    r.flag = a.flag | b.flag;
    if (b.flag) {
        r.val = b.val;
        r.cnt = b.cnt;
    } else {
        r.val = (a.cnt == 0) ? b.val : ((b.cnt == 0) ? a.val : red_apply<T>(op, a.val, b.val));
        r.cnt = a.cnt + b.cnt;
    }
    return r;
}

template <typename T>
__device__ __forceinline__ Run<T> run_shfl_up(const Run<T> &x, int o) {
    Run<T> r;
    r.flag = __shfl_up_sync(0xffffffffu, x.flag, o);
    r.val = __shfl_up_sync(0xffffffffu, x.val, o);
    r.cnt = __shfl_up_sync(0xffffffffu, x.cnt, o);
    return r;
}

// One tile of the SINGLE-pass segmented reduction.
// Loads and stores go through shared memory so that global accesses are fully coalesced: the tile's 2048 (key, value)
// pairs are loaded with unit stride, each thread then reads its 8 consecutive pairs from a padded layout
// (index e + e/8: 2-way instead of 16-way bank conflicts), and the finished runs of the tile -- which occupy one
// contiguous range of output slots -- are staged in the same buffers and written out with unit stride.
// The carry-in of a tile (the run still open at its first element + the number of run heads before it) comes from a
// decoupled look-back over the tile descriptors of its predecessors (Merrill & Garland): tiles are taken in TICKET
// order, every tile publishes its own aggregate before it waits for anything and only ever waits on smaller tickets
// (CTAs that are already running), so the wait cannot deadlock.  The head count travels in ONE word with its status
// (aggregate / inclusive prefix), so its look-back needs no fences; the carry-in RUN only ever needs the predecessors'
// aggregates back to the nearest tile that contains a head (usually the immediate predecessor), which are published
// (payload, __threadfence, status) before that tile waits for anything.
constexpr int RD_PAD = RD_TILE + RD_TILE / 8 + 8;
__device__ __forceinline__ int rd_pad(int e) { return e + (e >> 3); }

enum : uint64_t { RD_AGG = 1ull << 62, RD_PREFIX = 2ull << 62, RD_VALUE = (1ull << 62) - 1 };
template <typename T>
struct RdDesc {  // per-tile look-back descriptors (device arrays of ntiles entries each)
    uint64_t *heads;     // (status << 62) | number of run heads: the tile's own (AGG) or the inclusive prefix (PREFIX)
    T *run_val;          // the tile's aggregate run (no carry-in): value ...
    int64_t *run_meta;   // ... and (count << 1) | "the tile contains a head"; valid once heads[] is non-zero
};

// IS_ADD: the operator is known at compile time for sums (the common case): no per-element switch
template <typename T, bool IS_ADD>
__global__ void __launch_bounds__(RD_THREADS, 4)
reduce_tile_kernel(const int64_t *__restrict__ keys, const T *__restrict__ vals, int64_t n, int64_t ncols,
                   FastDiv fcols, int op_rt, RdDesc<T> desc, unsigned int *__restrict__ ticket, T fill, int apply_fix,
                   T result_fill, int64_t *__restrict__ out_gid, T *__restrict__ out_val,
                   unsigned long long *__restrict__ counters /* [0] results equal to result_fill, [1] groups */) {
    __shared__ int64_t sk[RD_PAD];
    __shared__ T sv[RD_PAD];
    __shared__ int s_flag[RD_THREADS / 32];
    __shared__ T s_val[RD_THREADS / 32];
    __shared__ int64_t s_cnt[RD_THREADS / 32];
    __shared__ int s_heads[RD_THREADS / 32];
    __shared__ int64_t s_tile, s_hexcl, s_ccnt;
    __shared__ int s_cflag;
    __shared__ T s_cval;
    const int op = IS_ADD ? (int)RF_ADD : op_rt;
    if (threadIdx.x == 0) s_tile = (int64_t)atomicAdd(ticket, 1u);
    __syncthreads();
    const int64_t tile = s_tile;
    const int64_t tile_base = tile * RD_TILE;
    const int64_t base = tile_base + (int64_t)threadIdx.x * RD_ITEMS;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;

    // coalesced tile load: slot e holds element tile_base + e (group id, value); slot -1 / RD_TILE = neighbours
#pragma unroll
    for (int i = 0; i < RD_ITEMS; ++i) {
        const int e = threadIdx.x + i * RD_THREADS;
        const int64_t p = tile_base + e;
        int64_t gk = -1;
        T vv = T(0);
        if (p < n) {
            gk = (int64_t)fcols.div((uint64_t)keys[p]);
            vv = vals[p];
        }
        sk[rd_pad(e)] = gk;
        sv[rd_pad(e)] = vv;
    }
    __shared__ int64_t s_edge[2];
    if (threadIdx.x == 0) {
        s_edge[0] = (tile_base > 0) ? (int64_t)fcols.div((uint64_t)keys[tile_base - 1]) : -1;
        s_edge[1] = (tile_base + RD_TILE < n) ? (int64_t)fcols.div((uint64_t)keys[tile_base + RD_TILE]) : -1;
    }
    __syncthreads();

    int64_t g[RD_ITEMS];
    T v[RD_ITEMS];
    bool head[RD_ITEMS];
    const int e0 = threadIdx.x * RD_ITEMS;
    const int64_t gprev = (threadIdx.x == 0) ? s_edge[0] : sk[rd_pad(e0 - 1)];
    const int64_t gnext_thread = (threadIdx.x == RD_THREADS - 1) ? s_edge[1] : sk[rd_pad(e0 + RD_ITEMS)];
#pragma unroll
    for (int i = 0; i < RD_ITEMS; ++i) {
        const int64_t p = base + i;
        g[i] = sk[rd_pad(e0 + i)];
        v[i] = sv[rd_pad(e0 + i)];
        head[i] = (p < n) && ((p == 0) || (g[i] != (i == 0 ? gprev : g[i - 1])));
    }
    // thread summary: run still open at the end of the thread's range
    Run<T> mine;
    mine.flag = 0;
    mine.val = T(0);
    mine.cnt = 0;
    int nheads = 0;
#pragma unroll
    for (int i = 0; i < RD_ITEMS; ++i) {
        if (base + i < n) {
            if (head[i]) {
                mine.flag = 1;
                mine.val = v[i];
                mine.cnt = 1;
                ++nheads;
            } else {
                mine.val = mine.cnt == 0 ? v[i] : red_apply<T>(op, mine.val, v[i]);
                mine.cnt += 1;
            }
        }
    }
    // block-level inclusive segmented scan of the thread summaries (+ plain scan of head counts)
    Run<T> incl = mine;
    int hincl = nheads;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const Run<T> up = run_shfl_up(incl, o);
        const int hu = __shfl_up_sync(0xffffffffu, hincl, o);
        if (lane >= o) {
            incl = run_combine<T>(op, up, incl);
            hincl += hu;
        }
    }
    if (lane == 31) {
        s_flag[w] = incl.flag;
        s_val[w] = incl.val;
        s_cnt[w] = incl.cnt;
        s_heads[w] = hincl;
    }
    __syncthreads();  // (also: every thread has copied its inputs out of sk / sv)
    Run<T> wcarry;  // warps before this one, no carry-in yet
    wcarry.flag = 0;
    wcarry.val = T(0);
    wcarry.cnt = 0;
    Run<T> tile_agg = wcarry;
    int hbefore_local = 0, tile_heads = 0;
#pragma unroll
    for (int q = 0; q < RD_THREADS / 32; ++q) {
        Run<T> wq;
        wq.flag = s_flag[q];
        wq.val = s_val[q];
        wq.cnt = s_cnt[q];
        if (q < w) {
            wcarry = run_combine<T>(op, wcarry, wq);
            hbefore_local += s_heads[q];
        }
        tile_agg = run_combine<T>(op, tile_agg, wq);
        tile_heads += s_heads[q];
    }
    // publish the aggregate (tile 0: already the inclusive prefix) before waiting for anybody: run payload first,
    // then the status word that makes it visible
    if (threadIdx.x == 0) {
        *(volatile T *)&desc.run_val[tile] = tile_agg.val;
        *(volatile int64_t *)&desc.run_meta[tile] = (tile_agg.cnt << 1) | (int64_t)tile_agg.flag;
        __threadfence();
        *(volatile uint64_t *)&desc.heads[tile] = ((tile == 0 ? 2ull : 1ull) << 62) | (uint64_t)tile_heads;
    }
    // the staging buffers alias the input buffers: mark every slot empty
    for (int i = threadIdx.x; i < RD_TILE + 1; i += RD_THREADS) sk[i] = -1;
    if (w == 0) {
        Run<T> excl;
        excl.flag = 0;
        excl.val = T(0);
        excl.cnt = 0;
        int64_t hexcl = 0;
        if (tile != 0) {
            int64_t p = tile - 1;  // lane 0 looks at the nearest predecessor
            // (1) the carry-in RUN: predecessors' aggregates, nearest first, up to the nearest tile that contains a
            //     head -- almost always the immediate predecessor, so one window is the common case
            for (int64_t q = p;;) {
                const int64_t idx = q - lane;
                uint64_t hv = idx >= 0 ? *(volatile uint64_t *)&desc.heads[idx] : (uint64_t)RD_PREFIX;
                while (__any_sync(0xffffffffu, (hv >> 62) == 0)) {
                    __nanosleep(64);  // leave the issue slots to the warps that still have work
                    if ((hv >> 62) == 0) hv = *(volatile uint64_t *)&desc.heads[idx];
                }
                __threadfence();
                const int64_t meta = idx >= 0 ? *(volatile int64_t *)&desc.run_meta[idx] : 1;  // before tile 0: a head
                const unsigned fm = __ballot_sync(0xffffffffu, (meta & 1) != 0);
                const int firstf = fm ? __ffs(fm) - 1 : 31;
                Run<T> x;
                x.flag = 0;
                x.val = T(0);
                x.cnt = 0;
                if (lane <= firstf && idx >= 0) {
                    x.flag = (int)(meta & 1);
                    x.cnt = meta >> 1;
                    x.val = *(volatile T *)&desc.run_val[idx];
                }
                // ordered reduction: lane + o holds an EARLIER tile, so it goes on the left
                const int steps = firstf == 0 ? 0 : 32;
                for (int o = 1; o < steps; o <<= 1) {
                    Run<T> other;
                    other.flag = __shfl_down_sync(0xffffffffu, x.flag, o);
                    other.val = __shfl_down_sync(0xffffffffu, x.val, o);
                    other.cnt = __shfl_down_sync(0xffffffffu, x.cnt, o);
                    if (lane + o < 32) x = run_combine<T>(op, other, x);
                }
                Run<T> win;
                win.flag = __shfl_sync(0xffffffffu, x.flag, 0);
                win.val = __shfl_sync(0xffffffffu, x.val, 0);
                win.cnt = __shfl_sync(0xffffffffu, x.cnt, 0);
                excl = run_combine<T>(op, win, excl);  // this window lies before everything gathered so far
                if (fm) break;
                q -= 32;
            }
            // (2) the number of heads before this tile: single-word look-back, 64 predecessors per step
            for (;;) {
                const int64_t i0 = p - lane, i1 = p - 32 - lane;
                uint64_t v0 = i0 >= 0 ? *(volatile uint64_t *)&desc.heads[i0] : (uint64_t)RD_PREFIX;
                uint64_t v1 = i1 >= 0 ? *(volatile uint64_t *)&desc.heads[i1] : (uint64_t)RD_PREFIX;
                while (__any_sync(0xffffffffu, (v0 >> 62) == 0)) {
                    __nanosleep(64);
                    if ((v0 >> 62) == 0) v0 = *(volatile uint64_t *)&desc.heads[i0];
                }
                const unsigned pm0 = __ballot_sync(0xffffffffu, (v0 >> 62) == 2);
                int64_t c;
                unsigned done = pm0;
                if (pm0) {
                    c = lane <= __ffs(pm0) - 1 ? (int64_t)(v0 & RD_VALUE) : 0;  // up to the nearest inclusive prefix
                } else {
                    while (__any_sync(0xffffffffu, (v1 >> 62) == 0)) {
                        __nanosleep(64);
                        if ((v1 >> 62) == 0) v1 = *(volatile uint64_t *)&desc.heads[i1];
                    }
                    const unsigned pm1 = __ballot_sync(0xffffffffu, (v1 >> 62) == 2);
                    const int first1 = pm1 ? __ffs(pm1) - 1 : 31;
                    c = (int64_t)(v0 & RD_VALUE) + (lane <= first1 ? (int64_t)(v1 & RD_VALUE) : 0);
                    done = pm1;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
                hexcl += __shfl_sync(0xffffffffu, c, 0);
                if (done) break;
                p -= 64;
            }
            if (lane == 0) *(volatile uint64_t *)&desc.heads[tile] = RD_PREFIX | (uint64_t)(hexcl + tile_heads);
        }
        if (lane == 0) {
            s_hexcl = hexcl;
            s_cflag = excl.flag;
            s_cval = excl.val;
            s_ccnt = excl.cnt;
            if (tile == (int64_t)gridDim.x - 1) counters[1] = (unsigned long long)(hexcl + tile_heads);
        }
    }
    __syncthreads();
    Run<T> carry;
    carry.flag = s_cflag;
    carry.val = s_cval;
    carry.cnt = s_ccnt;
    carry = run_combine<T>(op, carry, wcarry);
    const int64_t hbefore = s_hexcl + hbefore_local;
    const int64_t slot0 = s_hexcl - 1;  // output slot of a run that started before this tile
    Run<T> prev = run_shfl_up(incl, 1);
    int hprev = __shfl_up_sync(0xffffffffu, hincl, 1);
    Run<T> st = carry;
    int64_t hcount = hbefore;  // heads strictly before this thread's first element
    if (lane > 0) {
        st = run_combine<T>(op, carry, prev);
        hcount += hprev;
    }
    T rv = st.val;
    int64_t rc = st.cnt;
#pragma unroll
    for (int i = 0; i < RD_ITEMS; ++i) {
        const int64_t p = base + i;
        if (p < n) {
            if (head[i]) {
                rv = v[i];
                rc = 1;
                ++hcount;
            } else {
                rv = rc == 0 ? v[i] : red_apply<T>(op, rv, v[i]);
                rc += 1;
            }
            const bool last = (p == n - 1) ||
                              ((i + 1 < RD_ITEMS) ? (base + i + 1 < n && head[i + 1]) : (g[i] != gnext_thread));
            if (last) {
                const int loc = (int)(hcount - 1 - slot0);  // 0 .. RD_TILE
                sk[loc] = g[i];
                sv[loc] = apply_fix ? fill_fix<T>(op, rv, rc, ncols, fill) : rv;
            }
        }
    }
    __syncthreads();
    int eq = 0;
    for (int l = threadIdx.x; l < RD_TILE + 1; l += RD_THREADS) {
        const int64_t gid = sk[l];
        if (gid >= 0) {
            const int64_t idx = slot0 + l;
            const T outv = sv[l];
            out_val[idx] = outv;
            out_gid[idx] = gid;
            bool same;
            if constexpr (sizeof(T) == 1) same = (*(const uint8_t *)&outv) == (*(const uint8_t *)&result_fill);
            else if constexpr (sizeof(T) == 4) {
                uint32_t x, y;
                memcpy(&x, &outv, 4);
                memcpy(&y, &result_fill, 4);
                same = x == y;
            } else {
                uint64_t x, y;
                memcpy(&x, &outv, 8);
                memcpy(&y, &result_fill, 8);
                same = x == y;
            }
            eq += same ? 1 : 0;
        }
    }
    eq = __reduce_add_sync(0xffffffffu, eq);
    if (lane == 0 && eq) atomicAdd(&counters[0], (unsigned long long)eq);
}

// ---------------------------------------------------------------------------------------------------------------
// Communication-free form for SHORT runs (ncols <= RD_TILE, i.e. a run never spans more than two tile boundaries):
//   pass 1  rd_count_kernel   reads the keys only and counts the run heads of every tile;
//   scan    exclusive sum of the 2048-entry tiles' head counts = the tiles' output offsets (+ the group count);
//   pass 2  rd_emit_kernel    every tile reduces the runs that START in it.  The run that is still open at the tile's end
//           is finished by one warp reading AHEAD (at most ncols - 1 elements of the following tiles); the elements in
//           front of the tile's first head belong to a run the previous tile finishes the same way and are skipped.
// No tile ever waits for another one: no look-back, no descriptors, no polling -- the single-pass kernel above spends
// most of its time at the barrier behind warp 0's look-back.
// The price is one extra pass over the keys (8 of the 16 input bytes per entry).
// ---------------------------------------------------------------------------------------------------------------
template <typename E, bool VEC>
__device__ __forceinline__ void rd_load_items(const E *__restrict__ p, int64_t first, E (&out)[RD_ITEMS]) {
    if constexpr (VEC && (RD_ITEMS * sizeof(E)) % 16 == 0) {
        constexpr int NV = (int)(RD_ITEMS * sizeof(E) / 16);
        const uint4 *src = reinterpret_cast<const uint4 *>(p + first);
        uint4 tmp[NV];
#pragma unroll
        for (int q = 0; q < NV; ++q) tmp[q] = __ldg(src + q);
        memcpy(out, tmp, sizeof(out));
    } else {
#pragma unroll
        for (int i = 0; i < RD_ITEMS; ++i) out[i] = p[first + i];
    }
}

// group ids of a thread's RD_ITEMS consecutive elements, the valid mask, the head mask (an element past the end counts
// as a head) and the group ids of the two neighbours outside the thread's range (-2: none)
template <bool VEC>
__device__ __forceinline__ void rd_thread_keys(const int64_t *__restrict__ keys, int64_t n, int64_t base,
                                               const FastDiv &fcols, int lane, int64_t (&g)[RD_ITEMS], unsigned &vm,
                                               unsigned &hm, int64_t &gnext) {
    vm = 0xFFu;
    if (base + RD_ITEMS <= n) {
        rd_load_items<int64_t, VEC>(keys, base, g);
#pragma unroll
        for (int i = 0; i < RD_ITEMS; ++i) g[i] = (int64_t)fcols.div((uint64_t)g[i]);
    } else {
        vm = 0;
#pragma unroll
        for (int i = 0; i < RD_ITEMS; ++i) {
            const int64_t p = base + i;
            g[i] = -1;
            if (p < n) {
                g[i] = (int64_t)fcols.div((uint64_t)keys[p]);
                vm |= 1u << i;
            }
        }
    }
    int64_t gprev = __shfl_up_sync(0xffffffffu, g[RD_ITEMS - 1], 1);
    gnext = __shfl_down_sync(0xffffffffu, g[0], 1);
    if (lane == 0) gprev = (base > 0 && base - 1 < n) ? (int64_t)fcols.div((uint64_t)keys[base - 1]) : -2;
    if (lane == 31) gnext = base + RD_ITEMS < n ? (int64_t)fcols.div((uint64_t)keys[base + RD_ITEMS]) : -2;
    hm = (g[0] != gprev) ? 1u : 0u;
#pragma unroll
    for (int i = 1; i < RD_ITEMS; ++i) hm |= (g[i] != g[i - 1]) ? (1u << i) : 0u;
    hm |= ~vm & 0xFFu;
}

template <bool VEC>
__global__ void __launch_bounds__(RD_THREADS)
rd_count_kernel(const int64_t *__restrict__ keys, int64_t n, FastDiv fcols, int64_t *__restrict__ tile_heads) {
    __shared__ int s_h[RD_THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t base = (int64_t)blockIdx.x * RD_TILE + (int64_t)threadIdx.x * RD_ITEMS;
    int64_t g[RD_ITEMS], gnext;
    unsigned vm, hm;
    rd_thread_keys<VEC>(keys, n, base, fcols, lane, g, vm, hm, gnext);
    int c = __popc(hm & vm);
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) s_h[w] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
#pragma unroll
        for (int q = 0; q < RD_THREADS / 32; ++q) t += s_h[q];
        tile_heads[blockIdx.x] = t;
    }
}

// value of the run that is open at some position + the GLOBAL position of its head (-1: the head lies before the range)
template <typename T>
struct RunP {
    T val;
    int64_t hp;
};
template <typename T>
__device__ __forceinline__ RunP<T> runp_combine(int op, const RunP<T> &a, const RunP<T> &b) {  // b comes after a
    RunP<T> r;
    r.hp = a.hp > b.hp ? a.hp : b.hp;
    const T both = red_apply<T>(op, a.val, b.val);
    r.val = b.hp >= 0 ? b.val : both;
    return r;
}

template <typename T, int OP, bool VEC>
__global__ void __launch_bounds__(RD_THREADS, 4)
rd_emit_kernel(const int64_t *__restrict__ keys, const T *__restrict__ vals, int64_t n, int64_t ncols, FastDiv fcols,
               int op_rt, const int64_t *__restrict__ tile_off, T fill, int apply_fix, T result_fill,
               int64_t *__restrict__ out_gid, T *__restrict__ out_val, unsigned long long *__restrict__ counters) {
    __shared__ int64_t sk[RD_TILE + 1];
    __shared__ T sv[RD_TILE + 1];
    __shared__ T s_val[RD_THREADS / 32];
    __shared__ int64_t s_hp[RD_THREADS / 32];
    __shared__ int s_heads[RD_THREADS / 32];
    const int op = OP >= 0 ? OP : op_rt;
    const int64_t tile = blockIdx.x;
    const int64_t tile_base = tile * RD_TILE;
    const int64_t base = tile_base + (int64_t)threadIdx.x * RD_ITEMS;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int64_t g[RD_ITEMS], gnext;
    T v[RD_ITEMS];
    unsigned vm, hm;
    // the value loads are issued BEFORE the keys are consumed: one round trip to memory for both arrays
    if (base + RD_ITEMS <= n) {
        rd_load_items<T, VEC>(vals, base, v);
    } else {
#pragma unroll
        for (int i = 0; i < RD_ITEMS; ++i) v[i] = (base + i < n) ? vals[base + i] : T(0);
    }
    rd_thread_keys<VEC>(keys, n, base, fcols, lane, g, vm, hm, gnext);
    const unsigned lastm = ((hm >> 1) | ((g[RD_ITEMS - 1] != gnext) ? (1u << (RD_ITEMS - 1)) : 0u)) & vm;
    const int nheads = __popc(hm & vm);
    // thread summary: the run still open at the end of the thread's range
    RunP<T> mine;
    mine.val = v[0];
    mine.hp = (hm & 1u) ? base : -1;
#pragma unroll
    for (int i = 1; i < RD_ITEMS; ++i) {
        const bool h = (hm >> i) & 1u;
        const T both = red_apply<T>(op, mine.val, v[i]);
        mine.val = h ? v[i] : both;
        mine.hp = h ? base + i : mine.hp;
    }
    // inclusive segmented scan over the warp, warp aggregates through shared memory
    RunP<T> incl = mine;
    int hincl = nheads;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        RunP<T> up;
        up.val = __shfl_up_sync(0xffffffffu, incl.val, o);
        up.hp = __shfl_up_sync(0xffffffffu, incl.hp, o);
        const int hu = __shfl_up_sync(0xffffffffu, hincl, o);
        if (lane >= o) {
            incl = runp_combine<T>(op, up, incl);
            hincl += hu;
        }
    }
    if (lane == 31) {
        s_val[w] = incl.val;
        s_hp[w] = incl.hp;
        s_heads[w] = hincl;
    }
    __syncthreads();
    RunP<T> wcarry;  // the run open in front of this warp, as far as it lies inside the tile
    wcarry.val = T(0);
    wcarry.hp = -1;
    RunP<T> tile_agg = wcarry;
    int hbefore = 0, tile_heads = 0;
    bool have_w = false, have_t = false;
#pragma unroll
    for (int q = 0; q < RD_THREADS / 32; ++q) {
        RunP<T> wq;
        wq.val = s_val[q];
        wq.hp = s_hp[q];
        if (q < w) {
            wcarry = have_w ? runp_combine<T>(op, wcarry, wq) : wq;
            have_w = true;
            hbefore += s_heads[q];
        }
        tile_agg = have_t ? runp_combine<T>(op, tile_agg, wq) : wq;
        have_t = true;
        tile_heads += s_heads[q];
    }
    for (int i = threadIdx.x; i < tile_heads; i += RD_THREADS) sk[i] = -1;
    __syncthreads();
    // second walk over the thread's elements with the carry-in.  A run whose head lies before the tile (hp < 0 after
    // the combination) is not ours: the previous tile finishes it by reading ahead.
    RunP<T> st = wcarry;
    RunP<T> prev;
    prev.val = (T)__shfl_up_sync(0xffffffffu, incl.val, 1);
    prev.hp = __shfl_up_sync(0xffffffffu, incl.hp, 1);
    const int hprev = __shfl_up_sync(0xffffffffu, hincl, 1);
    int hcount = hbefore;  // heads of the tile strictly before this thread's first element
    if (lane > 0) {
        st = have_w ? runp_combine<T>(op, st, prev) : prev;
        hcount += hprev;
    }
    T rv = st.val;
    int64_t rhp = (lane > 0 || have_w) ? st.hp : -1;
#pragma unroll
    for (int i = 0; i < RD_ITEMS; ++i) {
        const bool h = (hm >> i) & 1u;
        const T both = red_apply<T>(op, rv, v[i]);
        rv = h ? v[i] : both;
        rhp = h ? base + i : rhp;
        hcount += (hm & vm) >> i & 1u;
        if (((lastm >> i) & 1u) && rhp >= tile_base) {
            sk[hcount - 1] = g[i];
            sv[hcount - 1] = apply_fix ? fill_fix<T>(op, rv, base + i - rhp + 1, ncols, fill) : rv;
        }
    }
    // the run that is still open at the end of the tile (and started in it): warp 0 reads ahead until the group changes
    if (w == 0 && tile_heads > 0) {
        const int64_t tile_end = tile_base + RD_TILE;
        const int64_t last_g = tile_end - 1 < n ? (int64_t)fcols.div((uint64_t)keys[tile_end - 1]) : -3;
        if (tile_end < n && tile_agg.hp >= tile_base &&
            (int64_t)fcols.div((uint64_t)keys[tile_end]) == last_g) {
            T acc = tile_agg.val;
            int64_t p = tile_end;
            for (;;) {
                const int64_t q = p + lane;
                bool same = false;
                T x = T(0);
                if (q < n) {
                    same = (int64_t)fcols.div((uint64_t)keys[q]) == last_g;
                    x = vals[q];
                }
                const unsigned m = __ballot_sync(0xffffffffu, same);
                const int take = (m == 0xffffffffu) ? 32 : __ffs(~m) - 1;  // leading lanes that still belong to the run
                // ordered fold of the `take` leading values into acc (lane order = stored order)
                for (int j = 0; j < take; ++j) {
                    const T xv = __shfl_sync(0xffffffffu, x, j);
                    acc = red_apply<T>(op, acc, xv);
                }
                p += take;
                if (take < 32) break;
            }
            if (lane == 0) {
                sk[tile_heads - 1] = last_g;
                sv[tile_heads - 1] = apply_fix ? fill_fix<T>(op, acc, p - tile_agg.hp, ncols, fill) : acc;
            }
        }
    }
    __syncthreads();
    const int64_t off = tile_off[tile];
    int eq = 0;
    for (int l = threadIdx.x; l < tile_heads; l += RD_THREADS) {
        const int64_t gid = sk[l];
        if (gid >= 0) {
            const T outv = sv[l];
            out_val[off + l] = outv;
            out_gid[off + l] = gid;
            bool same;
            if constexpr (sizeof(T) == 1) same = (*(const uint8_t *)&outv) == (*(const uint8_t *)&result_fill);
            else if constexpr (sizeof(T) == 4) {
                uint32_t x, y;
                memcpy(&x, &outv, 4);
                memcpy(&y, &result_fill, 4);
                same = x == y;
            } else {
                uint64_t x, y;
                memcpy(&x, &outv, 8);
                memcpy(&y, &result_fill, 8);
                same = x == y;
            }
            eq += same ? 1 : 0;
        }
    }
    eq = __reduce_add_sync(0xffffffffu, eq);
    if (lane == 0 && eq) atomicAdd(&counters[0], (unsigned long long)eq);
}

// host side of the communication-free form; scratch: counters[2] | tile_heads i64[nt + 1] | tile_off i64[nt + 1]
template <typename T>
static int rd_twopass_t(const int64_t *keys, const void *vals, int64_t n, int64_t ncols, int op, const void *fill_host,
                        int apply_fix, const void *result_fill_host, int64_t *gid_out, void *vals_out, int64_t nt,
                        void *scratch, cudaStream_t s) {
    char *b = (char *)scratch;
    unsigned long long *counters = (unsigned long long *)b;
    int64_t *tile_heads = (int64_t *)(b + 16);
    int64_t *tile_off = tile_heads + (nt + 1);
    T fill, rfill;
    memcpy(&fill, fill_host, sizeof(T));
    memcpy(&rfill, result_fill_host, sizeof(T));
    const bool vec = (((uintptr_t)keys | (uintptr_t)vals) & 15) == 0;
    const FastDiv fd = make_fastdiv((uint64_t)ncols);
    if (vec) rd_count_kernel<true><<<(unsigned)nt, RD_THREADS, 0, s>>>(keys, n, fd, tile_heads);
    else rd_count_kernel<false><<<(unsigned)nt, RD_THREADS, 0, s>>>(keys, n, fd, tile_heads);
    B2S_CHECK_LAUNCH();
    {
        size_t tb = 0;
        void *tmp = nullptr;
        B2S_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, tile_heads, tile_off, (int)(nt + 1), s));
        int rc = scratch_alloc(&tmp, tb, s);
        if (rc) return rc;
        B2S_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, tile_heads, tile_off, (int)(nt + 1), s));
        count_launch(2);
        scratch_free(tmp, s);
        // the group count travels with the other counter: counters[1] = tile_off[nt]
        B2S_CUDA(cudaMemcpyAsync(counters + 1, tile_off + nt, 8, cudaMemcpyDeviceToDevice, s));
    }
#define B2S_RE(OPC)                                                                                                   \
    do {                                                                                                              \
        if (vec)                                                                                                      \
            rd_emit_kernel<T, OPC, true><<<(unsigned)nt, RD_THREADS, 0, s>>>(                                         \
                keys, (const T *)vals, n, ncols, fd, op, tile_off, fill, apply_fix, rfill, gid_out, (T *)vals_out,    \
                counters);                                                                                            \
        else                                                                                                          \
            rd_emit_kernel<T, OPC, false><<<(unsigned)nt, RD_THREADS, 0, s>>>(                                        \
                keys, (const T *)vals, n, ncols, fd, op, tile_off, fill, apply_fix, rfill, gid_out, (T *)vals_out,    \
                counters);                                                                                            \
    } while (0)
    switch (op) {  // the common operators are compile-time constants of their own instantiation
        case RF_ADD: B2S_RE(RF_ADD); break;
        case RF_MAX: B2S_RE(RF_MAX); break;
        case RF_MIN: B2S_RE(RF_MIN); break;
        default: B2S_RE(-1); break;
    }
#undef B2S_RE
    B2S_CHECK_LAUNCH();
    return B2S_OK;
}

template <typename T>
static int rd_single_t(const int64_t *keys, const void *vals, int64_t n, int64_t ncols, int op, const void *fill_host,
                       int apply_fix, const void *result_fill_host, int64_t *gid_out, void *vals_out, int64_t nt,
                       void *scratch, cudaStream_t s) {
    // scratch layout: counters[2] (u64) | ticket (u64 slot) | heads u64[nt] | run_meta i64[nt] | run_val T[nt] (8-B slots)
    char *b = (char *)scratch;
    unsigned long long *counters = (unsigned long long *)b;
    unsigned int *ticket = (unsigned int *)(b + 16);
    b += 24;
    RdDesc<T> d;
    d.heads = (uint64_t *)b;
    b += (size_t)nt * 8;
    d.run_meta = (int64_t *)b;
    b += (size_t)nt * 8;
    d.run_val = (T *)b;
    T fill, rfill;
    memcpy(&fill, fill_host, sizeof(T));
    memcpy(&rfill, result_fill_host, sizeof(T));
    if (op == RF_ADD)
        reduce_tile_kernel<T, true><<<(unsigned)nt, RD_THREADS, 0, s>>>(keys, (const T *)vals, n, ncols,
                                                                       make_fastdiv((uint64_t)ncols), op, d, ticket,
                                                                       fill, apply_fix, rfill, gid_out, (T *)vals_out,
                                                                       counters);
    else
        reduce_tile_kernel<T, false><<<(unsigned)nt, RD_THREADS, 0, s>>>(keys, (const T *)vals, n, ncols,
                                                                        make_fastdiv((uint64_t)ncols), op, d, ticket,
                                                                        fill, apply_fix, rfill, gid_out,
                                                                        (T *)vals_out, counters);
    B2S_CHECK_LAUNCH();
    return B2S_OK;
}

static int g_reduce_form = 0;  // 0 = by ncols, 1 = always the single-pass look-back kernel, 2 = always count / scan / emit

}  // namespace b2s

using namespace b2s;

extern "C" {

/* test hook: force one of the two forms of b2s_reduce_single (0 = choose by ncols) */
int b2s_reduce_set_form(int form) {
    g_reduce_form = (form == 1 || form == 2) ? form : 0;
    return B2S_OK;
}

/*
 * Segmented reduction of `vals` over runs of equal group id (= key / ncols) of the sorted `keys`, in ONE pass:
 * group ids and values (fill-value contribution applied when apply_fill_fix) are written densely from offset 0 into
 * caller buffers with room for `capacity` >= n entries (there cannot be more groups than entries); returns the
 * number of groups and the number of results bitwise equal to result_fill (so the caller can skip the prune
 * compaction when it is 0).  One stream sync.
 */
int b2s_reduce_single(int dtype, int op, const int64_t *keys_dev, const void *vals_dev, int64_t n, int64_t ncols,
                      const void *fill_host, int apply_fill_fix, const void *result_fill_host, int64_t capacity,
                      int64_t *gid_out_dev, void *vals_out_dev, int64_t *n_groups_out, int64_t *n_equal_fill_out,
                      void *stream) {
    B2S_REQUIRE(n_groups_out && n_equal_fill_out, B2S_ERR_INVALID, "reduce_single: NULL output");
    B2S_REQUIRE(n >= 0 && ncols >= 1, B2S_ERR_INVALID, "reduce_single: bad sizes");
    *n_groups_out = 0;
    *n_equal_fill_out = 0;
    if (n == 0) return B2S_OK;
    B2S_REQUIRE(capacity >= n && gid_out_dev && vals_out_dev, B2S_ERR_INVALID,
                "reduce_single: output capacity %lld < %lld entries", (long long)capacity, (long long)n);
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t nt = (n + RD_TILE - 1) / RD_TILE;
    B2S_REQUIRE(nt < 2147483647LL, B2S_ERR_OVERFLOW, "reduce: too many tiles");
    const size_t bytes = 24 + (size_t)(nt + 1) * 3 * 8;
    void *scratch = nullptr;
    int rc = scratch_alloc(&scratch, bytes, s);
    if (rc) return rc;
    // short runs (a group holds at most ncols entries): the communication-free count / scan / emit form; long runs: the
    // single-pass kernel with the decoupled look-back
    const bool two_pass = g_reduce_form == 0 ? (ncols <= RD_TILE) : (g_reduce_form == 2);
    if (two_pass) {
        B2S_CUDA(cudaMemsetAsync(scratch, 0, 16 + (size_t)(nt + 1) * 8, s));  // counters, head counts (+ sentinel)
        switch (dtype) {
            case B2S_F32: rc = rd_twopass_t<float>(keys_dev, vals_dev, n, ncols, op, fill_host, apply_fill_fix, result_fill_host, gid_out_dev, vals_out_dev, nt, scratch, s); break;
            case B2S_F64: rc = rd_twopass_t<double>(keys_dev, vals_dev, n, ncols, op, fill_host, apply_fill_fix, result_fill_host, gid_out_dev, vals_out_dev, nt, scratch, s); break;
            case B2S_I32: rc = rd_twopass_t<int32_t>(keys_dev, vals_dev, n, ncols, op, fill_host, apply_fill_fix, result_fill_host, gid_out_dev, vals_out_dev, nt, scratch, s); break;
            case B2S_I64: rc = rd_twopass_t<int64_t>(keys_dev, vals_dev, n, ncols, op, fill_host, apply_fill_fix, result_fill_host, gid_out_dev, vals_out_dev, nt, scratch, s); break;
            case B2S_BOOL: rc = rd_twopass_t<uint8_t>(keys_dev, vals_dev, n, ncols, op, fill_host, apply_fill_fix, result_fill_host, gid_out_dev, vals_out_dev, nt, scratch, s); break;
            default: set_error("reduce_single: dtype %d", dtype); rc = B2S_ERR_UNSUPPORTED;
        }
    } else {
    B2S_CUDA(cudaMemsetAsync(scratch, 0, 24 + (size_t)nt * 8, s));  // counters, ticket and every status word start at 0
    switch (dtype) {
        case B2S_F32: rc = rd_single_t<float>(keys_dev, vals_dev, n, ncols, op, fill_host, apply_fill_fix, result_fill_host, gid_out_dev, vals_out_dev, nt, scratch, s); break;
        case B2S_F64: rc = rd_single_t<double>(keys_dev, vals_dev, n, ncols, op, fill_host, apply_fill_fix, result_fill_host, gid_out_dev, vals_out_dev, nt, scratch, s); break;
        case B2S_I32: rc = rd_single_t<int32_t>(keys_dev, vals_dev, n, ncols, op, fill_host, apply_fill_fix, result_fill_host, gid_out_dev, vals_out_dev, nt, scratch, s); break;
        case B2S_I64: rc = rd_single_t<int64_t>(keys_dev, vals_dev, n, ncols, op, fill_host, apply_fill_fix, result_fill_host, gid_out_dev, vals_out_dev, nt, scratch, s); break;
        case B2S_BOOL: rc = rd_single_t<uint8_t>(keys_dev, vals_dev, n, ncols, op, fill_host, apply_fill_fix, result_fill_host, gid_out_dev, vals_out_dev, nt, scratch, s); break;
        default: set_error("reduce_single: dtype %d", dtype); rc = B2S_ERR_UNSUPPORTED;
    }
    }
    unsigned long long h[2] = {0, 0};
    if (rc == B2S_OK) {
        cudaError_t e = cudaMemcpyAsync(h, scratch, 16, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) {
            set_error("reduce_single: %s", cudaGetErrorString(e));
            rc = B2S_ERR_CUDA;
        }
    }
    scratch_free(scratch, s);
    *n_equal_fill_out = (int64_t)h[0];
    *n_groups_out = (int64_t)h[1];
    return rc;
}

}  // extern "C"
