// core.h -- per-cluster consensus algorithms of the cuteSV hot path, written once over a "team"
// abstraction (a warp, a CTA, or -- in the CPU emulation used only by tests -- a single thread).
//
// Compiled by nvcc into the product kernels (cutesv_b200.cu) and by g++ into the test-only
// emulator (tests/emul/emul.cpp) which checks the *logic* against the oracle without a GPU.
// Reference citations: "cuteSV:N" = src/cuteSV/cuteSV line N; other files relative to src/cuteSV/.
//
// Floating point: every fp64 expression below must round exactly like CPython/numpy; build with
// -fmad=false (nvcc) / -ffp-contract=off (g++).
#pragma once
#include <stdint.h>
#include <math.h>
#include "../../include/cutesv_b200.h"

#ifdef __CUDACC__
#define CSV_HD __host__ __device__ __forceinline__
#define CSV_D __device__ __forceinline__
#else
#define CSV_HD inline
#define CSV_D inline
#endif

namespace csv {

// ------------------------------------------------------------------------------------------
// atomics (device) / plain ops (single-threaded emulation)
// ------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
CSV_D uint32_t atomic_add_u32(uint32_t* p, uint32_t v) { return atomicAdd(p, v); }
CSV_D int32_t atomic_add_i32(int32_t* p, int32_t v) { return atomicAdd(p, v); }
CSV_D void atomic_or_u32(uint32_t* p, uint32_t v) { atomicOr(p, v); }
CSV_D void atomic_max_u32(uint32_t* p, uint32_t v) { atomicMax(p, v); }
#else
inline uint32_t atomic_add_u32(uint32_t* p, uint32_t v) { uint32_t o = *p; *p += v; return o; }
inline int32_t atomic_add_i32(int32_t* p, int32_t v) { int32_t o = *p; *p += v; return o; }
inline void atomic_or_u32(uint32_t* p, uint32_t v) { *p |= v; }
inline void atomic_max_u32(uint32_t* p, uint32_t v) { if (v > *p) *p = v; }
#endif

// Team policies.  SIZE threads cooperate; tid() in [0, SIZE); sync() is a barrier + memory fence
// for the team's shared arena.
struct HostTeam {
    static constexpr int SIZE = 1;
    CSV_HD int tid() const { return 0; }
    CSV_HD void sync() const {}
};
#ifdef __CUDACC__
template <int N>
struct CudaTeam {
    static constexpr int SIZE = N;
    __device__ __forceinline__ int tid() const { return N == 32 ? (int)(threadIdx.x & 31) : (int)threadIdx.x; }
    __device__ __forceinline__ void sync() const {
        if (N == 32) __syncwarp(); else __syncthreads();
    }
};
#endif

// status word bits written by kernels (csv_ctx reports them as CSV_E_INPUT / internal errors)
enum : uint32_t {
    ST_BAD_CHROM = 1u, ST_BAD_POS = 2u, ST_NEG_FIELD = 4u, ST_POW_TABLE = 8u, ST_CAND_OVERFLOW = 16u,
    ST_NAMES_OVERFLOW = 32u, ST_LIST_OVERFLOW = 64u, ST_INTERNAL = 128u, ST_UNSORTED = 256u, ST_BIG_RUN = 512u, ST_SKIPPED = 1024u,
    ST_BAD_GROUPS = 2048u   // contig_off of a grouped upload from device memory is not 0 .. n non-decreasing
};

// counters block in device memory (one per csv_cluster call)
struct Counters {
    uint32_t status;        // ST_* bits
    uint32_t n_cand;        // candidates emitted (temp order)
    uint32_t n_names;       // names buffer fill
    uint32_t max_support;   // largest allele support seen (pow table sizing)
    uint32_t n_kept[CSV_NTYPES];   // kept chain clusters per type
    uint32_t n_big[CSV_NTYPES];    // deferred to the CTA-sized team
    uint32_t n_giant[CSV_NTYPES];  // deferred to the global-scratch team
    uint32_t n_windows;     // (read, window) pairs of the genotype pass
    uint32_t n_dom[CSV_NTYPES];    // size of the sorted domain per type when only the device knows it
                                   // (INDEL: survivors of the density filter; others: after duplicate removal)
    uint32_t n_members[CSV_NTYPES]; // signatures inside kept chain clusters (roofline accounting)
    uint32_t pad[2];
};

struct Limits {
    uint32_t cap_cand, cap_names, pow_n;
};

// Everything a cluster routine needs to emit rows.
struct Emit {
    csv_cand* cand;         // temp-order candidate records
    int32_t* names;         // names buffer
    uint32_t* cnt;          // per kept-cluster candidate count (indexed by global kept slot)
    Counters* ctr;
    const double* pow_half; // pow_half[n] = n ** 0.5 as libm pow evaluates it (cal_CIPOS)
    Limits lim;
    // Append cursor, (candidates << 32) | names, in a cache line of its own: ONE returning atomic per emitted row.  (Two
    // atomics per row on ctr->n_cand / n_names + an atomicMax on ctr->max_support, all in the Counters line, serialise at
    // one L2 slice -- that, not the arithmetic, was the floor of the cluster kernels.)
    // null: the counters themselves are the cursor (single-threaded emulator).
    unsigned long long* cursor;
};

// ------------------------------------------------------------------------------------------
// team primitives (all over the team's shared arena; `red` has SIZE+1 int64 slots)
// ------------------------------------------------------------------------------------------
CSV_HD int pow2ceil(int n) { int p = 1; while (p < n) p <<= 1; return p; }

template <class Team>
CSV_HD int64_t team_sum(Team tm, int64_t v, int64_t* red) {
#if defined(__CUDA_ARCH__)
    if (Team::SIZE == 32) {  // warp team: shuffles, no shared memory round trips
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    }
#endif
    const int t = tm.tid();
    red[t] = v;
    tm.sync();
    for (int s = Team::SIZE / 2; s > 0; s >>= 1) {
        if (t < s) red[t] += red[t + s];
        tm.sync();
    }
    int64_t r = red[0];
    tm.sync();
    return r;
}
template <class Team>
CSV_HD int64_t team_min(Team tm, int64_t v, int64_t* red) {
#if defined(__CUDA_ARCH__)
    if (Team::SIZE == 32) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { const int64_t y = __shfl_xor_sync(0xffffffffu, v, o); if (y < v) v = y; }
        return v;
    }
#endif
    const int t = tm.tid();
    red[t] = v;
    tm.sync();
    for (int s = Team::SIZE / 2; s > 0; s >>= 1) {
        if (t < s) { if (red[t + s] < red[t]) red[t] = red[t + s]; }
        tm.sync();
    }
    int64_t r = red[0];
    tm.sync();
    return r;
}
template <class Team>
CSV_HD int64_t team_bcast(Team tm, int64_t v, int src, int64_t* red) {
    if (tm.tid() == src) red[0] = v;
    tm.sync();
    int64_t r = red[0];
    tm.sync();
    return r;
}
// in-place exclusive scan of arr[0..n); returns the total
template <class Team>
CSV_HD uint32_t team_excl_scan(Team tm, uint32_t* arr, int n, int64_t* red) {
    const int t = tm.tid();
    const int chunk = (n + Team::SIZE - 1) / Team::SIZE;
    int lo = t * chunk; if (lo > n) lo = n;
    int hi = lo + chunk; if (hi > n) hi = n;
    uint32_t s = 0;
    for (int i = lo; i < hi; i++) s += arr[i];
#if defined(__CUDA_ARCH__)
    if (Team::SIZE == 32) {
        uint32_t incl = s;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, incl, d); if (t >= d) incl += y; }
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        uint32_t run = incl - s;
        for (int i = lo; i < hi; i++) { uint32_t x = arr[i]; arr[i] = run; run += x; }
        tm.sync();
        return total;
    }
#endif
    red[t] = s;
    tm.sync();
    if (t == 0) {
        int64_t run = 0;
        for (int k = 0; k < Team::SIZE; k++) { int64_t x = red[k]; red[k] = run; run += x; }
        red[Team::SIZE] = run;
    }
    tm.sync();
    uint32_t run = (uint32_t)red[t];
    for (int i = lo; i < hi; i++) { uint32_t x = arr[i]; arr[i] = run; run += x; }
    uint32_t total = (uint32_t)red[Team::SIZE];
    tm.sync();
    return total;
}

// in-place exclusive scan of a 0/1 flag array; returns the number of set flags
template <class Team>
CSV_HD uint32_t team_flag_scan(Team tm, uint32_t* arr, int n, int64_t* red) {
#if defined(__CUDA_ARCH__)
    if (Team::SIZE == 32) {  // warp team: one ballot per 32 flags
        const int lane = tm.tid();
        uint32_t run = 0;
        for (int base = 0; base < n; base += 32) {
            const int i = base + lane;
            const bool f = i < n && arr[i] != 0;
            const uint32_t mask = __ballot_sync(0xffffffffu, f);
            if (i < n) arr[i] = run + (uint32_t)__popc(mask & ((1u << lane) - 1u));
            run += (uint32_t)__popc(mask);
        }
        __syncwarp();
        return run;
    }
#endif
    return team_excl_scan(tm, arr, n, red);
}

struct alignas(16) K128 { uint64_t hi, lo; };
CSV_HD bool k128_gt(const K128& a, const K128& b) { return a.hi > b.hi || (a.hi == b.hi && a.lo > b.lo); }

#if defined(__CUDA_ARCH__)
// Warp-team bitonic sort held in registers: element i = e*32 + lane lives in register slot e of its
// lane.  Exchange distances < 32 are butterfly shuffles (every lane busy, no shared-memory round
// trips); distances >= 32 are register-to-register inside the lane with a direction known at compile
// time.  KW = key width in 64-bit words (1: `hi` only), HASV = carry a 32-bit payload.  All keys in
// this file are unique (an index is part of every key), so any correct sort gives the same result
// as the shared-memory version below.
template <int E, int KW, bool HASV>
__device__ __noinline__ void warp_sort_regs(uint64_t* a, uint32_t* v, int M) {
    const int lane = (int)(threadIdx.x & 31);
    uint64_t hi[E], lo[E];
    uint32_t pv[E];
#pragma unroll
    for (int e = 0; e < E; e++) {
        const int i = e * 32 + lane;
        if (i < M) {
            if (KW == 2) { const ulonglong2 x = *reinterpret_cast<const ulonglong2*>(a + 2 * i); hi[e] = x.x; lo[e] = x.y; }
            else { hi[e] = a[i]; lo[e] = 0; }
            pv[e] = HASV ? v[i] : 0u;
        } else { hi[e] = ~0ull; lo[e] = ~0ull; pv[e] = 0u; }
    }
    // one butterfly stage at distance j < 32 inside blocks of size k (rolled: the code stays small enough
    // for the instruction cache; j and k are warp-uniform run-time values)
    auto shuffle_stage = [&](int k, int j) {
        const bool lower = (lane & j) == 0;
#pragma unroll
        for (int e = 0; e < E; e++) {
            const bool up = (((e * 32 + lane) & k) == 0);
            const uint64_t ohi = __shfl_xor_sync(0xffffffffu, hi[e], j);
            const uint64_t olo = KW == 2 ? __shfl_xor_sync(0xffffffffu, lo[e], j) : 0ull;
            const uint32_t opv = HASV ? __shfl_xor_sync(0xffffffffu, pv[e], j) : 0u;
            const bool gt = hi[e] > ohi || (KW == 2 && hi[e] == ohi && lo[e] > olo);
            const bool lt = hi[e] < ohi || (KW == 2 && hi[e] == ohi && lo[e] < olo);
            // the lower index keeps the minimum in an ascending region, the maximum otherwise
            const bool take = (lower == up) ? gt : lt;
            if (take) { hi[e] = ohi; if (KW == 2) lo[e] = olo; if (HASV) pv[e] = opv; }
        }
    };
    const int kmax = M < 32 ? M : 32;   // M < 32: the padding lanes already hold all-ones and never move
#pragma unroll 1
    for (int k = 2; k <= kmax; k <<= 1) {
#pragma unroll 1
        for (int j = k >> 1; j > 0; j >>= 1) shuffle_stage(k, j);
    }
#pragma unroll
    for (int k = 64; k <= 32 * E; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j >= 32; j >>= 1) {   // register-to-register inside the lane, direction known statically
#pragma unroll
            for (int e = 0; e < E; e++) {
                const int pe = e ^ (j >> 5);
                if (pe > e) {
                    const bool up = ((e * 32) & k) == 0;
                    const bool gt = hi[e] > hi[pe] || (KW == 2 && hi[e] == hi[pe] && lo[e] > lo[pe]);
                    if (gt == up) {
                        uint64_t t0 = hi[e]; hi[e] = hi[pe]; hi[pe] = t0;
                        if (KW == 2) { uint64_t t1 = lo[e]; lo[e] = lo[pe]; lo[pe] = t1; }
                        if (HASV) { uint32_t t2 = pv[e]; pv[e] = pv[pe]; pv[pe] = t2; }
                    }
                }
            }
        }
#pragma unroll 1
        for (int j = 16; j > 0; j >>= 1) shuffle_stage(k, j);
    }
#pragma unroll
    for (int e = 0; e < E; e++) {
        const int i = e * 32 + lane;
        if (i < M) {
            if (KW == 2) *reinterpret_cast<ulonglong2*>(a + 2 * i) = make_ulonglong2(hi[e], lo[e]);
            else a[i] = hi[e];
            if (HASV) v[i] = pv[e];
        }
    }
    __syncwarp();
}
template <int KW, bool HASV>
__device__ __forceinline__ void warp_sort_dispatch(uint64_t* a, uint32_t* v, int M) {
    if (M <= 32) warp_sort_regs<1, KW, HASV>(a, v, M);
    else if (M <= 64) warp_sort_regs<2, KW, HASV>(a, v, M);
    else warp_sort_regs<4, KW, HASV>(a, v, M);
}
#define CSV_WARP_SORT(KW, HASV, a, v, M) \
    if (Team::SIZE == 32 && (M) <= 128) { warp_sort_dispatch<KW, HASV>((uint64_t*)(a), (v), (M)); return; }
#else
#define CSV_WARP_SORT(KW, HASV, a, v, M)
#endif

// bitonic sorts, ascending, M a power of two (callers pad with all-ones keys)
template <class Team>
CSV_HD void team_sort_k128(Team tm, K128* a, int M) {
    CSV_WARP_SORT(2, false, a, (uint32_t*)nullptr, M)
    for (int k = 2; k <= M; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tm.tid(); i < M; i += Team::SIZE) {
                int l = i ^ j;
                if (l > i) {
                    bool up = (i & k) == 0;
                    K128 x = a[i], y = a[l];
                    if (k128_gt(x, y) == up) { a[i] = y; a[l] = x; }
                }
            }
            tm.sync();
        }
}
template <class Team>
CSV_HD void team_sort_k128_kv(Team tm, K128* a, uint32_t* v, int M) {
    CSV_WARP_SORT(2, true, a, v, M)
    for (int k = 2; k <= M; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tm.tid(); i < M; i += Team::SIZE) {
                int l = i ^ j;
                if (l > i) {
                    bool up = (i & k) == 0;
                    K128 x = a[i], y = a[l];
                    if (k128_gt(x, y) == up) {
                        a[i] = y; a[l] = x;
                        uint32_t vx = v[i]; v[i] = v[l]; v[l] = vx;
                    }
                }
            }
            tm.sync();
        }
}
template <class Team>
CSV_HD void team_sort_u64(Team tm, uint64_t* a, int M) {
    CSV_WARP_SORT(1, false, a, (uint32_t*)nullptr, M)
    for (int k = 2; k <= M; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tm.tid(); i < M; i += Team::SIZE) {
                int l = i ^ j;
                if (l > i) {
                    bool up = (i & k) == 0;
                    uint64_t x = a[i], y = a[l];
                    if ((x > y) == up) { a[i] = y; a[l] = x; }
                }
            }
            tm.sync();
        }
}
template <class Team>
CSV_HD void team_sort_kv(Team tm, uint64_t* a, uint32_t* v, int M) {
    CSV_WARP_SORT(1, true, a, v, M)
    for (int k = 2; k <= M; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tm.tid(); i < M; i += Team::SIZE) {
                int l = i ^ j;
                if (l > i) {
                    bool up = (i & k) == 0;
                    uint64_t x = a[i], y = a[l];
                    if ((x > y) == up) {
                        a[i] = y; a[l] = x;
                        uint32_t vx = v[i]; v[i] = v[l]; v[l] = vx;
                    }
                }
            }
            tm.sync();
        }
}

CSV_HD uint32_t ord32(int32_t x) { return (uint32_t)x ^ 0x80000000u; }  // order-preserving
CSV_HD int32_t unord32(uint32_t x) { return (int32_t)(x ^ 0x80000000u); }
CSV_HD uint32_t hi32(uint64_t x) { return (uint32_t)(x >> 32); }
CSV_HD uint32_t lo32(uint64_t x) { return (uint32_t)x; }
CSV_HD uint64_t pack64(uint32_t h, uint32_t l) { return ((uint64_t)h << 32) | l; }

// ------------------------------------------------------------------------------------------
// numpy's pairwise summation (np.std's reduction), non-recursive.  get(i) -> double.
// ------------------------------------------------------------------------------------------
template <class F>
CSV_HD double np_pairwise_leaf(F get, int64_t lo, int64_t n) {
    if (n < 8) {
        double res = 0.;
        for (int64_t i = 0; i < n; i++) res += get(lo + i);
        return res;
    }
    double r0 = get(lo), r1 = get(lo + 1), r2 = get(lo + 2), r3 = get(lo + 3), r4 = get(lo + 4), r5 = get(lo + 5),
           r6 = get(lo + 6), r7 = get(lo + 7);
    int64_t i;
    for (i = 8; i < n - (n % 8); i += 8) {
        r0 += get(lo + i); r1 += get(lo + i + 1); r2 += get(lo + i + 2); r3 += get(lo + i + 3);
        r4 += get(lo + i + 4); r5 += get(lo + i + 5); r6 += get(lo + i + 6); r7 += get(lo + i + 7);
    }
    double res = ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7));
    for (; i < n; i++) res += get(lo + i);
    return res;
}
template <class F>
CSV_HD double np_pairwise_sum(F get, int64_t n) {
    if (n <= 128) return np_pairwise_leaf(get, 0, n);
    struct Fr { int64_t lo, n; int stage; double left; };
    Fr st[48];
    int sp = 0;
    double ret = 0.;
    st[sp].lo = 0; st[sp].n = n; st[sp].stage = 0; st[sp].left = 0.; sp++;
    while (sp > 0) {
        Fr& f = st[sp - 1];
        if (f.stage == 0) {
            if (f.n <= 128) { ret = np_pairwise_leaf(get, f.lo, f.n); sp--; }
            else {
                int64_t n2 = f.n / 2; n2 -= n2 % 8;
                f.stage = 1;
                st[sp].lo = f.lo; st[sp].n = n2; st[sp].stage = 0; st[sp].left = 0.; sp++;
            }
        } else if (f.stage == 1) {
            f.left = ret;
            int64_t n2 = f.n / 2; n2 -= n2 % 8;
            f.stage = 2;
            st[sp].lo = f.lo + n2; st[sp].n = f.n - n2; st[sp].stage = 0; st[sp].left = 0.; sp++;
        } else {
            ret = f.left + ret;
            sp--;
        }
    }
    return ret;
}
// np.std of get_int(i), i in [0, n): mean = sum/n (exact integer sum), sqrt(pairwise(x*x)/n)
template <class G>
CSV_HD double np_std(G get_int, int64_t n, int64_t sum) {
    double mean = (double)sum / (double)n;
    auto sq = [&](int64_t i) { double x = (double)get_int(i) - mean; return x * x; };
    double ret = np_pairwise_sum(sq, n);
    ret = ret / (double)n;
    return sqrt(ret);
}
// cal_CIPOS (cuteSV_genotype.py:58-60) with the libm-pow table
CSV_HD int32_t cal_cipos(double std, int64_t n, const double* pow_half) { return (int32_t)(1.96 * std / pow_half[n]); }

#if defined(__CUDA_ARCH__)
// np.std of n <= 128 values for TWO arrays at once on a warp: lanes 0-7 own numpy's eight strided
// accumulators r0..r7 of array 0, lanes 8-15 those of array 1 (np_pairwise_leaf above, same additions
// in the same order: the r_j chains are independent, the tree (r0+r1)+(r2+r3)... is a xor-butterfly
// of commutative adds, the tail is added sequentially).  Returns the std in lanes 0-7 / 8-15.
template <class G0, class G1>
__device__ __forceinline__ double warp_np_std2(G0 get0, G1 get1, int n, int64_t sum0, int64_t sum1) {
    const int lane = (int)(threadIdx.x & 31);
    const int which = (lane >> 3) & 1, j = lane & 7;
    const double mean = (double)(which ? sum1 : sum0) / (double)n;
    auto sq = [&](int i) { const double x = (double)(which ? get1(i) : get0(i)) - mean; return x * x; };
    double res;
    if (n < 8) {
        res = 0.;
        for (int i = 0; i < n; i++) res += sq(i);
    } else {
        const int n8 = n - (n % 8);
        double r = sq(j);
        for (int i = 8 + j; i < n8; i += 8) r += sq(i);
        r = r + __shfl_xor_sync(0xffffffffu, r, 1);
        r = r + __shfl_xor_sync(0xffffffffu, r, 2);
        r = r + __shfl_xor_sync(0xffffffffu, r, 4);
        res = r;
        for (int i = n8; i < n; i++) res += sq(i);
    }
    res = res / (double)n;
    return sqrt(res);
}
#endif

// rescale_read_counts (cuteSV_genotype.py:25-31) + index into the host-built cal_GL table
// (table[c0*101+c1] for c0+c1 <= 100; slots 10201 / 10202 hold the (3,1) and (6,2) specials).
CSV_HD int32_t gl_index(int32_t c0, int32_t c1) {
    if (c0 == 3 && c1 == 1) return 10201;
    if (c0 == 6 && c1 == 2) return 10202;
    int32_t total = c0 + c1;
    if (total > 100) {
        double f = (double)c0 / (double)total;
        c0 = (int32_t)(100.0 * f);
        c1 = 100 - c0;
    }
    return c0 * 101 + c1;
}
static constexpr int GL_TABLE_N = 10203;

// ------------------------------------------------------------------------------------------
// views of the inputs of one SV type
// ------------------------------------------------------------------------------------------
// INDEL: raw (unsorted) columns + the permutation produced by the radix sort of the linearised
// position; members of a chain cluster are sidx[s .. s+m).
struct alignas(16) IndelRec { int32_t a, b, rid; uint32_t idx; };   // one 16 B record per signature of the sorted domain
struct IndelView {
    const int32_t *chrom, *a, *b, *rid, *c;
    const uint32_t* sidx;
    int is_ins;
    // record mode (rec != nullptr): member j of the sorted domain is rec[j] (+ recc[j] = column c of INS); the
    // columns above are then only used for the contig of a cluster.  Otherwise members are gathered through sidx.
    const IndelRec* rec;
    const int32_t* recc;
};
// DUP / INV / TRA: columns already in the reference's full sort order with exact duplicates
// removed (cuteSV:783-802, 958-969); oidx = original input index.
struct SortedView {
    const int32_t *chrom, *a, *b, *rid, *c;
};

struct ClusterParams {
    int32_t min_support, min_support_allele, min_size, max_size, bias;
    double ratio;   // INDEL: diff_ratio_merging_*; TRA: diff_ratio_filtering_TRA
    double keep;    // remain_reads_ratio clamped to <= 1 (resolveINDEL.py:46-47)
    int32_t genotype;
};

// bytes of arena per padded member for the INDEL routine
static constexpr int INDEL_ARENA_PER = 64;
// arena carve-up for capacity M
struct IndelArena {
    K128* A0;        // 16 B: sort-1 keys -> sort-2 keys (u64) -> remain-sort keys
    int32_t* A1;     // 12 B: arrival a/aux/idx -> K3 (u64) + V3 (u32)
    int32_t* D;      // 20 B: pos,len,rid,aux,idx after dedup
    uint32_t* F;     // 4 B flags / scans
    uint64_t* KA;    // 8 B allele keys
    uint32_t* VA;    // 4 B allele starts
    CSV_HD IndelArena(char* base, int M) {
        A0 = (K128*)base;
        KA = (uint64_t*)(base + (size_t)16 * M);
        A1 = (int32_t*)(base + (size_t)24 * M);
        D = (int32_t*)(base + (size_t)36 * M);
        F = (uint32_t*)(base + (size_t)56 * M);
        VA = (uint32_t*)(base + (size_t)60 * M);
    }
};

// two halves so that a caller can issue the two returning atomics early and look at their results
// only after other work (their round trip to L2 is ~1 us)
CSV_HD void emit_reserve_issue(const Emit& E, uint32_t n_names, uint32_t* slot, uint32_t* noff) {
#if defined(__CUDA_ARCH__)
    if (E.cursor) {
        const unsigned long long old = atomicAdd(E.cursor, (1ull << 32) | (unsigned long long)n_names);
        *slot = (uint32_t)(old >> 32);
        *noff = (uint32_t)old;
        return;
    }
#endif
    *slot = atomic_add_u32(&E.ctr->n_cand, 1u);
    *noff = atomic_add_u32(&E.ctr->n_names, n_names);
}
// largest allele support seen (sizes the n ** 0.5 table): a plain look first, the atomic only when it would change something
CSV_HD void note_support(const Emit& E, uint32_t n) {
    if (n > *(volatile uint32_t*)&E.ctr->max_support) atomic_max_u32(&E.ctr->max_support, n);
}
CSV_HD bool emit_reserve_check(const Emit& E, uint32_t n_names, uint32_t s, uint32_t o) {
    if (s >= E.lim.cap_cand) { atomic_or_u32(&E.ctr->status, ST_CAND_OVERFLOW); return false; }
    if ((uint64_t)o + n_names > E.lim.cap_names) { atomic_or_u32(&E.ctr->status, ST_NAMES_OVERFLOW); return false; }
    return true;
}
CSV_HD bool emit_reserve(const Emit& E, uint32_t n_names, uint32_t* slot, uint32_t* noff) {
    // called by one thread
    emit_reserve_issue(E, n_names, slot, noff);
    return emit_reserve_check(E, n_names, *slot, *noff);
}

// ------------------------------------------------------------------------------------------
// INS / DEL: generate_del_cluster / generate_ins_cluster (resolveINDEL.py:110-219, 319-432)
// on the m signatures sidx[s..s+m) of one chain cluster.  M = pow2 >= m arena capacity.
// kslot = global kept-cluster slot (indexes Emit::cnt); returns nothing, emits rows.
// ------------------------------------------------------------------------------------------
// SV / KEEPALL >= 0 fix the SV type / "remain_reads_ratio keeps every member" at compile time (the hot warp kernels are
// instantiated per type so that the other type's branches and the trimming sorts are not part of their instruction stream).
template <class Team, int SV = -1, int KEEPALL = -1>
CSV_HD void indel_cluster(Team tm, const IndelView& in, int64_t s, int m, int M, char* arena, int64_t* red,
                          const ClusterParams& P, int svtype_rt, uint32_t kslot, const Emit& E) {
    const int svtype = SV >= 0 ? SV : svtype_rt;
    const int t = tm.tid();
    IndelArena A(arena, M);
    int32_t* ar_a = A.A1;
    int32_t* ar_aux = A.A1 + M;
    int32_t* ar_idx = A.A1 + 2 * M;
    uint32_t* SJ = (uint32_t*)A.KA;  // 4 B * M inside the (still unused) allele-key region
    // 1. load members.  ONE sort by (read, pos, len, arrival) serves three purposes at once:
    //    exact duplicates become adjacent (remove_duplicates_sorted, cuteSV:958-969), every read's
    //    signatures become one run whose first element is the read's first occurrence in the
    //    reference's (pos, len, name) order (cuteSV:764,774), and the run is in that order.
    for (int j = t; j < M; j += Team::SIZE) {
        K128 k;
        if (j < m) {
            uint32_t i;
            int32_t a, bb, rr, aux;
            if (in.rec) {   // one 16 B record (+ 4 B) per member, consecutive in the sorted domain
                const IndelRec r = in.rec[s + j];
                i = r.idx; a = r.a; bb = r.b; rr = r.rid; aux = in.recc ? in.recc[s + j] : 0;
            } else {
                i = in.sidx[s + j];
                a = in.a[i]; bb = in.b[i]; rr = in.rid[i]; aux = in.c ? in.c[i] : 0;
            }
            int32_t pos = in.is_ins ? (a >> 1) : a;
            ar_a[j] = a;
            ar_aux[j] = aux;
            ar_idx[j] = (int32_t)i;
            k.hi = pack64(ord32(rr), (uint32_t)pos);
            k.lo = pack64(ord32(bb), i);   // ties: original input index (independent of arrival order)
        } else {
            k.hi = ~0ull; k.lo = ~0ull;
        }
        A.A0[j] = k;
        SJ[j] = (uint32_t)j;                     // payload: arrival slot (addresses ar_a / ar_aux / ar_idx)
    }
    tm.sync();
    team_sort_k128_kv(tm, A.A0, SJ, M);
    // 2. remove_duplicates_sorted: adjacent identical tuples
    auto keep_fn = [&](int q) -> bool {
        if (q == 0) return true;
        K128 x = A.A0[q], y = A.A0[q - 1];
        if (x.hi != y.hi || hi32(x.lo) != hi32(y.lo)) return true;
        int jx = (int)SJ[q], jy = (int)SJ[q - 1];
        return !(ar_a[jx] == ar_a[jy] && ar_aux[jx] == ar_aux[jy]);
    };
    for (int q = t; q < m; q += Team::SIZE) A.F[q] = keep_fn(q) ? 1u : 0u;
    tm.sync();
    const int m2 = (int)team_flag_scan(tm, A.F, m, red);
    int32_t* D_pos = A.D; int32_t* D_len = A.D + M; int32_t* D_rid = A.D + 2 * M; int32_t* D_aux = A.D + 3 * M;
    int32_t* D_idx = A.D + 4 * M;
    for (int q = t; q < m; q += Team::SIZE) {
        if (keep_fn(q)) {
            K128 x = A.A0[q];
            int j = (int)SJ[q];
            uint32_t d = A.F[q];
            D_pos[d] = (int32_t)lo32(x.hi); D_len[d] = unord32(hi32(x.lo)); D_rid[d] = unord32(hi32(x.hi));
            D_aux[d] = ar_aux[j]; D_idx[d] = ar_idx[j];
        }
    }
    tm.sync();
    if (m2 < P.min_support) {  // len(semi_del_cluster) >= read_count (resolveINDEL.py:62)
        if (t == 0) E.cnt[kslot] = 0;
        return;
    }
    // 3. per-read dedup (resolveINDEL.py:125-131): one entry per read = its longest signature
    //    (strictly larger replaces), kept at the dict position of the read's first occurrence
    for (int q = t; q < m2; q += Team::SIZE) A.F[q] = (q == 0 || D_rid[q] != D_rid[q - 1]) ? 1u : 0u;
    tm.sync();
    const int u = (int)team_flag_scan(tm, A.F, m2, red);
    if (u < P.min_support) {  // len(read_tag) < read_count (:133)
        if (t == 0) E.cnt[kslot] = 0;
        return;
    }
    K128* K3 = A.A0;               // sort-1 keys are dead: everything lives in the D arrays now
    uint32_t* V3 = (uint32_t*)A.A1;  // arrival arrays are dead too
    const int M3 = pow2ceil(u);
    for (int q = t; q < m2; q += Team::SIZE) {
        const bool head = q == 0 || D_rid[q] != D_rid[q - 1];
        if (head) {
            int best = q;
            for (int r = q + 1; r < m2 && D_rid[r] == D_rid[q]; r++)
                if (D_len[r] > D_len[best]) best = r;  // strictly larger replaces (:130)
            const uint32_t g = A.F[q];
            // sorted(read_tag.values(), key=len) is stable on the dict order = order of first occurrence in the
            // (pos, len, name) sorted cluster; names differ between reads, so (pos, len, name) of the first
            // occurrence is a total tie-break
            K128 k;
            k.hi = pack64(ord32(D_len[best]), (uint32_t)D_pos[q]);
            k.lo = pack64(ord32(D_len[q]), ord32(D_rid[q]));
            K3[g] = k;
            V3[g] = (uint32_t)best;
        }
    }
    tm.sync();
    for (int q = u + t; q < M3; q += Team::SIZE) { K128 k; k.hi = ~0ull; k.lo = ~0ull; K3[q] = k; V3[q] = 0; }
    tm.sync();
    team_sort_k128_kv(tm, K3, V3, M3);
    // 4. allele split on the length-sorted unique reads (:137-162)
    int64_t part = 0;
    for (int i = t; i < u; i += Team::SIZE) part += D_len[V3[i]];
    const int64_t sum_len = team_sum(tm, part, red);
    const double thr = P.ratio * ((double)sum_len / (double)u);
    auto brk = [&](int i) -> bool {
        return i > 0 && (double)(D_len[V3[i]] - D_len[V3[i - 1]]) > thr;
    };
    for (int i = t; i < u; i += Team::SIZE) A.F[i] = brk(i) ? 1u : 0u;
    tm.sync();
    const int na = (int)team_flag_scan(tm, A.F, u, red) + 1;
    for (int i = t; i < u; i += Team::SIZE)
        if (i == 0 || brk(i)) A.VA[A.F[i] + (brk(i) ? 1u : 0u)] = (uint32_t)i;
    tm.sync();
    const int MA = pow2ceil(na);
    for (int a = t; a < MA; a += Team::SIZE) {
        if (a < na) {
            uint32_t st = A.VA[a], en = a + 1 < na ? A.VA[a + 1] : (uint32_t)u;
            A.KA[a] = pack64(en - st, (uint32_t)a);  // sorted(allele_collect, key=[support]) stable (:163)
        } else A.KA[a] = ~0ull;
    }
    tm.sync();
    if (na > 1) team_sort_kv(tm, A.KA, A.VA, MA);
    // 5. one candidate per allele with enough support (:165-219 / 370-432)
    uint32_t n_emit = 0;
    for (int k = 0; k < na; k++) {
        const int n = (int)hi32(A.KA[k]);
        const int st = (int)A.VA[k];
        if (n < P.min_support_allele) continue;
        int64_t remain = (int64_t)(P.keep * (double)n);
        if (remain < 1) remain = 1;
        if (KEEPALL == 1) remain = n;   // (the host only picks this instantiation when keep == 1.0)
        int64_t pp = 0, pl = 0;
        for (int i = t; i < n; i += Team::SIZE) { uint32_t e = V3[st + i]; pp += D_pos[e]; pl += D_len[e]; }
        const int64_t sp = team_sum(tm, pp, red);
        const int64_t sl = team_sum(tm, pl, red);
        // members closest to the mean: order by |x - mean| == order by |n*x - sum| (exact), index tie-break
        int64_t kept_pos_sum = sp, kept_len_sum = sl;
        int32_t search = 0;
        {
            int64_t best = INT64_MAX;
            for (int i = t; i < n; i += Team::SIZE) {
                int64_t d = (int64_t)n * D_pos[V3[st + i]] - sp; if (d < 0) d = -d;
                if (d < best) best = d;
            }
            const int64_t dmin = team_min(tm, best, red);
            int64_t bi = INT64_MAX;
            for (int i = t; i < n; i += Team::SIZE) {
                int64_t d = (int64_t)n * D_pos[V3[st + i]] - sp; if (d < 0) d = -d;
                if (d == dmin && i < bi) bi = i;
            }
            const int64_t imin = team_min(tm, bi, red);
            search = D_pos[V3[st + imin]];  // search_threshold = allele_list[0] (:177)
        }
        // INS: first member (allele order) whose sequence is long enough (:399-405).  It needs signalLen, which
        // with remain == n (the default remain_reads_ratio) is known here, otherwise only after the remain sort.
        int32_t pos_pick = 0, aux = 0;
        uint32_t slot = 0, noff = 0;
        bool reserved = false;
        if (svtype != CSV_INS || remain >= n) {
            bool drop = false;
            if (svtype == CSV_INS) {
                const int32_t need = (int32_t)((double)sl / (double)remain);
                int64_t bi = INT64_MAX;
                for (int i = t; i < n; i += Team::SIZE)
                    if (D_aux[V3[st + i]] >= need && i < bi) bi = i;
                const int64_t pick = team_min(tm, bi, red);
                if (pick == INT64_MAX) drop = true;  // ideal_ins_seq == '<INS>' -> dropped
                else { pos_pick = D_pos[V3[st + pick]]; aux = D_idx[V3[st + pick]]; }
            }
            if (drop) continue;
            if (t == 0) emit_reserve_issue(E, (uint32_t)n, &slot, &noff);   // results are looked at after the std work
            reserved = true;
        }
        if (KEEPALL != 1 && remain < n) {
            // keep only the `remain` closest members (remain_reads_ratio < 1)
            K128* R = A.A0;
            const int MR = pow2ceil(n);
            for (int pass = 0; pass < 2; pass++) {
                const int32_t* src = pass == 0 ? D_pos : D_len;
                const int64_t tot = pass == 0 ? sp : sl;
                for (int i = t; i < MR; i += Team::SIZE) {
                    K128 x;
                    if (i < n) {
                        int64_t d = (int64_t)n * src[V3[st + i]] - tot; if (d < 0) d = -d;
                        x.hi = (uint64_t)d; x.lo = (uint64_t)i;
                    } else { x.hi = ~0ull; x.lo = ~0ull; }
                    R[i] = x;
                }
                tm.sync();
                team_sort_k128(tm, R, MR);
                int64_t ps = 0;
                for (int i = t; i < remain; i += Team::SIZE) ps += src[V3[st + (int)R[i].lo]];
                const int64_t tot_keep = team_sum(tm, ps, red);
                if (pass == 0) kept_pos_sum = tot_keep; else kept_len_sum = tot_keep;
            }
        }
        const double breakpointStart = (double)kept_pos_sum / (double)remain;
        const double signalLen = (double)kept_len_sum / (double)remain;
        // n ** 0.5 comes from a table of pow_n entries.  An allele at least that large reads entry 1 instead: it sets
        // ST_POW_TABLE below, the host grows the table and reruns, and this call's records are discarded.
        const int64_t n_pow = (uint32_t)n < E.lim.pow_n ? n : 1;
        // CIPOS / CILEN: np.std over the whole allele (:191-194); two lanes work concurrently
#if defined(__CUDA_ARCH__)
        if (Team::SIZE == 32) {  // warp team: 16 lanes share the two reductions (n <= 128 here)
            auto g0 = [&](int i) { return (int64_t)D_pos[V3[st + i]]; };
            auto g1 = [&](int i) { return (int64_t)D_len[V3[st + i]]; };
            const double sd = warp_np_std2(g0, g1, n, sp, sl);
            if (t == 0 || t == 8) red[t >> 3] = cal_cipos(sd, n_pow, E.pow_half);
        } else
#endif
        if (Team::SIZE > 1) {
            if (t < 2) {  // lanes 0 / 1 run the SAME instruction stream on pos / len
                const int32_t* src = t == 0 ? D_pos : D_len;
                auto gv = [&](int64_t i) { return (int64_t)src[V3[st + i]]; };
                red[t] = cal_cipos(np_std(gv, n, t == 0 ? sp : sl), n_pow, E.pow_half);
            }
        } else {
            auto gp = [&](int64_t i) { return (int64_t)D_pos[V3[st + i]]; };
            red[0] = cal_cipos(np_std(gp, n, sp), n_pow, E.pow_half);
            auto gl = [&](int64_t i) { return (int64_t)D_len[V3[st + i]]; };
            red[1] = cal_cipos(np_std(gl, n, sl), n_pow, E.pow_half);
        }
        tm.sync();
        const int32_t cipos = (int32_t)red[0], cilen = (int32_t)red[1];
        tm.sync();
        int32_t pos_out = (int32_t)breakpointStart;
        if (svtype == CSV_INS) {
            if (!reserved) {  // remain < n: signalLen is only known now
                const int32_t need = (int32_t)signalLen;
                int64_t bi = INT64_MAX;
                for (int i = t; i < n; i += Team::SIZE)
                    if (D_aux[V3[st + i]] >= need && i < bi) bi = i;
                const int64_t pick = team_min(tm, bi, red);
                if (pick == INT64_MAX) continue;  // ideal_ins_seq == '<INS>' -> dropped
                pos_pick = D_pos[V3[st + pick]];
                aux = D_idx[V3[st + pick]];
            }
            pos_out = pos_pick;
            search = pos_out;
        }
        int64_t ok = 0;
        if (t == 0) {
            if ((uint32_t)n >= E.lim.pow_n) atomic_or_u32(&E.ctr->status, ST_POW_TABLE);
            note_support(E, (uint32_t)n);
            if (!reserved) emit_reserve_issue(E, (uint32_t)n, &slot, &noff);
            ok = emit_reserve_check(E, (uint32_t)n, slot, noff) ? 1 : 0;
            red[0] = ok; red[1] = slot; red[2] = noff;
        }
        tm.sync();
        ok = red[0]; slot = (uint32_t)red[1]; noff = (uint32_t)red[2];
        tm.sync();
        if (ok) {
            for (int i = t; i < n; i += Team::SIZE) E.names[noff + i] = D_rid[V3[st + i]];
            if (t == 0) {
                csv_cand c;
                c.svtype = svtype; c.chrom = in.chrom[in.rec ? in.rec[s].idx : in.sidx[s]]; c.pos = pos_out;
                c.len = svtype == CSV_DEL ? (int32_t)(-signalLen) : (int32_t)signalLen;
                c.support = n; c.cipos = cipos; c.cilen = cilen; c.search_pos = search; c.pos2 = 0; c.aux = aux;
                c.names_off = (int32_t)noff; c.names_cnt = n; c.cluster = (int32_t)kslot; c.flags = 0;
                c.reserved[0] = (int32_t)n_emit; c.reserved[1] = 0;
                E.cand[slot] = c;
            }
        }
        n_emit++;
    }
    if (t == 0) E.cnt[kslot] = n_emit;
}

// ------------------------------------------------------------------------------------------
// helpers shared by DUP / INV / TRA: members q in [0,m) are rows s+q of a SortedView.
// Arena per member: 16 (K128) + 8 (u64) + 4 (F) + 4 (SUB) + 4 (X) = 36 B, see OtherArena.
// ------------------------------------------------------------------------------------------
static constexpr int OTHER_ARENA_PER = 40;
struct OtherArena {
    K128* K;        // 16 B
    uint64_t* O;    // 8 B: (b, q) order
    uint32_t* F;    // 4 B
    uint32_t* SUB;  // 4 B: sub-cluster start table
    uint32_t* X;    // 4 B: scratch (distinct ids / first positions)
    uint32_t* Y;    // 4 B
    CSV_HD OtherArena(char* base, int M) {
        K = (K128*)base;
        O = (uint64_t*)(base + (size_t)16 * M);
        F = (uint32_t*)(base + (size_t)24 * M);
        SUB = (uint32_t*)(base + (size_t)28 * M);
        X = (uint32_t*)(base + (size_t)32 * M);
        Y = (uint32_t*)(base + (size_t)36 * M);
    }
};

// number of distinct read ids among rows s+O-order positions [lo, hi) (ordered by O); leaves
// the sorted (rid, position) keys in kbuf[0..n) and the head flags scanned in F.
template <class Team>
CSV_HD int distinct_reads(Team tm, const SortedView& in, int64_t s, const uint64_t* O, int lo, int hi, uint64_t* kbuf,
                          uint32_t* F, int64_t* red) {
    const int t = tm.tid();
    const int n = hi - lo;
    const int Mn = pow2ceil(n);
    for (int i = t; i < Mn; i += Team::SIZE)
        kbuf[i] = i < n ? pack64(ord32(in.rid[s + (O ? lo32(O[lo + i]) : (uint32_t)(lo + i))]), (uint32_t)i) : ~0ull;
    tm.sync();
    team_sort_u64(tm, kbuf, Mn);
    for (int i = t; i < n; i += Team::SIZE) F[i] = (i == 0 || hi32(kbuf[i]) != hi32(kbuf[i - 1])) ? 1u : 0u;
    tm.sync();
    return (int)team_flag_scan(tm, F, n, red);
}

// sort members by (b, q) and split into sub-clusters where the b gap exceeds bias.
// Returns ns; SUB[k] = start (in O order) of sub-cluster k (k < ns); use sub_end() for the end.
template <class Team>
CSV_HD int split_on_b(Team tm, const SortedView& in, int64_t s, int m, int M, OtherArena& A, int32_t bias, int64_t* red) {
    const int t = tm.tid();
    for (int q = t; q < M; q += Team::SIZE) A.O[q] = q < m ? pack64(ord32(in.b[s + q]), (uint32_t)q) : ~0ull;
    tm.sync();
    team_sort_u64(tm, A.O, M);
    auto brk = [&](int i) -> bool {
        return i > 0 && (int64_t)unord32(hi32(A.O[i])) - (int64_t)unord32(hi32(A.O[i - 1])) > bias;
    };
    for (int i = t; i < m; i += Team::SIZE) A.F[i] = brk(i) ? 1u : 0u;
    tm.sync();
    const int ns = (int)team_flag_scan(tm, A.F, m, red) + 1;
    for (int i = t; i < m; i += Team::SIZE)
        if (i == 0 || brk(i)) A.SUB[A.F[i] + (brk(i) ? 1u : 0u)] = (uint32_t)i;
    tm.sync();
    return ns;
}

CSV_HD int sub_end(const OtherArena& A, int k, int ns, int m) { return k + 1 < ns ? (int)A.SUB[k + 1] : m; }

template <class Team>
CSV_HD bool emit_other(Team tm, const Emit& E, int64_t* red, const csv_cand& proto, int n_names, const uint32_t* ids,
                       uint32_t kslot, uint32_t n_emit) {
    // ids[0..n_names): read ids (ord32-encoded) in output order, in team memory
    const int t = tm.tid();
    if (t == 0) {
        uint32_t slot = 0, noff = 0;
        int64_t ok = emit_reserve(E, (uint32_t)n_names, &slot, &noff) ? 1 : 0;
        red[0] = ok; red[1] = slot; red[2] = noff;
    }
    tm.sync();
    const int64_t ok = red[0];
    const uint32_t slot = (uint32_t)red[1], noff = (uint32_t)red[2];
    tm.sync();
    if (!ok) return false;
    for (int i = t; i < n_names; i += Team::SIZE) E.names[noff + i] = unord32(ids[i]);
    if (t == 0) {
        csv_cand c = proto;
        c.names_off = (int32_t)noff; c.names_cnt = n_names; c.cluster = (int32_t)kslot;
        c.reserved[0] = (int32_t)n_emit; c.reserved[1] = 0;
        E.cand[slot] = c;
    }
    return true;
}

// ------------------------------------------------------------------------------------------
// DUP: generate_dup_cluster (resolveDUP.py:79-131)
// ------------------------------------------------------------------------------------------
template <class Team>
CSV_HD void dup_cluster(Team tm, const SortedView& in, int64_t s, int m, int M, char* arena, int64_t* red,
                        const ClusterParams& P, uint32_t kslot, const Emit& E) {
    const int t = tm.tid();
    OtherArena A(arena, M);
    uint64_t* kb = (uint64_t*)A.K;
    if (distinct_reads(tm, in, s, (const uint64_t*)nullptr, 0, m, kb, A.F, red) < P.min_support) {  // :82-84
        if (t == 0) E.cnt[kslot] = 0;
        return;
    }
    const int ns = split_on_b(tm, in, s, m, M, A, P.bias, red);  // :86-94
    uint32_t n_emit = 0;
    for (int k = 0; k < ns; k++) {
        const int lo = (int)A.SUB[k], hi = sub_end(A, k, ns, m), n = hi - lo;
        const int u = distinct_reads(tm, in, s, A.O, lo, hi, kb, A.F, red);  // :96
        if (u < P.min_support) continue;
        // distinct ids, ascending (the reference's list(set()) order is unspecified)
        for (int i = t; i < n; i += Team::SIZE)
            if (i == 0 || hi32(kb[i]) != hi32(kb[i - 1])) A.X[A.F[i]] = hi32(kb[i]);
        const int low_b = (int)((double)n * 0.4), up_b = (int)((double)n * 0.6);  // :99-100
        int64_t bp1, bp2;
        if (low_b == up_b) {
            uint32_t q = lo32(A.O[lo + low_b]);
            bp1 = in.a[s + q]; bp2 = in.b[s + q];
        } else {
            int64_t p1 = 0, p2 = 0;
            for (int i = low_b + t; i < up_b; i += Team::SIZE) { uint32_t q = lo32(A.O[lo + i]); p1 += in.a[s + q]; p2 += in.b[s + q]; }
            const int64_t s1 = team_sum(tm, p1, red), s2 = team_sum(tm, p2, red);
            bp1 = (int64_t)((double)s1 / (double)(up_b - low_b));
            bp2 = (int64_t)((double)s2 / (double)(up_b - low_b));
        }
        tm.sync();
        const int64_t d = bp2 - bp1;
        if ((P.min_size <= d && d <= P.max_size) || (P.min_size <= d && P.max_size == -1)) {  // :112
            csv_cand c;
            c.svtype = CSV_DUP; c.chrom = in.chrom[s]; c.pos = (int32_t)bp1; c.len = (int32_t)d; c.support = u;
            c.cipos = 0; c.cilen = 0; c.search_pos = 0; c.pos2 = (int32_t)bp2; c.aux = 0; c.flags = 0;
            emit_other(tm, E, red, c, u, A.X, kslot, n_emit);
            n_emit++;
        }
        tm.sync();
    }
    if (t == 0) E.cnt[kslot] = n_emit;
}

// ------------------------------------------------------------------------------------------
// INV: generate_semi_inv_cluster (resolveINV.py:101-203)
// ------------------------------------------------------------------------------------------
template <class Team>
CSV_HD void inv_cluster(Team tm, const SortedView& in, int64_t s, int m, int M, char* arena, int64_t* red,
                        const ClusterParams& P, uint32_t kslot, const Emit& E) {
    const int t = tm.tid();
    OtherArena A(arena, M);
    uint64_t* kb = (uint64_t*)A.K;
    uint64_t* kb2 = kb + M;  // second half of the K128 region
    if (distinct_reads(tm, in, s, (const uint64_t*)nullptr, 0, m, kb, A.F, red) < P.min_support) {  // :106-109
        if (t == 0) E.cnt[kslot] = 0;
        return;
    }
    const int ns = split_on_b(tm, in, s, m, M, A, P.bias, red);  // :111-125
    uint32_t n_emit = 0;
    for (int k = 0; k < ns; k++) {
        const int lo = (int)A.SUB[k], hi = sub_end(A, k, ns, m), n = hi - lo;
        if (n < P.min_support) continue;  // temp_count >= read_count (:126,173)
        const int u = distinct_reads(tm, in, s, A.O, lo, hi, kb, A.F, red);
        // temp_id keys: distinct names in first-occurrence order of the bp2-sorted sub-cluster
        const int Mu = pow2ceil(u);
        for (int i = t; i < n; i += Team::SIZE)
            if (i == 0 || hi32(kb[i]) != hi32(kb[i - 1])) kb2[A.F[i]] = pack64(lo32(kb[i]), hi32(kb[i]));  // (first pos, rid)
        for (int i = u + t; i < Mu; i += Team::SIZE) kb2[i] = ~0ull;
        tm.sync();
        team_sort_u64(tm, kb2, Mu);
        for (int i = t; i < u; i += Team::SIZE) A.X[i] = lo32(kb2[i]);
        int64_t p1 = 0, p2 = 0;
        for (int i = t; i < n; i += Team::SIZE) { uint32_t q = lo32(A.O[lo + i]); p1 += in.a[s + q]; p2 += in.b[s + q]; }
        const int64_t s1 = team_sum(tm, p1, red), s2 = team_sum(tm, p2, red);
        const int64_t bp1 = (int64_t)rint((double)s1 / (double)n);  // round(): half-to-even (:129)
        const int64_t bp2 = (int64_t)rint((double)s2 / (double)n);
        const int64_t inv_len = bp2 - bp1;
        if (inv_len >= P.min_size && u >= P.min_support && (inv_len <= P.max_size || P.max_size == -1)) {  // :132-134
            csv_cand c;
            c.svtype = CSV_INV; c.chrom = in.chrom[s]; c.pos = (int32_t)bp1; c.len = (int32_t)inv_len; c.support = u;
            c.cipos = 0; c.cilen = 0; c.search_pos = 0; c.pos2 = (int32_t)bp2; c.aux = in.c[s]; c.flags = 0;
            emit_other(tm, E, red, c, u, A.X, kslot, n_emit);
            n_emit++;
        }
        tm.sync();
    }
    if (t == 0) E.cnt[kslot] = n_emit;
}

// ------------------------------------------------------------------------------------------
// TRA: generate_semi_tra_cluster (resolveTRA.py:106-254); call_gt stays on the host
// ------------------------------------------------------------------------------------------
template <class Team>
CSV_HD void tra_cluster(Team tm, const SortedView& in, int64_t s, int m, int M, char* arena, int64_t* red,
                        const ClusterParams& P, uint32_t kslot, const Emit& E) {
    const int t = tm.tid();
    OtherArena A(arena, M);
    uint64_t* kb = (uint64_t*)A.K;
    const int ns = split_on_b(tm, in, s, m, M, A, P.bias, red);  // :109-124
    if (distinct_reads(tm, in, s, (const uint64_t*)nullptr, 0, m, kb, A.F, red) < P.min_support) {  // :128
        if (t == 0) E.cnt[kslot] = 0;
        return;
    }
    // distinct reads per sub-cluster; keep the two best by (-distinct, order) (:131 stable sort)
    int best0 = -1, best1 = -1, d0 = -1, d1 = -1;
    for (int k = 0; k < ns; k++) {
        const int d = distinct_reads(tm, in, s, A.O, (int)A.SUB[k], sub_end(A, k, ns, m), kb, A.F, red);
        if (d > d0) { best1 = best0; d1 = d0; best0 = k; d0 = d; }
        else if (d > d1) { best1 = k; d1 = d; }
    }
    int n_out = 0;
    if (ns > 1 && (double)d1 >= 0.5 * (double)P.min_support) {  // :133
        if ((double)(d0 + d1) >= (double)m * P.ratio) n_out = 2;  // :134
    } else {
        if ((double)d0 >= (double)m * P.ratio) n_out = 1;  // :211
    }
    uint32_t n_emit = 0;
    for (int w = 0; w < n_out; w++) {
        const int k = w == 0 ? best0 : best1;
        const int lo = (int)A.SUB[k], hi = sub_end(A, k, ns, m), n = hi - lo;
        const int u = distinct_reads(tm, in, s, A.O, lo, hi, kb, A.F, red);
        for (int i = t; i < n; i += Team::SIZE)
            if (i == 0 || hi32(kb[i]) != hi32(kb[i - 1])) A.X[A.F[i]] = hi32(kb[i]);
        int64_t p1 = 0, p2 = 0;
        for (int i = t; i < n; i += Team::SIZE) { uint32_t q = lo32(A.O[lo + i]); p1 += in.a[s + q]; p2 += in.b[s + q]; }
        int64_t s1 = team_sum(tm, p1, red), s2 = team_sum(tm, p2, red);
        int64_t listlen = n;
        if (k == 0) {  // the loop revisits element 0: counted twice (:113-124)
            uint32_t q0 = lo32(A.O[0]);
            s1 += in.a[s + q0]; s2 += in.b[s + q0]; listlen += 1;
        }
        csv_cand c;
        c.svtype = CSV_TRA; c.chrom = in.chrom[s];
        c.pos = (int32_t)((double)s1 / (double)listlen);   // int(temp[k][0]/len(temp[k][2])) (:173)
        c.pos2 = (int32_t)((double)s2 / (double)listlen);
        c.len = 0; c.support = u; c.cipos = 0; c.cilen = 0; c.search_pos = 0; c.aux = in.c[s];
        c.flags = P.genotype ? CSV_F_GT_HOST : 0;
        emit_other(tm, E, red, c, u, A.X, kslot, n_emit);
        n_emit++;
        tm.sync();
    }
    if (t == 0) E.cnt[kslot] = n_emit;
}

// ------------------------------------------------------------------------------------------
// genotype windows (call_gt of resolveINDEL.py:450-451, resolveDUP.py:146-151,
// resolveINV.py:218-221): integer windows [s, e] with "covered by read r" == r.start <= s and
// r.end >= e, which is what overlap_cover's event order computes (cuteSV_genotype.py:100-138).
// Half-integer windows (bias/2) are mapped to s = floor, e = ceil (equivalent for integer reads).
// ------------------------------------------------------------------------------------------
struct GtParams { int32_t bias_del, gt_bias_ins, bias_dup, bias_inv; };
CSV_HD int64_t floor_half(int64_t twice) { return twice >= 0 ? twice / 2 : -((-twice + 1) / 2); }
CSV_HD int64_t ceil_half(int64_t twice) { return twice >= 0 ? (twice + 1) / 2 : -((-twice) / 2); }
CSV_HD int n_windows_of(const csv_cand& c) {
    return (c.svtype == CSV_DEL || c.svtype == CSV_INS) ? 1 : (c.svtype == CSV_DUP || c.svtype == CSV_INV) ? 2 : 0;
}
CSV_HD void window_of(const csv_cand& c, int which, const GtParams& G, int64_t* s, int64_t* e) {
    if (c.svtype == CSV_DEL || c.svtype == CSV_INS) {
        const int64_t b = c.svtype == CSV_INS ? G.gt_bias_ins : G.bias_del;
        int64_t lo = (int64_t)c.search_pos - b; if (lo < 0) lo = 0;
        *s = lo; *e = (int64_t)c.search_pos + b;
        return;
    }
    int64_t nb;
    if (c.svtype == CSV_DUP) { nb = (int64_t)c.pos2 - c.pos; if (G.bias_dup < nb) nb = G.bias_dup; }
    else nb = G.bias_inv;
    const int64_t x = which == 0 ? c.pos : c.pos2;
    int64_t lo = floor_half(2 * x - nb); if (2 * x - nb < 0) lo = 0;
    *s = lo; *e = ceil_half(2 * x + nb);
}

// ------------------------------------------------------------------------------------------
// TRA genotyping from a packed all-alignments table: call_gt (resolveTRA.py:260-309) with
// count_coverage (cuteSV_genotype.py:72-93) and threshold_ref_count (:62-70).
// ------------------------------------------------------------------------------------------
struct AlnView {
    const int32_t *chrom, *start, *end, *rid;
    const uint8_t* prim;
    const uint32_t* off;       // first record of every contig, n_contigs + 1 entries
    const int32_t* max_span;   // longest record per contig
    const int64_t* contig_len;
};
CSV_HD int32_t threshold_ref_count(int32_t num) { return num <= 2 ? 20 * num : num <= 5 ? 9 * num : num <= 15 ? 7 * num : 5 * num; }
CSV_HD bool sorted_contains(const int32_t* v, int n, int32_t x) {
    int lo = 0, hi = n;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (v[mid] < x) lo = mid + 1; else hi = mid; }
    return lo < n && v[lo] == x;
}
// bam.fetch(chr, s, e) in BAM order: records of the contig with start < e and end > s, by start.
// Returns status (1, -1 or 0 = loop ran to completion); nset / dr accumulate over both regions.
// (xs, xe): a window on the same contig whose spanning reads are ALREADY in the set (second region
// of an intra-contig pair); xs > xe disables it.
CSV_HD int tra_count_coverage(const AlnView& A, int32_t chr, int64_t s, int64_t e, const int32_t* sup, int n_sup, int32_t up_bound,
                              int32_t itround, int32_t* nset, int32_t* dr, int64_t xs, int64_t xe) {
    int64_t iteration = 0, primary = 0;
    const uint32_t lo0 = A.off[chr], hi0 = A.off[chr + 1];
    // first record that can still overlap: start >= s - max_span
    uint32_t lo = lo0, hi = hi0;
    const int64_t min_start = s - (int64_t)A.max_span[chr];
    while (lo < hi) { uint32_t mid = lo + (hi - lo) / 2; if ((int64_t)A.start[mid] < min_start) lo = mid + 1; else hi = mid; }
    for (uint32_t i = lo; i < hi0 && (int64_t)A.start[i] < e; i++) {
        if (!((int64_t)A.end[i] > s)) continue;  // not returned by fetch
        iteration++;
        if (!A.prim[i]) continue;               // flag not in (0, 16): `continue` also skips the itround check
        primary++;
        if ((int64_t)A.start[i] < s && (int64_t)A.end[i] > e) {
            const bool seen = xs <= xe && (int64_t)A.start[i] < xs && (int64_t)A.end[i] > xe;  // set.add of a known name
            if (!seen) {
                (*nset)++;                       // read_count.add(name): one primary record per name
                if (!sorted_contains(sup, n_sup, A.rid[i])) (*dr)++;
            }
            if (*nset >= up_bound) return 1;
        }
        if (iteration >= itround) return ((double)primary / (double)iteration) <= 0.2 ? 1 : -1;
    }
    return 0;
}
// The call_gt window of a breakpoint: [max(pos - bias, 0), min(pos + bias, contig length)] (resolveTRA.py:264-265, 292-293)
CSV_HD void tra_window(const AlnView& A, int32_t chr, int64_t pos, int32_t bias, int64_t* s, int64_t* e) {
    *s = pos - bias; if (*s < 0) *s = 0;
    *e = pos + bias; if (*e > A.contig_len[chr]) *e = A.contig_len[chr];
}
// call_gt of one breakpoint pair.  sup: the n_sup supporting read ids (ascending, duplicates allowed; DV = n_sup).
// CC runs count_coverage: TraCountCoverage below for the host, the warp-cooperative scan in kernels.cuh for the device.
template <class CC>
CSV_HD csv_geno tra_call_gt_rules(const CC& cc, const AlnView& A, int32_t chr1, int64_t pos1, int32_t chr2, int64_t pos2, const int32_t* sup,
                                  int32_t n_sup, int32_t bias, int32_t gt_round, const csv_geno* gl_table) {
    const int32_t up = threshold_ref_count(n_sup);
    int32_t nset = 0, dr = 0;
    int64_t s, e;
    tra_window(A, chr1, pos1, bias, &s, &e);
    const int st = cc(A, chr1, s, e, sup, n_sup, up, gt_round, &nset, &dr, 1, 0);
    csv_geno g;
    if (st == -1) {  // DR '.', GT './.' (resolveTRA.py:277-282)
        g.dr = -1; g.dv = n_sup; g.gt = -1; g.pl[0] = g.pl[1] = g.pl[2] = 0; g.gq = 0; g.status = 2; g.qual = 0.0;
        return g;
    }
    if (st == 0) {  // the second window's status is not used (resolveTRA.py:301)
        const int64_t s1 = s, e1 = e;
        tra_window(A, chr2, pos2, bias, &s, &e);
        if (chr2 == chr1) cc(A, chr2, s, e, sup, n_sup, up, gt_round, &nset, &dr, s1, e1);
        else cc(A, chr2, s, e, sup, n_sup, up, gt_round, &nset, &dr, 1, 0);
    }
    g = gl_table[gl_index(dr, n_sup)];
    g.dr = dr; g.dv = n_sup;
    return g;
}
struct TraCountCoverage {
    CSV_HD int operator()(const AlnView& A, int32_t chr, int64_t s, int64_t e, const int32_t* sup, int n_sup, int32_t up_bound, int32_t itround,
                          int32_t* nset, int32_t* dr, int64_t xs, int64_t xe) const {
        return tra_count_coverage(A, chr, s, e, sup, n_sup, up_bound, itround, nset, dr, xs, xe);
    }
};
CSV_HD csv_geno tra_call_gt(const AlnView& A, int32_t chr1, int64_t pos1, int32_t chr2, int64_t pos2, const int32_t* sup, int32_t n_sup,
                            int32_t bias, int32_t gt_round, const csv_geno* gl_table) {
    return tra_call_gt_rules(TraCountCoverage{}, A, chr1, pos1, chr2, pos2, sup, n_sup, bias, gt_round, gl_table);
}
// One TRA candidate of csv_cluster (chr2 = aux >> 2); sup: its names slice.
CSV_HD void tra_call_gt(const AlnView& A, const csv_cand& c, const int32_t* sup, int32_t bias, int32_t gt_round, const csv_geno* gl_table,
                        csv_geno* g) {
    *g = tra_call_gt(A, c.chrom, c.pos, c.aux >> 2, c.pos2, sup, c.names_cnt, bias, gt_round, gl_table);
}

// ------------------------------------------------------------------------------------------
// standalone overlap_cover (cuteSV_genotype.py:95-159) over arbitrary windows and reads rows, in half units
// (window (s2, e2) = 2 * (s, e), read (2 * start, 2 * end)).  The event order sv-right 0 < read-left 1 <
// read-right 2 < sv-left 3 makes a row overlap a window iff start < e and end > s, and cover it iff
// start <= s and end >= e (end > s follows from e > s, which the caller guarantees).
// ------------------------------------------------------------------------------------------
CSV_HD bool gc_overlaps(int64_t rs2, int64_t re2, int64_t s2, int64_t e2) { return rs2 < e2 && re2 > s2; }
CSV_HD bool gc_covers(int64_t rs2, int64_t re2, int64_t s2, int64_t e2) { return rs2 <= s2 && re2 >= e2 && re2 > s2; }
// Bins of 2^GC_SHIFT half units per contig; coordinates below 0 fall into bin 0.  A window is listed in every bin of
// [s2, e2 - 1], a row visits every bin of [rs2, re2].  An overlapping pair is taken in one bin only, that of
// max(rs2, s2): the point lies in both ranges, so both sides reach that bin.
static constexpr int GC_SHIFT = 12;
CSV_HD int64_t gc_bin(int64_t x2) { return x2 < 0 ? 0 : (x2 >> GC_SHIFT); }
CSV_HD bool gc_pair_home(int64_t rs2, int64_t s2, int64_t bin) { return gc_bin(rs2 > s2 ? rs2 : s2) == bin; }

// Sort + deduplicate one segment of name ids (a window's cover or overlap list) into out[0, k), ascending; returns k.
// Team-parallel rank sort: first[i] marks the first occurrence of a value, and a first occurrence goes to the number of
// distinct smaller values.  O(n^2 / team size): a warp takes short segments, a CTA the pile-ups.  `first` holds n bytes.
template <class Team>
CSV_HD int gc_sort_unique(const Team& tm, const int32_t* in, int n, uint8_t* first, int32_t* out) {
    for (int i = tm.tid(); i < n; i += Team::SIZE) {
        const int32_t v = in[i];
        bool f = true;
        for (int j = 0; j < i && f; j++) f = in[j] != v;
        first[i] = f ? 1 : 0;
    }
    tm.sync();
    for (int i = tm.tid(); i < n; i += Team::SIZE) {
        if (!first[i]) continue;
        const int32_t v = in[i];
        int pos = 0;
        for (int j = 0; j < n; j++) pos += (first[j] && in[j] < v) ? 1 : 0;
        out[pos] = v;
    }
    int k = 0;
    for (int j = 0; j < n; j++) k += first[j];
    tm.sync();
    return k;
}

// assign_gt's DR for one candidate (cuteSV_genotype.py:161-173, windows united as in resolveDUP.py:155-157):
// |a ∪ b \ sup| for ascending unique a, b and ascending sup (duplicates allowed).
CSV_HD int32_t gc_union_minus(const int32_t* a, int na, const int32_t* b, int nb, const int32_t* sup, int nsup) {
    int32_t dr = 0;
    int i = 0, j = 0;
    while (i < na || j < nb) {
        int32_t v;
        if (j >= nb || (i < na && a[i] < b[j])) v = a[i++];
        else if (i >= na || b[j] < a[i]) v = b[j++];
        else { v = a[i++]; j++; }
        if (!sorted_contains(sup, nsup, v)) dr++;
    }
    return dr;
}

// ------------------------------------------------------------------------------------------
// INS/DEL density filter of one genome partition of bp 256-bp buckets (kernels.cuh k_part_filter).  Bucket b is kept
// when it holds a signature and the buckets [b - rb, b + rb] hold >= need signatures; outside [0, bp) the window reads
// the halo: hl[j] = signatures in the (j + 1)-th last bucket of the previous partition, hr[j] = in bucket j of the next
// one (j < rb <= 64, zero where there is no neighbour).  h(b) is the count of bucket b in [0, bp).  A thread owns the
// strip [b0, b0 + n) of n <= 64 consecutive buckets.
// ------------------------------------------------------------------------------------------
template <class H>
CSV_HD uint32_t pf_count(const H& h, int k, int bp, const uint32_t* hl, const uint32_t* hr) {
    return k < 0 ? hl[-k - 1] : k >= bp ? hr[k - bp] : h(k);
}

// An interior strip: every window [b - rb, b + rb] of its buckets lies inside [0, bp) and reaches at most the neighbouring
// strips (rb <= n), so it needs neither the halo nor a bounds test.
CSV_HD bool pf_strip_interior(int b0, int n, int bp, int rb) { return rb <= n && b0 - rb >= 0 && b0 + n - 1 + rb < bp; }

// pf_strip_flags of an interior strip.  hs(s, j) = h(b0 + s * n + j) for s = -1, 0, 1 and 0 <= j < n: the caller indexes
// its histogram directly (k_part_filter's transposed histogram: word (j << 9) + thread + s).
template <class HS>
CSV_HD uint64_t pf_strip_flags_interior(const HS& hs, int n, int rb, uint32_t need, uint32_t* kept) {
    uint32_t win = 0, sum = 0;
#pragma unroll 1
    for (int k = 1; k <= rb; k++) win += hs(-1, n - k);
#pragma unroll 1
    for (int k = 0; k <= rb && k < n; k++) win += hs(0, k);
    if (rb == n) win += hs(1, 0);
    uint64_t flags = 0;
    for (int j = 0; j < n; j++) {
        if (j) {   // in: bucket j + rb of this strip or the next; out: bucket j - rb - 1 of this strip or the previous
            const int ka = j + rb, sa = ka >= n ? 1 : 0;
            const int ks = j - rb - 1, ss = ks < 0 ? -1 : 0;
            win += hs(sa, ka - sa * n) - hs(ss, ks - ss * n);
        }
        const uint32_t c = hs(0, j);
        if (c > 0 && win >= need) { flags |= 1ull << j; sum += c; }
    }
    *kept = sum;
    return flags;
}

// Keep flags of a strip (bit j: bucket b0 + j) by a sliding window sum: 2 * rb + 1 reads for the first bucket, two for
// every later one.  *kept = signatures in the strip's kept buckets.  Interior strips take pf_strip_flags_interior over
// hs (as above); the others test every read against the partition's ends.
template <class H, class HS>
CSV_HD uint64_t pf_strip_flags(const H& h, const HS& hs, int b0, int n, int bp, int rb, uint32_t need, const uint32_t* hl,
                               const uint32_t* hr, uint32_t* kept) {
    if (pf_strip_interior(b0, n, bp, rb)) return pf_strip_flags_interior(hs, n, rb, need, kept);
    uint32_t win = 0, sum = 0;
    for (int k = b0 - rb; k <= b0 + rb; k++) win += pf_count(h, k, bp, hl, hr);
    uint64_t flags = 0;
    for (int j = 0; j < n; j++) {
        const int b = b0 + j;
        if (j) win += pf_count(h, b + rb, bp, hl, hr) - pf_count(h, b - rb - 1, bp, hl, hr);
        const uint32_t c = h(b);
        if (c > 0 && win >= need) { flags |= 1ull << j; sum += c; }
    }
    *kept = sum;
    return flags;
}

// The same with the strip read through h alone.
template <class H>
CSV_HD uint64_t pf_strip_flags(const H& h, int b0, int n, int bp, int rb, uint32_t need, const uint32_t* hl, const uint32_t* hr,
                               uint32_t* kept) {
    return pf_strip_flags(h, [&](int s, int j) -> uint32_t { return h(b0 + s * n + j); }, b0, n, bp, rb, need, hl, hr, kept);
}

// Exclusive offsets of a strip's kept buckets, the first at `base`: put(j, offset, kept, count) for every bucket of the
// strip in order (count 0 for a dropped bucket, whose offset is that of the next kept one).
template <class H, class F>
CSV_HD void pf_strip_offsets(const H& h, int b0, int n, uint64_t flags, uint32_t base, F put) {
    for (int j = 0; j < n; j++) {
        const bool f = (flags >> j) & 1u;
        const uint32_t c = f ? h(b0 + j) : 0u;
        put(j, base, f, c);
        base += c;
    }
}

// ------------------------------------------------------------------------------------------
// INS/DEL chain clusters of one k_select_heads tile, read from its link mask: bit q (word q >> 5, bit q & 31) is set
// when element q is chained to element q - 1.  The caller's mask holds a halo of words on both sides of the tile and
// indexes it so that every q these routines read stays inside it.
// ------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
CSV_D int ctz32(uint32_t x) { return __ffs((int)x) - 1; }
CSV_D int clz32(uint32_t x) { return __clz((int)x); }
#else
inline int ctz32(uint32_t x) { return __builtin_ctz(x); }
inline int clz32(uint32_t x) { return __builtin_clz(x); }
#endif

// set bits q, q + 1, ... up to the first clear one, at most cap (reads bits q .. q + cap + 31 at most)
CSV_HD int link_run_up(const uint32_t* link, int q, int cap) {
    int r = 0;
    while (r < cap) {
        const int bo = q & 31;
        const uint32_t z = ~(link[q >> 5] >> bo);   // bit k: bit q + k is clear; the 32 - bo vacated bits count as clear
        const int ones = z ? ctz32(z) : 32;
        r += ones;
        if (ones < 32 - bo) break;
        q += 32 - bo;
    }
    return r < cap ? r : cap;
}

// set bits q, q - 1, ... down to the first clear one, at most cap (reads bits q - cap - 31 .. q at most)
CSV_HD int link_run_down(const uint32_t* link, int q, int cap) {
    int r = 0;
    while (r < cap) {
        const int bo = q & 31;
        const uint32_t z = ~(link[q >> 5] << (31 - bo));   // bit 31 - k: bit q - k is clear; the vacated bits count as clear
        const int ones = z ? clz32(z) : 32;
        r += ones;
        if (ones < bo + 1) break;
        q -= bo + 1;
    }
    return r < cap ? r : cap;
}

// q starts a chain cluster of at least need members: it is not chained to q - 1, and q + 1 .. q + need - 1 are chained
CSV_HD bool chain_head(const uint32_t* link, int q, int need) {
    return !((link[q >> 5] >> (q & 31)) & 1u) && link_run_up(link, q + 1, need - 1) >= need - 1;
}

// q is a member of a chain cluster of at least need members, wherever its head lies: the chained steps before and after
// q, each counted up to need - 1, make need - 1 together
CSV_HD bool chain_member(const uint32_t* link, int q, int need) {
    return link_run_down(link, q, need - 1) + link_run_up(link, q + 1, need - 1) >= need - 1;
}

// size class of the cluster headed at q: its member count when it has at most 32 members, 33 for up to split members,
// 34 beyond (reads the forward run up to split links)
CSV_HD int chain_size_class(const uint32_t* link, int q, int split) {
    const int m = 1 + link_run_up(link, q + 1, split);
    return m <= 32 ? m : m <= split ? 33 : 34;
}

}  // namespace csv
