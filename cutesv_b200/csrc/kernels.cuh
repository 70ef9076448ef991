// kernels.cuh -- the pipeline's kernels around core.h:
//   keys      (contig, pos) -> one linear sortable coordinate (+ input validation)
//   segment   chain-linkage boundary votes (max_cluster_bias_*) + ordered compaction of the
//             clusters that can reach min_support
//   cluster   one warp / one CTA / one CTA with global scratch per kept cluster -> core.h
//   order     candidates into the reference's emission order
//   genotype  windows binned on the linear coordinate, ONE streaming pass over the reads table,
//             cal_GL through the host-built libm table
#pragma once
#include "core.h"
#include "devprims.cuh"
#include "radix.cuh"
#include <type_traits>

namespace csv {

static constexpr int WARP_M = 128;    // largest cluster a warp-sized team handles (shared memory)
static constexpr int BLOCK_M = 2048;  // largest cluster a CTA-sized team handles in shared memory
static constexpr int CL_THREADS = 256;

// ------------------------------------------------------------------------------------------
// description of one SV type's sorted domain, passed by value to the kernels
// ------------------------------------------------------------------------------------------
struct TypeJob {
    int svtype;
    int64_t n_host;          // upper bound of the sorted-domain size
    const uint32_t* n_dev;   // actual size when it is only known on the device (small types)
    // INDEL: linear keys in sorted order
    const uint32_t* keys32;
    const uint64_t* keys64;
    IndelView iv;
    // DUP / INV / TRA: fully sorted, de-duplicated columns
    SortedView sv;
    ClusterParams cp;
    uint32_t kslot_base;     // first global kept-cluster slot of this type
    const uint32_t* kept_start;
    uint32_t* big_list;
    uint32_t* giant_list;
    uint32_t big_cap, giant_cap;
    char* giant_arena;
    int small_path;          // INS / DEL: clusters of <= 32 members go through the register kernel (k_cluster_small) first
    uint32_t* rest_list;     // ... which lists the others here (kept-cluster ordinals); null: the general kernel takes every cluster
    const uint32_t* n_rest;
    // record mode: k_select_heads lists the clusters of more than REST_SPLIT members from the front of rest_list and the
    // others from its end (rest_cap words), so that the general kernel hands out the costly clusters first
    const uint32_t* n_rest_lo;
    uint32_t rest_cap;
    uint2* small_list;       // (ordinal, members) of the clusters of <= 32 members, written by k_select_heads in record mode
    const uint32_t* n_small;
};

__device__ __forceinline__ int64_t job_n(const TypeJob& J) { return J.n_dev ? (int64_t)*J.n_dev : J.n_host; }

// element i (> 0) belongs to the same chain cluster as element i-1
__device__ __forceinline__ bool job_linked(const TypeJob& J, int64_t i) {
    const int32_t bias = J.cp.bias;
    switch (J.svtype) {
        case CSV_DEL:
        case CSV_INS:  // resolveINDEL.py:61,271 -- contigs are padded by > bias in the linear key
            if (J.keys32) return (J.keys32[i] - J.keys32[i - 1]) <= (uint32_t)bias;
            return (J.keys64[i] - J.keys64[i - 1]) <= (uint64_t)bias;
        case CSV_DUP:  // resolveDUP.py:35
            return J.sv.chrom[i] == J.sv.chrom[i - 1] && !(J.sv.a[i] - J.sv.a[i - 1] > bias);
        case CSV_INV:  // resolveINV.py:56
            return J.sv.chrom[i] == J.sv.chrom[i - 1] && J.sv.c[i] == J.sv.c[i - 1] && !(J.sv.a[i] - J.sv.a[i - 1] > bias) &&
                   !(J.sv.b[i] - J.sv.b[i - 1] > bias);
        default:       // TRA resolveTRA.py:41,65
            return J.sv.chrom[i] == J.sv.chrom[i - 1] && J.sv.c[i] == J.sv.c[i - 1] && !(J.sv.a[i] - J.sv.a[i - 1] > bias);
    }
}

// predicate of the segment step: i starts a chain cluster with at least min_support members
struct HeadPred {
    TypeJob J;
    __device__ __forceinline__ bool operator()(int64_t i) const {
        if (i > 0 && job_linked(J, i)) return false;
        const int64_t n = job_n(J);
        const int need = J.cp.min_support;
        int cnt = 1;
        int64_t j = i + 1;
        while (cnt < need && j < n && job_linked(J, j)) { cnt++; j++; }
        return cnt >= need;
    }
};

// Segment step, specialised: the chain-linkage votes of a 2048-element tile are taken with
// coalesced loads and kept as a bit mask in shared memory (one __ballot_sync per 32 elements);
// "i starts a cluster of >= min_support members" is then a bit test (core.h chain_head).  Ordered compaction as in
// k_select.
static constexpr int HEAD_MAX_NEED_WORDS = 64;  // supports min_support up to ~2000 via the mask; above -> generic path
// INS / DEL record mode (MR.rec != nullptr): the tile then gathers ONE 16 B record (+ column c of INS) per member of a kept
// cluster that lies in it, written at the member's sorted position -- the cluster kernels read a cluster's members as
// one contiguous range instead of gathering four or five columns per member.  Membership is a bit test too (core.h
// chain_member, over a backward halo of the mask), so a cluster that crosses a tile edge is gathered by both tiles, and
// a thread issues the loads of several members before it stores any record.  Only members of kept clusters are touched
// (a fifth of the filter's survivors on 30x ONT).  The gather is bound by its scattered column loads (one 32 B sector
// each), not by their latency: DEL takes a from the key where it can.
struct MemberRec {
    IndelRec* rec; int32_t* recc;
    const int32_t *a, *b, *rid, *c;
    const uint32_t* sidx;
    // classification of the kept clusters by size (null: not wanted)
    uint2* small_list; uint32_t* n_small;    // (kept ordinal, members) for <= 32 members
    uint32_t* rest_list; uint32_t* n_rest;   // kept ordinal for the others: > REST_SPLIT members from the front,
    uint32_t* n_rest_lo; uint32_t rest_cap;  // ... the others from the end of the rest_cap words
    // DEL: the contigs' linear offsets (n_contigs + 1).  In a tile that lies on one contig a member's a is its key minus
    // the contig's offset, so the gather loads one scattered column fewer (null: load every column)
    const uint64_t* del_off; int n_contigs;
};
static constexpr int REST_SPLIT = 64;
static constexpr int GATHER_GROUP = 4;   // 32 registers per thread (eight CTAs per SM) hold a group of 4 members' loads
__global__ void __launch_bounds__(SEL_THREADS) k_select_heads(TypeJob J, uint32_t* out, uint32_t out_cap, uint32_t* out_count,
                                                              TileSync ts, uint32_t* status_word, uint32_t overflow_bit, MemberRec MR) {
    pdl_launch_dependents(); pdl_wait();   // programmatic dependent launch: resident early, starts when the previous kernel has finished
    constexpr int WORDS = SEL_TILE / 32;
    // mask words: [0, back) before the tile, then the tile's WORDS, then fwd after it
    __shared__ uint32_t s_link[HEAD_MAX_NEED_WORDS + WORDS + HEAD_MAX_NEED_WORDS];
    __shared__ uint32_t s_warp[9];
    __shared__ uint32_t s_tile, s_excl, s_aoff;
    __shared__ uint8_t s_msize[SEL_TILE];   // size lists: size class of the tile's h-th head (core.h chain_size_class)
    const int64_t n = job_n(J);
    const uint32_t gen = ts_gen(ts);
    const int need = J.cp.min_support;
    // record mode reads need - 1 links on both sides of every position, and REST_SPLIT links after a head
    const int back = MR.rec ? (need + 31) / 32 + 1 : 0;
    const int fwd = (MR.rec ? max((need + 31) / 32, (REST_SPLIT + 32) / 32) : (need + 31) / 32) + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    while (true) {
        if (threadIdx.x == 0) s_tile = atomicAdd(ts.ticket, 1u);
        __syncthreads();
        const uint32_t tile = s_tile;
        const int64_t base = (int64_t)tile * SEL_TILE;
        if (base >= n) break;
        // link bits for [base - 32*back, base + SEL_TILE + 32*fwd): votes are evaluated in batches
        // of 8 words per warp so that the key loads of a batch are all in flight together
        for (int w0 = warp; w0 < back + WORDS + fwd; w0 += 8 * (SEL_THREADS / 32)) {
            bool l[8];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int w = w0 + u * (SEL_THREADS / 32);
                const int64_t i = base + (int64_t)(w - back) * 32 + lane;
                l[u] = (w < back + WORDS + fwd && i > 0 && i < n) ? job_linked(J, i) : false;
            }
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int w = w0 + u * (SEL_THREADS / 32);
                const uint32_t m = __ballot_sync(0xffffffffu, l[u]);
                if (lane == 0 && w < back + WORDS + fwd) s_link[w] = m;
            }
        }
        // DEL: the contig of the tile's first key by a 32-ary search, kept when the tile's last key lies on it too (the last
        // warp does it: it has the fewest mask words)
        if (MR.del_off && warp == SEL_THREADS / 32 - 1) {
            const uint64_t k0 = J.keys32[base], k1 = J.keys32[min(base + SEL_TILE, n) - 1];
            int lo = 0, span = MR.n_contigs;   // off[lo] <= k0 < off[lo + span]
            while (span > 1) {
                const int step = (span + 31) / 32;
                const bool le = lane * step < span && MR.del_off[lo + lane * step] <= k0;
                const int j = 31 - __clz(__ballot_sync(0xffffffffu, le));
                lo += j * step;
                span = min(step, span - j * step);
            }
            if (lane == 0) s_aoff = k1 < MR.del_off[lo + 1] ? (uint32_t)MR.del_off[lo] : ~0u;   // ~0u: it crosses a contig end
        }
        __syncthreads();
        const int p0 = threadIdx.x * SEL_ITEMS, q0 = back * 32;   // tile position p is mask bit q0 + p
        uint32_t flags = 0, cnt = 0;
#pragma unroll
        for (int j = 0; j < SEL_ITEMS; j++) {
            const int p = p0 + j;
            if (base + p < n && chain_head(s_link, q0 + p, need)) { flags |= 1u << j; cnt++; }
        }
        uint32_t total;
        const uint32_t local = block_excl_scan<256>(cnt, s_warp, &total);
        if (MR.small_list) {   // the heads' size classes, in head order
            uint32_t o = local;
#pragma unroll
            for (int j = 0; j < SEL_ITEMS; j++)
                if (flags >> j & 1u) s_msize[o++] = (uint8_t)chain_size_class(s_link, q0 + p0 + j, REST_SPLIT);
        }
        // warp 0 waits for the look-back while the other warps gather the members (it gathers its share afterwards)
        if (threadIdx.x < 32) {
            const uint32_t ex = lookback_exclusive_warp(ts.status, gen, (int)tile, total);
            if (threadIdx.x == 0) {
                s_excl = ex;
                if (base + SEL_TILE >= n) *out_count = ex + total;
            }
        }
        if (MR.rec) {   // positions threadIdx.x + j * SEL_THREADS: every load instruction of a warp reads consecutive words
            uint32_t mem = 0;
#pragma unroll 1
            for (int j = 0; j < SEL_ITEMS; j++) {
                const int p = threadIdx.x + j * SEL_THREADS;
                if (base + p < n && chain_member(s_link, q0 + p, need)) mem |= 1u << j;
            }
            const uint32_t* __restrict__ sidx = MR.sidx;
            const int32_t *__restrict__ ca = MR.a, *__restrict__ cb = MR.b, *__restrict__ cr = MR.rid, *__restrict__ cc = MR.c;
            IndelRec* __restrict__ rec = MR.rec;
            int32_t* __restrict__ recc = MR.recc;
            const uint32_t aoff = MR.del_off ? s_aoff : ~0u;
            uint32_t bad = 0;
#pragma unroll 1
            for (int j0 = 0; j0 < SEL_ITEMS; j0 += GATHER_GROUP) {   // a group's column loads in flight together
                uint32_t x[GATHER_GROUP];
#pragma unroll
                for (int u = 0; u < GATHER_GROUP; u++)
                    if (mem >> (j0 + u) & 1u) x[u] = sidx[base + threadIdx.x + (j0 + u) * SEL_THREADS];
#pragma unroll
                for (int u = 0; u < GATHER_GROUP; u++) {
                    if (mem >> (j0 + u) & 1u) {
                        const int64_t i = base + threadIdx.x + (j0 + u) * SEL_THREADS;
                        IndelRec r;
                        r.a = aoff != ~0u ? (int32_t)(J.keys32[i] - aoff) : ca[x[u]];
                        r.b = cb[x[u]]; r.rid = cr[x[u]]; r.idx = x[u];
                        const int32_t c5 = cc ? cc[x[u]] : 0;
                        if (r.rid < 0 || r.b < 0 || c5 < 0) bad |= ST_NEG_FIELD;
                        *reinterpret_cast<int4*>(&rec[i]) = *reinterpret_cast<const int4*>(&r);
                        if (recc) recc[i] = c5;
                    }
                }
            }
            if (bad) atomicOr(status_word, bad);
        }
        __syncthreads();
        uint32_t o = s_excl + local;
#pragma unroll
        for (int j = 0; j < SEL_ITEMS; j++) {
            if (flags >> j & 1u) {
                if (o < out_cap) out[o] = (uint32_t)(base + p0 + j);
                else atomicOr(status_word, overflow_bit);
                o++;
            }
        }
        if (MR.small_list) {   // the size lists of the cluster kernels, one atomic per warp and list; kept ordinal = s_excl + h
            const uint32_t ex = s_excl;
            for (uint32_t h0 = warp * 32; h0 < total; h0 += SEL_THREADS) {
                const uint32_t h = h0 + lane;
                const uint32_t sz = h < total ? s_msize[h] : 255u;
                const uint32_t lt = (1u << lane) - 1u;
                const uint32_t m_small = __ballot_sync(0xffffffffu, sz <= 32u);
                const uint32_t m_lo = __ballot_sync(0xffffffffu, sz == 33u), m_hi = __ballot_sync(0xffffffffu, sz == 34u);
                uint32_t b_small = 0, b_lo = 0, b_hi = 0;
                if (lane == 0) {
                    if (m_small) b_small = atomicAdd(MR.n_small, (uint32_t)__popc(m_small));
                    if (m_lo) b_lo = atomicAdd(MR.n_rest_lo, (uint32_t)__popc(m_lo));
                    if (m_hi) b_hi = atomicAdd(MR.n_rest, (uint32_t)__popc(m_hi));
                }
                b_small = __shfl_sync(0xffffffffu, b_small, 0);
                b_lo = __shfl_sync(0xffffffffu, b_lo, 0);
                b_hi = __shfl_sync(0xffffffffu, b_hi, 0);
                if (sz <= 32u) MR.small_list[b_small + __popc(m_small & lt)] = make_uint2(ex + h, sz);
                else if (sz == 33u) MR.rest_list[MR.rest_cap - 1u - (b_lo + __popc(m_lo & lt))] = ex + h;
                else if (sz == 34u) MR.rest_list[b_hi + __popc(m_hi & lt)] = ex + h;
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------
// keys
// ------------------------------------------------------------------------------------------
struct ContigTab {
    const uint64_t* off;   // linear offset of every contig (padded by > max bias), n+1 entries
    const int64_t* len;
    int32_t n;
};

// Density pre-filter (INS/DEL).  A chain cluster with >= min_support members has all of them
// within R = (min_support-1)*bias of each other, so a signature whose +-R neighbourhood holds fewer
// than min_support signatures can never be part of a cluster the reference would keep
// (resolveINDEL.py:62: len(cluster) >= read_count) and dropping it cannot merge or complete any
// other cluster.  Neighbourhood counts come from a coarse bucket histogram (conservative: whole
// buckets).  On 30x ONT noise this removes ~90 % of the signatures BEFORE the sort.
static constexpr int BKT_SHIFT = 8;   // 256 bp buckets
static constexpr int BKT_PAD = 64;   // >= largest neighbourhood radius in buckets

// grouped uploads from device memory: the offsets were never seen by the host, so they are checked here (off[0] == 0,
// off[n_contigs] == n, non-decreasing) before k_expand_contigs trusts them; reads only the n_contigs + 1 offsets
__global__ void __launch_bounds__(256) k_check_contig_off(const int64_t* __restrict__ off, int n_contigs, int64_t n, uint32_t* bad) {
    bool ok = true;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k <= n_contigs; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t o = off[k];
        if (k == 0 && o != 0) ok = false;
        if (k == n_contigs && o != n) ok = false;
        if (k < n_contigs && off[k + 1] < o) ok = false;
    }
    if (!ok) atomicOr(bad, ST_BAD_GROUPS);
}
// csv_cluster: an upload's device-side check result joins the call's status word (the upload ran before the counters were reset)
__global__ void k_fold_status(const uint32_t* __restrict__ src, uint32_t* dst) {
    if (threadIdx.x == 0 && *src) atomicOr(dst, *src);
}

// grouped uploads: chrom[i] = the contig k with off[k] <= i < off[k+1] (four consecutive rows per thread).
// bad != nullptr: the result of k_check_contig_off; failed offsets give contig 0 to every row instead (never read out of range)
__global__ void __launch_bounds__(256) k_expand_contigs(const int64_t* __restrict__ off, int n_contigs, int64_t n, int32_t* __restrict__ chrom,
                                                        const uint32_t* __restrict__ bad) {
    if (bad && *bad) {
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) chrom[i] = 0;
        return;
    }
    for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v * 4 < n; v += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i0 = v * 4;
        int lo = 0, hi = n_contigs;   // last k with off[k] <= i0
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (__ldg(&off[mid]) <= i0) lo = mid; else hi = mid; }
        int k = lo;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int64_t i = i0 + j;
            if (i >= n) break;
            while (__ldg(&off[k + 1]) <= i) k++;   // skips empty contigs; off[n_contigs] == n > i ends it
            chrom[i] = k;
        }
    }
}

// Four consecutive signatures per thread and iteration through 128-bit loads (64 B of loads in flight per
// thread: the kernel is a latency-bound stream); a scalar loop takes the tail / unaligned columns.
template <typename K>
__global__ void __launch_bounds__(256) k_indel_keys(const int32_t* __restrict__ chrom, const int32_t* __restrict__ a, const int32_t* __restrict__ b,
                             const int32_t* __restrict__ rid, int64_t n, int is_ins, ContigTab ct, K* __restrict__ keys,
                             uint32_t* status) {
    auto one = [&](int32_t c, int32_t raw, int32_t bb, int32_t rr, uint32_t& bad) -> K {
        K key = 0;
        if (c < 0 || c >= ct.n) bad |= ST_BAD_CHROM;
        else {
            const int64_t pos = is_ins ? (raw >> 1) : raw;
            if (raw < 0 || pos > ct.len[c]) bad |= ST_BAD_POS;
            else key = (K)(ct.off[c] + (uint64_t)pos);
        }
        if (rr < 0 || bb < 0) bad |= ST_NEG_FIELD;
        return key;
    };
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    const bool aligned = ((((uintptr_t)chrom) | ((uintptr_t)a) | ((uintptr_t)b) | ((uintptr_t)rid) | ((uintptr_t)keys)) & 15) == 0;
    const int64_t nv = aligned ? (n >> 2) : 0;
    uint32_t bad = 0;
    for (int64_t v = tid; v < nv; v += stride) {
        const int4 c4 = reinterpret_cast<const int4*>(chrom)[v], a4 = reinterpret_cast<const int4*>(a)[v];
        const int4 b4 = reinterpret_cast<const int4*>(b)[v], r4 = reinterpret_cast<const int4*>(rid)[v];
        const K k0 = one(c4.x, a4.x, b4.x, r4.x, bad), k1 = one(c4.y, a4.y, b4.y, r4.y, bad);
        const K k2 = one(c4.z, a4.z, b4.z, r4.z, bad), k3 = one(c4.w, a4.w, b4.w, r4.w, bad);
        if (sizeof(K) == 4) reinterpret_cast<uint4*>(keys)[v] = make_uint4((uint32_t)k0, (uint32_t)k1, (uint32_t)k2, (uint32_t)k3);
        else {
            reinterpret_cast<ulonglong2*>(keys)[2 * v] = make_ulonglong2((uint64_t)k0, (uint64_t)k1);
            reinterpret_cast<ulonglong2*>(keys)[2 * v + 1] = make_ulonglong2((uint64_t)k2, (uint64_t)k3);
        }
    }
    for (int64_t i = nv * 4 + tid; i < n; i += stride) {
        const K key = one(chrom[i], a[i], b[i], rid[i], bad);
        keys[i] = key;
    }
    if (bad) atomicOr(status, bad);
}

__device__ __forceinline__ uint32_t indel_key32(int32_t c, int32_t raw, int is_ins, const ContigTab& ct, uint32_t& bad) {
    if (c < 0 || c >= ct.n) { bad |= ST_BAD_CHROM; return 0u; }
    const int64_t pos = is_ins ? (raw >> 1) : raw;
    if (raw < 0 || pos > ct.len[c]) { bad |= ST_BAD_POS; return 0u; }   // len < 0: contig not owned by this shard
    return (uint32_t)(ct.off[c] + (uint64_t)pos);
}

// ------------------------------------------------------------------------------------------
// INS / DEL front end, partitioned: the genome's linear coordinate is cut into P partitions of 2^W bp (W <= 22, so a
// partition has at most 16384 buckets of 256 bp).  The density filter then needs no genome-sized bucket table: every
// partition's histogram is built, flagged, scanned and used inside one CTA's shared memory.
//    k_part_scatter  8 B/sig read (chrom, a),        -> the (key, index) pairs, every partition's written to its own pages
//                    8 B/sig written                    of a shared pool (fill counters, page table); halo counts at
//                                                       partition edges; input validation
//    k_part_filter   8 B/sig read (twice, the second  -> survivors in key order, 8 B per survivor written; the partition's
//                    mostly from L2) + the page ids     fill counter and page-table entries reset
// ------------------------------------------------------------------------------------------
static constexpr int PART_MAX = 1024;        // partitions: 32-bit keys, W = 22
static constexpr int PART_W_MAX = 22;
static constexpr int PART_W_MIN = 16;        // >= 256 buckets per partition: the +-BKT_PAD halo reaches the neighbours only
static constexpr int PF_STAGE = 5632;        // survivors of one partition ordered in shared memory; more spill to global
static constexpr int FIX_SMALL = 64;         // buckets with more survivors than this are ordered by a counting sort
static constexpr int PF_BIG_CAP = 256;       // buckets of more than FIX_SMALL survivors listed per partition
__host__ __device__ constexpr size_t pf_smem_bytes(int w) {
    return (size_t)(1u << (w - BKT_SHIFT)) * 4 + (size_t)(1u << (w - BKT_SHIFT)) / 32 * 4 + (size_t)PF_STAGE * 8;
}

// Paged partitions: the pairs of partition p take the ordinals 0 .. fill[p] - 1 of p, in pages of PART_PAGE pairs drawn
// from one pool; pt[p * ptw + k] = 1 + the pool page that holds ordinals k * PART_PAGE .., 0 while the page is unassigned.
// At most one page per partition is partly filled, so a pool of ceil(n / PART_PAGE) + P pages and rows of
// ptw = ceil(n / PART_PAGE) + 1 entries always suffice.  Both fill and pt are all zero between calls: k_part_filter
// resets every entry the scatter set.
static constexpr int PART_PAGE = 2048;   // 16 KB of pairs
static_assert(PART_PAGE % 2 == 0, "k_part_filter reads pairs two at a time, 16 B aligned");

// One 1024-thread CTA per round of PART_ROUND rows (round c: rows c * PART_ROUND ..), one CTA per SM.  The round's
// (key, row) pairs are grouped by partition in shared memory; thread p reserves the next cnt ordinals of partition p
// (atomicAdd on fill[p]) and takes a pool page for every page that starts inside its reservation (one atomicAdd on the
// pool counter), and publishes them in pt after the placement.  The page that holds its first ordinal, if that ordinal is
// not a page start, belongs to the reservation before it: the thread then waits for that entry.  The wait cannot
// deadlock: the owner's CTA reserved earlier, so it is resident or done, and no thread waits on another CTA before it
// has published its own pages (only the CTA's own barriers lie between its reservation and its publication).  The grouped
// round is then written out in order, position q (partition p) to ordinal resv[p] + q - run_off[p] of p, through the
// page ids cached in shared memory, so a warp's stores stay consecutive within every run.  16384 rows give 513 rounds of
// a type on config 2, about 3.9 waves of one CTA per SM on 132 SMs.
// The round's `chrom` and `a` come in by two 1-D bulk copies on one mbarrier, into the shared memory that later holds the
// grouped pairs; `chrom` and `a` must be 16 B aligned (run_indel checks it), and only the rows of the input's last
// partial 4-row group are loaded row by row.  Every thread then reads its PART_ROUND_V 4-row groups with conflict-free
// 16 B shared loads and keeps their keys in registers until they are placed.  Rows in the first or last rb buckets of a
// partition are counted into edge[p][j] (j < BKT_PAD: the j-th bucket of p; BKT_PAD + j: its j-th bucket from the end),
// the halo of the neighbours' windows.
static constexpr int PS_THREADS = 1024;
static constexpr int PART_ROUND = 16384, PART_ROUND_V = PART_ROUND / 4 / PS_THREADS;   // 4-row groups per thread
// pages one round touches: partition p's reservation of cnt rows spans at most cnt / PART_PAGE + 2 of them
static constexpr int PS_PAGES = PART_ROUND / PART_PAGE + 2 * PART_MAX;
__host__ __device__ constexpr size_t ps_smem_bytes() { return (size_t)PART_ROUND * 8 + (size_t)PART_MAX * 4 * 3 + (size_t)PS_PAGES * 4; }
static_assert(PART_MAX == PS_THREADS && PART_ROUND % (4 * PS_THREADS) == 0, "k_part_scatter tiling: one partition per thread");
// run offsets, ordinals and row indices are 32-bit (n < 2^32); one round must fit an SM's opt-in shared memory
static_assert(ps_smem_bytes() + 256 <= 227 * 1024, "k_part_scatter: one round per SM");
__global__ void __launch_bounds__(PS_THREADS, 1) k_part_scatter(const int32_t* __restrict__ chrom, const int32_t* __restrict__ a, int64_t n,
                                                                int is_ins, ContigTab ct, int W, int P, int rb, uint2* __restrict__ pool,
                                                                uint32_t* __restrict__ fill, uint32_t* pt, uint32_t ptw,
                                                                uint32_t* __restrict__ pool_next, uint32_t* __restrict__ edge,
                                                                uint32_t* status) {
    pdl_launch_dependents();
    extern __shared__ __align__(16) uint32_t s_dyn[];
    uint2* s_st = reinterpret_cast<uint2*>(s_dyn);                   // PART_ROUND pairs, grouped by partition
    int32_t* s_c = reinterpret_cast<int32_t*>(s_dyn);                // before that: the round's chrom ..
    int32_t* s_a = reinterpret_cast<int32_t*>(s_dyn) + PART_ROUND;   // .. and a
    uint32_t* s_fill = s_dyn + 2 * PART_ROUND;   // rows of the round per partition -> next free position of it in s_st
    uint32_t* s_d = s_fill + PART_MAX;           // partition p: ordinal - position in s_st (mod 2^32)
    uint32_t* s_pb = s_d + PART_MAX;             // partition p: index in s_pg of its page k, minus k (mod 2^32)
    uint32_t* s_pg = s_pb + PART_MAX;            // the pool pages of the round's reservations
    __shared__ uint32_t s_warp[32], s_npg;
    __shared__ __align__(8) uint64_t s_bar;
    const int t = (int)threadIdx.x, lane = t & 31, warp = t >> 5;
    const int64_t s0 = (int64_t)blockIdx.x * PART_ROUND;
    const int m = (int)min((int64_t)PART_ROUND, n - s0);
    const int m4 = m & ~3;   // rows of whole 4-row groups: the bulk copies' share
    if (t == 0) {
        mbar_init(&s_bar, 1);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the barrier init, visible to the async proxy
        if (m4) {
            mbar_expect_tx(&s_bar, (uint32_t)m4 * 8);
            bulk_copy(s_c, chrom + s0, (uint32_t)m4 * 4, &s_bar);
            bulk_copy(s_a, a + s0, (uint32_t)m4 * 4, &s_bar);
        } else {
            mbar_arrive(&s_bar);
        }
        s_npg = 0;
    }
    if (m4 + t < m) { s_c[m4 + t] = chrom[s0 + m4 + t]; s_a[m4 + t] = a[s0 + m4 + t]; }   // the input's last rows
    s_fill[t] = 0;
    __syncthreads();   // the barrier initialised; the tail rows and s_fill written
    mbar_wait(&s_bar, 0);
    uint32_t key[4 * PART_ROUND_V], bad = 0;   // row 4 * (j * PS_THREADS + thread) + i at key[4 * j + i]
#pragma unroll
    for (int j = 0; j < PART_ROUND_V; j++) {
        const int r = 4 * (j * PS_THREADS + t);
        const int4 cv = reinterpret_cast<const int4*>(s_c)[j * PS_THREADS + t];
        const int4 av = reinterpret_cast<const int4*>(s_a)[j * PS_THREADS + t];
        uint32_t b0 = 0, b1 = 0, b2 = 0, b3 = 0;   // rows past the input are not validated
        key[4 * j] = indel_key32(cv.x, av.x, is_ins, ct, b0);
        key[4 * j + 1] = indel_key32(cv.y, av.y, is_ins, ct, b1);
        key[4 * j + 2] = indel_key32(cv.z, av.z, is_ins, ct, b2);
        key[4 * j + 3] = indel_key32(cv.w, av.w, is_ins, ct, b3);
        bad |= (r < m ? b0 : 0u) | (r + 1 < m ? b1 : 0u) | (r + 2 < m ? b2 : 0u) | (r + 3 < m ? b3 : 0u);
    }
    if (bad) atomicOr(status, bad);
    const uint32_t bmask = (1u << (W - BKT_SHIFT)) - 1;
#pragma unroll
    for (int k = 0; k < 4 * PART_ROUND_V; k++) {
        if (4 * ((k >> 2) * PS_THREADS + t) + (k & 3) >= m) continue;
        const uint32_t p = key[k] >> W, bl = (key[k] >> BKT_SHIFT) & bmask;
        if (bl < (uint32_t)rb) atomicAdd(&edge[p * 2 * BKT_PAD + bl], 1u);
        if (bmask - bl < (uint32_t)rb) atomicAdd(&edge[p * 2 * BKT_PAD + BKT_PAD + (bmask - bl)], 1u);
        atomicAdd(&s_fill[p], 1u);
    }
    __syncthreads();   // every row counted, and read: the pairs may now overwrite the input
    // Reserve ordinals [r, r + v) of partition t (v > 0 only for t < P).  The latencies of the reservation, the page
    // allocation and the first probe of the page-table entry of a page begun earlier run under the scan and the placement.
    const uint32_t v = s_fill[t];
    const uint32_t r = v ? atomicAdd(&fill[t], v) : 0u;
    {   // exclusive scan of the per-partition counts, one partition per thread
        uint32_t incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += y;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const uint32_t w = s_warp[lane];
            uint32_t wi = w;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, wi, d);
                if (lane >= d) wi += y;
            }
            s_warp[lane] = wi - w;
        }
        __syncthreads();
        const uint32_t o = s_warp[warp] + incl - v;
        s_fill[t] = o;
        s_d[t] = r - o;
    }
    const uint32_t k0 = r / PART_PAGE, k1 = v ? (r + v - 1) / PART_PAGE : k0;
    const bool lead = v && r % PART_PAGE != 0;   // page k0 was taken by an earlier reservation
    const uint32_t np = v ? k1 - k0 + 1 : 0u, own = np - (lead ? 1u : 0u);
    uint32_t* row = pt + (size_t)t * ptw;
    const uint32_t id = own ? atomicAdd(pool_next, own) : 0u;
    uint32_t g = 1;
    if (lead) asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(g) : "l"(row + k0) : "memory");
    uint32_t base = np;   // warp scan of the page counts -> this partition's slots in s_pg
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, base, d);
        if (lane >= d) base += y;
    }
    uint32_t wbase = 0;
    if (lane == 31) wbase = atomicAdd(&s_npg, base);
    base = __shfl_sync(0xffffffffu, wbase, 31) + base - np;
    s_pb[t] = base - k0;
    __syncthreads();   // s_fill holds the run offsets
#pragma unroll
    for (int k = 0; k < 4 * PART_ROUND_V; k++) {
        const int q = 4 * ((k >> 2) * PS_THREADS + t) + (k & 3);
        if (q < m) s_st[atomicAdd(&s_fill[key[k] >> W], 1u)] = make_uint2(key[k], (uint32_t)(s0 + q));
    }
    // publish this partition's pages, then (only then) wait for the page an earlier reservation began
    for (uint32_t i = 0; i < own; i++) {
        const uint32_t k = k1 + 1 - own + i;
        asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(row + k), "r"(id + i + 1u) : "memory");
        s_pg[base + k - k0] = id + i;
    }
    if (lead) {
        while (g == 0) {
            __nanosleep(64);
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(g) : "l"(row + k0) : "memory");
        }
        s_pg[base] = g - 1u;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < PART_ROUND / PS_THREADS; j++) {
        const int q = j * PS_THREADS + t;
        if (q >= m) break;
        const uint2 pr = s_st[q];
        const uint32_t p = pr.x >> W, e = (uint32_t)q + s_d[p];
        pool[(size_t)s_pg[s_pb[p] + e / PART_PAGE] * PART_PAGE + e % PART_PAGE] = pr;
    }
}

// One partition per CTA iteration (partitions taken by ticket, in order):
//   1. 256-bp bucket histogram of the partition in shared memory, its pairs read from its pages (below)
//   2. one pass over every thread's strip of PER = BP / PF_THREADS consecutive buckets: keep flags by a sliding +-rb
//      window (the halo taken from the neighbours' edge counts -- the same rule as a genome-wide histogram; strips whose
//      windows stay inside the partition and reach only the neighbouring strips skip the halo tests) and the strip's
//      survivors; one CTA scan gives the partition's survivor total, published to the look-back at once, and every
//      strip's base
//   3. a second pass over the strip writes the exclusive offsets of the kept buckets and their flag bits; the pairs are
//      streamed again and every survivor is put into its bucket's slot range in the shared-memory stage (more than
//      PF_STAGE survivors: in `spill`, at the output's offsets)
//   4. order inside every bucket: rank against the bucket (<= FIX_SMALL members), or a counting sort on the low
//      BKT_SHIFT bits for larger buckets -> keys_out / idx_out at the partition's survivor base
// Bucket b is stored transposed, at phys(b) = (b % PER) * PF_THREADS + b / PER, so the threads reading the j-th bucket
// of their strips touch consecutive words.  Below PF_THREADS buckets (W = 16, BP = 256) PER is 1 and the threads at or
// past BP own an empty strip: run_indel's choice of W, and with it the partitions, stays what it is for small genomes,
// and the threads without a strip still load pairs and place survivors.  The look-back's exclusive base is awaited only
// where it is used: before the placement of a partition that spills, otherwise by warp 0 before its share of the
// placement, while the other warps place theirs.
// Both passes read the partition's ordinals e = 2 * thread, 2 * thread + 2 * PF_THREADS, .. two pairs (16 B) at a time,
// U loads in flight per thread: pool page pt[p][e / PART_PAGE] - 1, slot e % PART_PAGE.  One CTA step covers four pages,
// load u of a thread lying in page u / 2 of the step.  The page ids are read through L1: row p of the page table is read
// and reset by this CTA only.  Once both passes are done the CTA zeroes fill[p] and the entries of row p it read, which
// are exactly the ones the scatter set, so the next call starts from a clean table.
// 512 threads and 64 registers at most: two CTAs per SM fill its shared memory and its register file.
static constexpr int PF_THREADS = 512, PF_LT = 9;
static_assert(PF_THREADS == 1 << PF_LT, "k_part_filter: a power-of-two CTA");
static_assert((1 << (PART_W_MAX - BKT_SHIFT)) / PF_THREADS <= 64, "k_part_filter: a strip's keep flags fit one 64-bit word");
static_assert((1 << (PART_W_MIN - BKT_SHIFT)) % 32 == 0,
              "k_part_filter: below PF_THREADS buckets, one bucket per thread; whole warps own a strip or none");
__global__ void __launch_bounds__(PF_THREADS, 2) k_part_filter(const uint2* __restrict__ pool, uint32_t* __restrict__ fill, uint32_t* __restrict__ pt,
                                                     uint32_t ptw, int P, int W, int rb, uint32_t need, const uint32_t* __restrict__ edge, uint32_t* __restrict__ keys_out,
                                                     uint32_t* __restrict__ idx_out, uint2* __restrict__ spill, uint32_t* n_out, TileSync ts) {
    pdl_launch_dependents(); pdl_wait();
    extern __shared__ __align__(16) uint32_t s_dyn[];
    const int BP = 1 << (W - BKT_SHIFT);
    const int LPER = W - BKT_SHIFT > PF_LT ? W - BKT_SHIFT - PF_LT : 0, PER = 1 << LPER;   // PER buckets per strip
    uint32_t* s_h = s_dyn;                                        // BP words, bucket b at phys(b)
    uint32_t* s_f = s_dyn + BP;                                   // BP / 32 flag words, bit phys(b) % 32 of word phys(b) / 32
    uint2* s_st = reinterpret_cast<uint2*>(s_dyn + BP + BP / 32); // PF_STAGE pairs
    __shared__ uint32_t s_warp[PF_THREADS / 32 + 1];
    __shared__ uint32_t s_hl[BKT_PAD], s_hr[BKT_PAD];
    __shared__ uint32_t s_big[PF_BIG_CAP], s_cnt[256];
    __shared__ uint32_t s_tile, s_excl, s_nbig;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t gen = ts_gen(ts);
    const uint32_t bmask = BP - 1;
    auto phys = [&](uint32_t b) -> uint32_t { return ((b & (PER - 1)) << PF_LT) | (b >> LPER); };
    auto count = [&](int b) -> uint32_t { return s_h[phys(b)]; };
    const int b0 = (int)threadIdx.x * PER;                 // this thread's strip ..
    const int nst = (int)threadIdx.x < BP ? PER : 0;       // .. of nst buckets (uniform across a warp)
    while (true) {
        if (threadIdx.x == 0) { s_tile = atomicAdd(ts.ticket, 1u); s_nbig = 0; }
        for (int i = threadIdx.x; i < BP; i += PF_THREADS) s_h[i] = 0;
        __syncthreads();
        const int p = (int)s_tile;
        if (p >= P) break;
        if (threadIdx.x < 2 * BKT_PAD) {   // halo: s_hl[j] = the (j+1)-th last bucket of p-1, s_hr[j] = bucket j of p+1
            const int j = threadIdx.x % BKT_PAD, right = threadIdx.x / BKT_PAD;
            const int q = right ? p + 1 : p - 1;
            const bool ok = q >= 0 && q < P && j < rb;
            (right ? s_hr : s_hl)[j] = ok ? edge[(int64_t)q * 2 * BKT_PAD + (right ? 0 : BKT_PAD) + j] : 0u;
        }
        const uint32_t np = __ldcg(fill + p);
        uint32_t* row = pt + (size_t)p * ptw;
        auto walk = [&](auto f) {
            constexpr int U = 8;   // 16 B loads in flight per thread: a step of the CTA covers pages 4k .. 4k + 3 exactly
            static_assert(2 * PF_THREADS * U == 4 * PART_PAGE && 2 * PF_THREADS * 2 == PART_PAGE, "k_part_filter: four pages per step, two loads per page");
            for (uint32_t k = 0; 4 * PART_PAGE * k < np; k++) {
                const uint32_t e0 = 4 * PART_PAGE * k + 2 * threadIdx.x;
                uint32_t pg[4];   // pool pages of the step (page 4k + i past the partition's last: never read)
#pragma unroll
                for (int i = 0; i < 4; i++) pg[i] = PART_PAGE * (4 * k + i) < np ? __ldg(row + 4 * k + i) - 1u : 0u;
                uint4 v[U];
#pragma unroll
                for (int u = 0; u < U; u++) {
                    const uint32_t e = e0 + 2 * PF_THREADS * u;
                    v[u] = e < np ? __ldg(reinterpret_cast<const uint4*>(pool + (size_t)pg[u >> 1] * PART_PAGE + e % PART_PAGE))
                                  : make_uint4(0u, 0u, 0u, 0u);
                }
#pragma unroll
                for (int u = 0; u < U; u++) {
                    const uint32_t e = e0 + 2 * PF_THREADS * u;
                    if (e < np) f(make_uint2(v[u].x, v[u].y));
                    if (e + 1 < np) f(make_uint2(v[u].z, v[u].w));
                }
            }
        };
        // 1. histogram
        walk([&](uint2 pr) { atomicAdd(&s_h[phys((pr.x >> BKT_SHIFT) & bmask)], 1u); });
        __syncthreads();
        // 2. keep flags of the strip, the partition's survivor total and the strip's first slot.  Interior strips read the
        // transposed histogram straight: bucket b0 + s * PER + j of the strip s = -1, 0, 1 is at (j << PF_LT) + thread + s.
        uint32_t kept = 0, S;
        const uint64_t flags = nst ? pf_strip_flags(count, [&](int s, int j) -> uint32_t { return s_h[(j << PF_LT) + (int)threadIdx.x + s]; },
                                                    b0, PER, BP, rb, need, s_hl, s_hr, &kept)
                                   : 0ull;
        const uint32_t first = block_excl_scan<PF_THREADS>(kept, s_warp, &S);
        if (threadIdx.x == 0) {
            lookback_publish(ts.status, gen, p, S);
            if (S) atomicAdd(n_out, S);
        }
        const bool spilled = S > (uint32_t)PF_STAGE;
        if (spilled && warp == 0) {   // the spill area lies at the partition's output offsets
            const uint32_t ex = lookback_wait_warp(ts.status, gen, p, S);
            if (lane == 0) s_excl = ex;
        }
        // 3a. exclusive offsets of the kept buckets in place, their flag bits, the list of large buckets
        pf_strip_offsets([&](int b) -> uint32_t { return s_h[((b - b0) << PF_LT) | threadIdx.x]; }, b0, nst, flags, first,
                         [&](int j, uint32_t off, bool f, uint32_t c) {
            s_h[(j << PF_LT) | threadIdx.x] = off;   // phys(b0 + j)
            const uint32_t bits = __ballot_sync(0xffffffffu, f);
            if (lane == 0) s_f[(j << (PF_LT - 5)) | warp] = bits;
            if (c > FIX_SMALL) {
                const uint32_t q = atomicAdd(&s_nbig, 1u);
                if (q < PF_BIG_CAP) s_big[q] = (uint32_t)(b0 + j);
            }
        });
        __syncthreads();
        if (!spilled && warp == 0) {   // the other warps start placing meanwhile
            const uint32_t ex = lookback_wait_warp(ts.status, gen, p, S);
            if (lane == 0) s_excl = ex;
        }
        uint2* st = spilled ? spill + s_excl : s_st;
        // 3b. survivors into their buckets' slot ranges (afterwards s_h[phys(b)] = end of bucket b)
        walk([&](uint2 pr) {
            const uint32_t ph = phys((pr.x >> BKT_SHIFT) & bmask);
            if ((s_f[ph >> 5] >> (ph & 31)) & 1u) st[atomicAdd(&s_h[ph], 1u)] = pr;
        });
        __syncthreads();   // every page id and pair read
        for (uint32_t k = threadIdx.x; k < (np + PART_PAGE - 1) / PART_PAGE; k += PF_THREADS) row[k] = 0u;
        if (threadIdx.x == 0) fill[p] = 0u;
        const uint32_t obase = s_excl;
        // 4a. small buckets: rank against the bucket, ties by slot
        for (uint32_t q = threadIdx.x; q < S; q += PF_THREADS) {
            const uint2 pr = st[q];
            const uint32_t b = (pr.x >> BKT_SHIFT) & bmask;
            const uint32_t beg = b ? s_h[phys(b - 1)] : 0u, end = s_h[phys(b)];
            if (end - beg > FIX_SMALL) continue;
            uint32_t rank = 0;
            for (uint32_t j = beg; j < end; j++) {
                const uint32_t k = st[j].x;
                rank += (k < pr.x || (k == pr.x && j < q)) ? 1u : 0u;
            }
            keys_out[obase + beg + rank] = pr.x;
            idx_out[obase + beg + rank] = pr.y;
        }
        // 4b. large buckets: counting sort on the low BKT_SHIFT bits, one bucket at a time; the bins are threads 0 .. 255's
        static_assert((1 << BKT_SHIFT) == 256 && PF_THREADS >= 256, "one counting-sort bin per thread of the first 256");
        const uint32_t nbig = s_nbig;
        const uint32_t nb = nbig <= (uint32_t)PF_BIG_CAP ? nbig : (uint32_t)BP;   // list overflow: visit every bucket
        for (uint32_t k = 0; k < nb; k++) {
            const uint32_t b = nbig <= (uint32_t)PF_BIG_CAP ? s_big[k] : k;
            const uint32_t beg = b ? s_h[phys(b - 1)] : 0u, end = s_h[phys(b)];
            if (end - beg <= FIX_SMALL) continue;   // (uniform across the CTA)
            __syncthreads();
            if (threadIdx.x < 256) s_cnt[threadIdx.x] = 0;
            __syncthreads();
            for (uint32_t j = beg + threadIdx.x; j < end; j += PF_THREADS) atomicAdd(&s_cnt[st[j].x & 255u], 1u);
            __syncthreads();
            uint32_t total;
            const uint32_t ex = block_excl_scan<PF_THREADS>(threadIdx.x < 256 ? s_cnt[threadIdx.x] : 0u, s_warp, &total);
            if (threadIdx.x < 256) s_cnt[threadIdx.x] = ex;
            __syncthreads();
            for (uint32_t j = beg + threadIdx.x; j < end; j += PF_THREADS) {
                const uint2 pr = st[j];
                const uint32_t d = obase + beg + atomicAdd(&s_cnt[pr.x & 255u], 1u);
                keys_out[d] = pr.x;
                idx_out[d] = pr.y;
            }
        }
        __syncthreads();
    }
}

// small types: three sort keys per signature (name, second coordinate, primary)
// TRA_PAIR: k_prim receives only the TRA pair word chr1*4n + chr2*4+type, for contig counts at which the pair and pos1 do not
// fit one 64-bit key; k_tra_compact_key then replaces it by (dense rank of the pair, pos1)
template <bool TRA_PAIR>
__global__ void k_other_keys(const int32_t* __restrict__ chrom, const int32_t* __restrict__ a, const int32_t* __restrict__ b,
                             const int32_t* __restrict__ rid, const int32_t* __restrict__ c, int64_t n, int svtype, ContigTab ct,
                             uint32_t* __restrict__ k_rid, uint32_t* __restrict__ k_b, uint64_t* __restrict__ k_prim,
                             uint32_t* status) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        uint32_t bad = 0;
        const int32_t ch = chrom[i], ai = a[i], bi = b[i], ri = rid[i], ci = c ? c[i] : 0;
        if (ch < 0 || ch >= ct.n) bad |= ST_BAD_CHROM;
        else if (ct.len[ch] < 0) bad |= ST_BAD_POS;   // contig not owned by this shard
        if (ai < 0 || bi < 0 || ri < 0 || ci < 0) bad |= ST_NEG_FIELD;
        if (svtype == CSV_TRA && (ci >> 2) >= ct.n) bad |= ST_BAD_CHROM;
        if (svtype == CSV_INV && ci > 1) bad |= ST_NEG_FIELD;
        if (bad) atomicOr(status, bad);
        if (k_rid) { k_rid[i] = (uint32_t)ri; k_b[i] = (uint32_t)bi; }
        // (chr, a) for DUP cuteSV:783; (chr, strand, bp1) for INV cuteSV:792; (chr1, chr2, type, pos1) for TRA :801
        uint64_t hi = (uint64_t)(uint32_t)ch;
        if (svtype == CSV_INV) hi = hi * 2 + (uint32_t)ci;
        if (svtype == CSV_TRA) hi = hi * (uint64_t)(4 * ct.n) + (uint32_t)ci;   // chr2*4+type < 4*n_contigs
        k_prim[i] = TRA_PAIR ? hi : (hi << 31) | (uint32_t)ai;     // a < 2^31
    }
}

// flag[i] = 1 where the sorted TRA pair word changes after position i: the exclusive scan of the flags is the dense rank
// of pair[i] among the pairs present
__global__ void k_tra_pair_flags(const uint64_t* __restrict__ pair_sorted, int64_t n, uint32_t* __restrict__ flag) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        flag[i] = (i + 1 < n && pair_sorted[i + 1] != pair_sorted[i]) ? 1u : 0u;
}
// compact TRA primary key in input order: (rank of (chr1, chr2*4+type), pos1).  Ranks keep the pairs' order, so the key
// sorts, ties and runs exactly as (chr1, chr2*4+type, pos1) does.
__global__ void k_tra_compact_key(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ rank, const int32_t* __restrict__ a,
                                  int64_t n, uint64_t* __restrict__ k_prim) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t x = perm[i];
        k_prim[x] = ((uint64_t)rank[i] << 31) | (uint32_t)a[x];
    }
}

// Small types, second half of the tuple order: `perm` is sorted by the primary key only; inside every run of
// equal primary keys order by (b, name, input index) -- the rest of the reference's sort key (cuteSV:783,792,801) --
// by ranking each element against its run.  Runs are short (reads that report the same breakpoint); a run longer
// than RUN_MAX sets ST_BIG_RUN and the host reruns the type with the chained-sorts path.
static constexpr int RUN_MAX = 2048;
__global__ void __launch_bounds__(256) k_run_fixup(const uint64_t* __restrict__ kprim_sorted, const uint32_t* __restrict__ perm, int64_t n,
                                                   const int32_t* __restrict__ b, const int32_t* __restrict__ rid,
                                                   uint32_t* __restrict__ perm_out, uint32_t* status) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t k = kprim_sorted[i];
        const uint32_t x = perm[i];
        const bool alone = (i == 0 || kprim_sorted[i - 1] != k) && (i + 1 >= n || kprim_sorted[i + 1] != k);
        if (alone) { perm_out[i] = x; continue; }
        const int32_t bx = b[x], rx = rid[x];
        int64_t lo = i, hi = i + 1;
        uint32_t rank = 0;
        int seen = 1;
        auto less = [&](uint32_t y) { const int32_t by = b[y], ry = rid[y]; return by < bx || (by == bx && (ry < rx || (ry == rx && y < x))); };
        while (lo > 0 && kprim_sorted[lo - 1] == k && seen <= RUN_MAX) { rank += less(perm[lo - 1]) ? 1u : 0u; lo--; seen++; }
        while (hi < n && kprim_sorted[hi] == k && seen <= RUN_MAX) { rank += less(perm[hi]) ? 1u : 0u; hi++; seen++; }
        if (seen > RUN_MAX) { atomicOr(status, ST_BIG_RUN); perm_out[i] = x; continue; }
        perm_out[lo + rank] = x;
    }
}

// keys_out[i] = src[perm[i]] (perm == nullptr: identity)
template <typename K>
__global__ void k_gather_keys(const K* __restrict__ src, const uint32_t* __restrict__ perm, int64_t n, K* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = src[perm ? perm[i] : (uint32_t)i];
}

// small types: exact-duplicate removal (cuteSV:958-969) in the final order
struct DedupPred {
    const int32_t *chrom, *a, *b, *rid, *c;
    const uint32_t* perm;
    __device__ __forceinline__ bool operator()(int64_t i) const {
        if (i == 0) return true;
        const uint32_t x = perm[i], y = perm[i - 1];
        return !(chrom[x] == chrom[y] && a[x] == a[y] && b[x] == b[y] && rid[x] == rid[y] && (c ? c[x] == c[y] : true));
    }
};
// U columns = input columns gathered through perm[sel[k]]
__global__ void k_other_gather(const int32_t* __restrict__ chrom, const int32_t* __restrict__ a, const int32_t* __restrict__ b,
                               const int32_t* __restrict__ rid, const int32_t* __restrict__ c, const uint32_t* __restrict__ perm,
                               const uint32_t* __restrict__ sel, const uint32_t* n_sel, int32_t* u_chrom, int32_t* u_a, int32_t* u_b,
                               int32_t* u_rid, int32_t* u_c) {
    const int64_t n = *n_sel;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t x = perm[sel[k]];
        u_chrom[k] = chrom[x]; u_a[k] = a[x]; u_b[k] = b[x]; u_rid[k] = rid[x]; u_c[k] = c ? c[x] : 0;
    }
}

// ------------------------------------------------------------------------------------------
// cluster kernels
// ------------------------------------------------------------------------------------------
// KIND selects the one per-type routine a kernel instantiation contains (0 INS/DEL, 1 DUP, 2 INV, 3 TRA):
// one routine per kernel keeps the hot code inside the instruction cache.
__host__ __device__ constexpr int kind_of(int svtype) { return (svtype == CSV_DEL || svtype == CSV_INS) ? 0 : svtype == CSV_DUP ? 1 : svtype == CSV_INV ? 2 : 3; }
// KIND 4..7: INS / DEL with the type (and "every member is kept") fixed at compile time: DEL, INS, DEL keep-all, INS keep-all
template <int KIND, class Team>
__device__ __forceinline__ void run_cluster(Team tm, const TypeJob& J, int64_t s, int m, int M, char* arena, int64_t* red,
                                            uint32_t kslot, const Emit& E) {
    if (KIND == 4) indel_cluster<Team, CSV_DEL, 0>(tm, J.iv, s, m, M, arena, red, J.cp, J.svtype, kslot, E);
    else if (KIND == 5) indel_cluster<Team, CSV_INS, 0>(tm, J.iv, s, m, M, arena, red, J.cp, J.svtype, kslot, E);
    else if (KIND == 6) indel_cluster<Team, CSV_DEL, 1>(tm, J.iv, s, m, M, arena, red, J.cp, J.svtype, kslot, E);
    else if (KIND == 7) indel_cluster<Team, CSV_INS, 1>(tm, J.iv, s, m, M, arena, red, J.cp, J.svtype, kslot, E);
    else if (KIND == 0) indel_cluster(tm, J.iv, s, m, M, arena, red, J.cp, J.svtype, kslot, E);
    else if (KIND == 1) dup_cluster(tm, J.sv, s, m, M, arena, red, J.cp, kslot, E);
    else if (KIND == 2) inv_cluster(tm, J.sv, s, m, M, arena, red, J.cp, kslot, E);
    else tra_cluster(tm, J.sv, s, m, M, arena, red, J.cp, kslot, E);
}
__device__ __forceinline__ int arena_per(const TypeJob& J) {
    return (J.svtype == CSV_DEL || J.svtype == CSV_INS) ? INDEL_ARENA_PER : OTHER_ARENA_PER;
}
static constexpr int ARENA_PER_MAX = INDEL_ARENA_PER > OTHER_ARENA_PER ? INDEL_ARENA_PER : OTHER_ARENA_PER;

// size of the chain cluster starting at s, counting at most `limit`+1 members (warp-cooperative)
__device__ __forceinline__ int cluster_size_warp(const TypeJob& J, int64_t s, int64_t n, int limit) {
    const int lane = threadIdx.x & 31;
    int m = 1;
    while (m <= limit) {
        const int64_t i = s + m + lane;
        const bool brk = (i >= n) || !job_linked(J, i);
        const uint32_t mask = __ballot_sync(0xffffffffu, brk);
        if (mask) { m += __ffs(mask) - 1; return m; }
        m += 32;
    }
    return m;  // > limit
}

// ------------------------------------------------------------------------------------------
// INS / DEL clusters of at most 32 members, every member kept (remain_reads_ratio >= 1): the whole of
// generate_del_cluster / generate_ins_cluster (resolveINDEL.py:110-219, 319-432) in registers, one member per lane --
// no shared-memory arena, ~3x fewer instructions than the general routine (core.h indel_cluster) and, as a kernel of its
// own (k_cluster_small), a loop that stays inside the instruction cache (the general kernel spends most of its issue
// slots waiting for instructions: 47 KB of hot code, 24 warps per SM at different places in it).
//   exact duplicates / several signatures of one read: every lane looks at its peers (match.any on the read id); the
//   lowest lane of a read carries the read's entry = its longest signature (first of equal length in (pos, len, input)
//   order, resolveINDEL.py:125-131), ordered by the read's first occurrence (the dict order the stable sort by length
//   keeps): sort key (len_best, pos_first, len_first, name).
// 85 % of the kept clusters of 30x ONT have <= 32 members.
// ------------------------------------------------------------------------------------------
template <bool IS_INS>
__device__ __forceinline__ void indel_cluster_small(const IndelView& in, int64_t s, int m, const ClusterParams& P, uint32_t kslot, const Emit& E) {
    const int lane = (int)(threadIdx.x & 31);
    const bool act = lane < m;
    int32_t a = 0, len = 0, rid = -1 - lane, aux = 0;   // idle lanes: distinct negative ids
    uint32_t idx = 0;
    if (act) {
        if (in.rec) {
            const IndelRec r = in.rec[s + lane];
            a = r.a; len = r.b; rid = r.rid; idx = r.idx;
            if (IS_INS) aux = in.recc ? in.recc[s + lane] : 0;
        } else {
            idx = in.sidx[s + lane];
            a = in.a[idx]; len = in.b[idx]; rid = in.rid[idx];
            if (IS_INS) aux = in.c ? in.c[idx] : 0;
        }
    }
    const int32_t pos = IS_INS ? (a >> 1) : a;
    // the read's entry: best = its longest signature, first = its first occurrence in (pos, len, input index) order
    int32_t len_b = len, pos_b = pos, aux_b = aux, pos_f = pos, len_f = len;
    uint32_t idx_b = idx, idx_f = idx;
    bool rep = act;
    const uint32_t peers = __match_any_sync(0xffffffffu, rid);
    if (__any_sync(0xffffffffu, peers != (1u << lane))) {
        uint32_t rem = peers & ~(1u << lane);
        while (__any_sync(0xffffffffu, rem != 0u)) {
            const int j = rem ? __ffs(rem) - 1 : lane;
            rem &= rem - 1u;
            const int32_t pj = __shfl_sync(0xffffffffu, pos, j), lj = __shfl_sync(0xffffffffu, len, j), xj = __shfl_sync(0xffffffffu, aux, j);
            const uint32_t ij = __shfl_sync(0xffffffffu, idx, j);
            if (j != lane) {
                if (pj < pos_f || (pj == pos_f && (lj < len_f || (lj == len_f && ij < idx_f)))) { pos_f = pj; len_f = lj; idx_f = ij; }
                if (lj > len_b || (lj == len_b && (pj < pos_b || (pj == pos_b && ij < idx_b)))) { len_b = lj; pos_b = pj; aux_b = xj; idx_b = ij; }
            }
        }
        rep = act && (int)(__ffs(peers) - 1) == lane;   // one lane per read
    }
    const uint32_t reps = __ballot_sync(0xffffffffu, rep);
    const int u = __popc(reps);
    if (u < P.min_support) {   // len(read_tag) < read_count (:133); (the signature-count test :62 is implied)
        if (lane == 0) E.cnt[kslot] = 0;
        return;
    }
    // bitonic sort of the reads by (len_best, pos_first, len_first, name), carrying the lane that holds the entry
    uint64_t k0 = rep ? (((uint64_t)(uint32_t)len_b << 32) | (uint32_t)pos_f) : ~0ull;
    uint64_t k1 = rep ? (((uint64_t)(uint32_t)len_f << 32) | (uint32_t)rid) : ~0ull;
    int src = lane;
#pragma unroll 1
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll 1
        for (int j = k >> 1; j > 0; j >>= 1) {
            const uint64_t o0 = __shfl_xor_sync(0xffffffffu, k0, j), o1 = __shfl_xor_sync(0xffffffffu, k1, j);
            const int os = __shfl_xor_sync(0xffffffffu, src, j);
            const bool lower = (lane & j) == 0, up = (lane & k) == 0;
            const bool gt = k0 > o0 || (k0 == o0 && k1 > o1);
            const bool lt = k0 < o0 || (k0 == o0 && k1 < o1);
            if ((lower == up) ? gt : lt) { k0 = o0; k1 = o1; src = os; }
        }
    }
    // lane p < u now holds the read of sorted position p
    const bool act_s = lane < u;
    const int32_t len_s = (int32_t)(k0 >> 32), rid_s = (int32_t)(uint32_t)k1;
    const int32_t pos_s = __shfl_sync(0xffffffffu, pos_b, src);
    const int32_t aux_s = IS_INS ? __shfl_sync(0xffffffffu, aux_b, src) : 0;
    const uint32_t idx_s = IS_INS ? __shfl_sync(0xffffffffu, idx_b, src) : 0u;
    // allele split on the length-sorted reads (:137-162)
    int64_t sum_len = act_s ? (int64_t)len_s : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum_len += __shfl_xor_sync(0xffffffffu, sum_len, o);
    const double thr = P.ratio * ((double)sum_len / (double)u);
    const int32_t len_prev = __shfl_up_sync(0xffffffffu, len_s, 1);
    const bool brk = act_s && lane > 0 && (double)(len_s - len_prev) > thr;
    const uint32_t B = __ballot_sync(0xffffffffu, brk) | 1u;     // bit p: an allele starts at sorted position p
    const int na = __popc(B);
    // alleles in (support, order) order = sorted(allele_collect, key=[support]) stable (:163): lane q < na owns allele q
    int a_st = 0, a_n = 0, a_rank = 0;
    if (lane < na) {
        a_st = (int)__fns(B, 0, lane + 1);
        const int a_en = lane + 1 < na ? (int)__fns(B, 0, lane + 2) : u;
        a_n = a_en - a_st;
    }
    for (int q = 0; q < na; q++) {
        const int nq = __shfl_sync(0xffffffffu, a_n, q);
        if (lane < na && (nq < a_n || (nq == a_n && q < lane))) a_rank++;
    }
    uint32_t n_emit = 0;
    const int32_t chrom = in.chrom[in.rec ? in.rec[s].idx : in.sidx[s]];
    for (int k = 0; k < na; k++) {
        const uint32_t who = __ballot_sync(0xffffffffu, lane < na && a_rank == k);
        const int owner = __ffs(who) - 1;
        const int st = __shfl_sync(0xffffffffu, a_st, owner), n = __shfl_sync(0xffffffffu, a_n, owner);
        if (n < P.min_support_allele) continue;
        const bool mem = lane >= st && lane < st + n;
        int64_t sp = mem ? (int64_t)pos_s : 0, sl = mem ? (int64_t)len_s : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { sp += __shfl_xor_sync(0xffffffffu, sp, o); sl += __shfl_xor_sync(0xffffffffu, sl, o); }
        int32_t pos_out, search, aux_out = 0;
        if (IS_INS) {
            // first member (allele order) whose sequence is long enough (:399-405); signalLen = sl / n (every member kept)
            const int32_t need = (int32_t)((double)sl / (double)n);
            const uint32_t okm = __ballot_sync(0xffffffffu, mem && aux_s >= need);
            if (!okm) continue;   // ideal_ins_seq == '<INS>' -> dropped
            const int pick = __ffs(okm) - 1;
            pos_out = __shfl_sync(0xffffffffu, pos_s, pick);
            aux_out = (int32_t)__shfl_sync(0xffffffffu, idx_s, pick);
            search = pos_out;
        } else {
            // member closest to the mean position, index tie-break: |x - mean| ordered like |n*x - sum| (exact)
            int64_t d = (int64_t)n * pos_s - sp;
            if (d < 0) d = -d;
            uint64_t key = mem ? (((uint64_t)d << 5) | (uint32_t)(lane - st)) : ~0ull;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { const uint64_t y = __shfl_xor_sync(0xffffffffu, key, o); if (y < key) key = y; }
            search = __shfl_sync(0xffffffffu, pos_s, st + (int)(key & 31u));   // search_threshold (:177)
            pos_out = (int32_t)((double)sp / (double)n);
        }
        uint32_t slot = 0, noff = 0;
        if (lane == 0) emit_reserve_issue(E, (uint32_t)n, &slot, &noff);   // looked at after the std work
        // CIPOS / CILEN: np.std over the allele (:191-194), lanes 0-7 pos / 8-15 len = numpy's eight strided accumulators
        int32_t cipos, cilen;
        {
            const int which = (lane >> 3) & 1, j8 = lane & 7;
            const double mean = (double)(which ? sl : sp) / (double)n;
            auto sq = [&](int i) {
                const int32_t v0 = __shfl_sync(0xffffffffu, pos_s, (st + i) & 31), v1 = __shfl_sync(0xffffffffu, len_s, (st + i) & 31);
                const double x = (double)(which ? v1 : v0) - mean;
                return x * x;
            };
            double res;
            if (n < 8) {
                res = 0.;
                for (int i = 0; i < n; i++) res += sq(i);
            } else {
                const int n8 = n - (n % 8);
                double r = sq(j8);
                for (int i = 8 + j8; i < n8; i += 8) r += sq(i);
                r = r + __shfl_xor_sync(0xffffffffu, r, 1);
                r = r + __shfl_xor_sync(0xffffffffu, r, 2);
                r = r + __shfl_xor_sync(0xffffffffu, r, 4);
                res = r;
                for (int i = n8; i < n; i++) res += sq(i);
            }
            res = res / (double)n;
            const int32_t ci = cal_cipos(sqrt(res), n, E.pow_half);
            cipos = __shfl_sync(0xffffffffu, ci, 0);
            cilen = __shfl_sync(0xffffffffu, ci, 8);
        }
        int ok = 0;
        if (lane == 0) {
            note_support(E, (uint32_t)n);
            ok = emit_reserve_check(E, (uint32_t)n, slot, noff) ? 1 : 0;
        }
        ok = __shfl_sync(0xffffffffu, ok, 0);
        slot = __shfl_sync(0xffffffffu, slot, 0);
        noff = __shfl_sync(0xffffffffu, noff, 0);
        if (ok) {
            if (mem) E.names[noff + (uint32_t)(lane - st)] = rid_s;
            if (lane == 0) {
                const double signalLen = (double)sl / (double)n;
                csv_cand c;
                c.svtype = IS_INS ? CSV_INS : CSV_DEL; c.chrom = chrom; c.pos = pos_out;
                c.len = IS_INS ? (int32_t)signalLen : (int32_t)(-signalLen);
                c.support = n; c.cipos = cipos; c.cilen = cilen; c.search_pos = search; c.pos2 = 0; c.aux = aux_out;
                c.names_off = (int32_t)noff; c.names_cnt = n; c.cluster = (int32_t)kslot; c.flags = 0;
                c.reserved[0] = (int32_t)n_emit; c.reserved[1] = 0;
                E.cand[slot] = c;
            }
        }
        n_emit++;
    }
    if (lane == 0) E.cnt[kslot] = n_emit;
}

// one warp per kept cluster of <= 32 members.  Two ways in: (a) k_select_heads already sorted the kept clusters into
// `small_list` (ordinal, members) and `rest_list` while it gathered their records, so this kernel and the general kernel run
// side by side on two streams; (b) no lists (gather mode): every kept cluster is sized here and the larger ones are listed
// for the general kernel, which then runs after this one.
template <bool IS_INS>
__global__ void __launch_bounds__(256) k_cluster_small(TypeJob J, Emit E, Counters* ctr, uint32_t* work, uint32_t* n_rest) {
    pdl_launch_dependents(); pdl_wait();   // programmatic dependent launch: resident early, starts when the previous kernel has finished
    const int lane = threadIdx.x & 31;
    const int64_t n = job_n(J);
    const uint32_t n_todo = J.small_list ? *J.n_small : ctr->n_kept[J.svtype];
    uint32_t k_next = 0, n_done = 0, n_mem = 0;
    if (lane == 0) k_next = atomicAdd(work, 1u);
    while (true) {
        const uint32_t q = __shfl_sync(0xffffffffu, k_next, 0);
        if (q >= n_todo) break;
        if (lane == 0) k_next = atomicAdd(work, 1u);
        uint32_t k;
        int m;
        if (J.small_list) { const uint2 e = J.small_list[q]; k = e.x; m = (int)e.y; }
        else {
            k = q;
            m = cluster_size_warp(J, J.kept_start[k], n, 32);
            if (m > 32) {
                if (lane == 0) J.rest_list[atomicAdd(n_rest, 1u)] = k;   // (capacity = kept capacity of the type)
                continue;
            }
        }
        indel_cluster_small<IS_INS>(J.iv, J.kept_start[k], m, J.cp, J.kslot_base + k, E);
        n_done++; n_mem += (uint32_t)m;
    }
    if (lane == 0) {
        if (n_done) atomicAdd(&ctr->pad[0], n_done);
        if (n_mem) atomicAdd(&ctr->n_members[J.svtype], n_mem);
    }
}

// one warp per kept cluster; clusters larger than WARP_M are deferred to the CTA kernel
template <int KIND>
__global__ void __launch_bounds__(CL_THREADS) k_cluster_warp(TypeJob J, Emit E, Counters* ctr, uint32_t* work) {
    pdl_launch_dependents();   // the next kernel of the chain may become resident now (it waits for this grid to finish)
    extern __shared__ __align__(16) char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int WARPS = CL_THREADS / 32;
    char* arena = smem + (size_t)warp * (WARP_M * ARENA_PER_MAX);
    int64_t* red = (int64_t*)(smem + (size_t)WARPS * (WARP_M * ARENA_PER_MAX)) + warp * 40;
    const int64_t n = job_n(J);
    const uint32_t n_hi = J.rest_list ? *J.n_rest : ctr->n_kept[J.svtype];
    const uint32_t n_kept = n_hi + (J.n_rest_lo ? *J.n_rest_lo : 0u);
    CudaTeam<32> tm;
    // dynamic hand-out (one atomic per cluster): cluster costs vary, a static stride leaves a long tail
    // (the ticket of the NEXT cluster is requested before the current one is processed, so the atomic's round
    //  trip overlaps the work)
    uint32_t k_next = 0, n_mem = 0;
    if (lane == 0) k_next = atomicAdd(work, 1u);
    while (true) {
        const uint32_t q = __shfl_sync(0xffffffffu, k_next, 0);
        if (q >= n_kept) break;
        if (lane == 0) k_next = atomicAdd(work, 1u);
        // after k_cluster_small: only the clusters it left, the larger ones first
        const uint32_t k = !J.rest_list ? q : q < n_hi ? J.rest_list[q] : J.rest_list[J.rest_cap - 1u - (q - n_hi)];
        const int64_t s = J.kept_start[k];
        const int m = cluster_size_warp(J, s, n, WARP_M);
        if (m > WARP_M) {
            if (lane == 0) {
                const uint32_t o = atomicAdd(&ctr->n_big[J.svtype], 1u);
                if (o < J.big_cap) J.big_list[o] = k; else atomicOr(&ctr->status, ST_LIST_OVERFLOW);
            }
            continue;
        }
        n_mem += (uint32_t)m;
        run_cluster<KIND>(tm, J, s, m, pow2ceil(m), arena, red, J.kslot_base + k, E);
        __syncwarp();
    }
    if (lane == 0 && n_mem) atomicAdd(&ctr->n_members[J.svtype], n_mem);
}

// size of the chain cluster starting at s (CTA-cooperative, exact)
__device__ __forceinline__ int64_t cluster_size_block(const TypeJob& J, int64_t s, int64_t n, int64_t* red) {
    CudaTeam<CL_THREADS> tm;
    int64_t done = 1;
    while (true) {
        const int64_t i = s + done + threadIdx.x;
        const int64_t cand = ((i >= n) || !job_linked(J, i)) ? (done + threadIdx.x) : INT64_MAX;
        const int64_t first = team_min(tm, cand, red);
        if (first != INT64_MAX) return first;
        done += CL_THREADS;
    }
}

// one CTA per deferred cluster; clusters beyond the shared-memory arena (> BLOCK_M members) use global scratch
template <int KIND>
__global__ void __launch_bounds__(CL_THREADS) k_cluster_block(TypeJob J, Emit E, Counters* ctr) {
    pdl_launch_dependents(); pdl_wait();   // programmatic dependent launch: resident early, starts when the previous kernel has finished
    extern __shared__ __align__(16) char smem[];
    __shared__ int64_t red[CL_THREADS + 8];
    const int64_t n = job_n(J);
    const uint32_t n_list = min(ctr->n_big[J.svtype], J.big_cap);
    CudaTeam<CL_THREADS> tm;
    for (uint32_t q = blockIdx.x; q < n_list; q += gridDim.x) {
        const uint32_t k = J.big_list[q];
        const int64_t s = J.kept_start[k];
        const int64_t m = cluster_size_block(J, s, n, red);
        const bool giant = m > BLOCK_M;
        const int M = pow2ceil((int)m);
        if (threadIdx.x == 0) {
            atomicAdd(&ctr->n_members[J.svtype], (uint32_t)m);
            if (giant) atomicAdd(&ctr->n_giant[J.svtype], 1u);
        }
        // global scratch: clusters are disjoint ranges of the sorted order and M <= 2m
        char* arena = giant ? (J.giant_arena + (size_t)(2 * s) * ARENA_PER_MAX) : smem;
        run_cluster<KIND>(tm, J, s, (int)m, M, arena, red, J.kslot_base + k, E);
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------
// order: final position = (exclusive scan of per-cluster counts)[kslot] + emission rank
// ------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------
// genotype
// ------------------------------------------------------------------------------------------
// One genotype window, ready to be tested against a read: linear bounds of this window and (second window of DUP / INV
// only) of the candidate's first window, the slice of supporting read ids, the candidate index.  32 B = one sector.
struct alignas(16) WinRec { uint32_t S, E, S0, E0; int32_t names_off, names_cnt; uint32_t cand, second; };
struct GenoJob {
    csv_cand* cand;           // final order
    csv_geno* geno;
    const int32_t* names;
    const Counters* ctr;
    uint32_t cap_cand;
    ContigTab ct;
    GtParams gp;
    int shift;
    uint32_t n_bins;
    uint32_t* bin_start;      // n_bins + 1 (counts, then exclusive offsets)
    uint32_t* bin_fill;       // n_bins
    uint32_t* bin_bits;       // n_bins/32 + 1: bin holds at least one window (small, stays in L1)
    uint32_t* win_list;       // cand*2 + which, grouped by bin
    uint32_t win_cap;
    struct WinRec* win_rec;   // lin32 only: the same slots as 32 B records (window bounds in linear coordinates, names slice, cand)
    int lin32;                // the linear coordinate fits 32 bits: (read, window) pairs carry the read's coordinates
    uint32_t* dr;             // per candidate
    uint8_t* has_rows;        // per contig: reads table has rows (call_gt's `chr not in sigs_index["reads"]`)
    const csv_geno* gl_table;
    int genotype;
};

__device__ __forceinline__ uint32_t window_bin(const GenoJob& G, const csv_cand& c, int which) {
    int64_t s, e;
    window_of(c, which, G.gp, &s, &e);
    return (uint32_t)((G.ct.off[c.chrom] + (uint64_t)s) >> G.shift);
}

// candidates into the reference's emission order; when genotyping, the same pass counts the genotype windows per bin
__global__ void k_permute(const csv_cand* __restrict__ tmp, const uint32_t* __restrict__ base, Counters* ctr, uint32_t cap,
                          csv_cand* __restrict__ out, GenoJob G, const unsigned long long* cursor) {
    pdl_launch_dependents(); pdl_wait();   // programmatic dependent launch: resident early, starts when the previous kernel has finished
    const unsigned long long cur = *cursor;
    if (blockIdx.x == 0 && threadIdx.x == 0) { ctr->n_cand = (uint32_t)(cur >> 32); ctr->n_names = (uint32_t)cur; }   // for the kernels after this one
    const uint32_t n = min((uint32_t)(cur >> 32), cap);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        csv_cand c = tmp[i];
        const uint32_t dst = base[c.cluster] + (uint32_t)c.reserved[0];
        c.reserved[0] = 0;
        if (dst >= cap) continue;
        out[dst] = c;
        if (G.genotype) {
            const int nw = n_windows_of(c);
            for (int w = 0; w < nw; w++) {
                uint32_t b = window_bin(G, c, w);
                if (b >= G.n_bins) b = G.n_bins - 1;
                atomicAdd(&G.bin_start[b], 1u);
                atomicOr(&G.bin_bits[b >> 5], 1u << (b & 31));
            }
            G.dr[dst] = 0;
        }
    }
}

// pass 1: scatter the windows into their bins (bin_start already scanned; pass 0 = the counting is part of k_permute)
template <int PASS>
__global__ void k_windows(GenoJob G) {
    pdl_launch_dependents(); pdl_wait();   // programmatic dependent launch: resident early, starts when the previous kernel has finished
    const uint32_t n = min(G.ctr->n_cand, G.cap_cand);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const csv_cand c = G.cand[i];
        const int nw = n_windows_of(c);
        for (int w = 0; w < nw; w++) {
            uint32_t b = window_bin(G, c, w);
            if (b >= G.n_bins) b = G.n_bins - 1;
            if (PASS == 0) { atomicAdd(&G.bin_start[b], 1u); atomicOr(&G.bin_bits[b >> 5], 1u << (b & 31)); }
            else {
                const uint32_t o = G.bin_start[b] + atomicAdd(&G.bin_fill[b], 1u);
                if (o < G.win_cap) {
                    G.win_list[o] = i * 2u + (uint32_t)w;
                    if (G.lin32) {
                        const uint64_t coff = G.ct.off[c.chrom];
                        int64_t ws, we, s0 = 0, e0 = 0;
                        window_of(c, w, G.gp, &ws, &we);
                        if (w) window_of(c, 0, G.gp, &s0, &e0);
                        WinRec r;
                        r.S = (uint32_t)(coff + (uint64_t)ws); r.E = (uint32_t)(coff + (uint64_t)we);
                        r.S0 = (uint32_t)(coff + (uint64_t)s0); r.E0 = (uint32_t)(coff + (uint64_t)e0);
                        r.names_off = c.names_off; r.names_cnt = c.names_cnt; r.cand = i; r.second = (uint32_t)w;
                        *reinterpret_cast<uint4*>(&G.win_rec[o]) = *reinterpret_cast<const uint4*>(&r);
                        *(reinterpret_cast<uint4*>(&G.win_rec[o]) + 1) = *(reinterpret_cast<const uint4*>(&r) + 1);
                    }
                }
            }
        }
        if (PASS == 0) G.dr[i] = 0;
    }
}

// Is `rid` one of names[off, off + n)?  The slice is read as the 16 B-aligned quads that hold it, two per step (a names
// slice is about 22 ids on config 2: at most four steps instead of 22 scattered 4 B loads); ids of a quad outside the slice are
// masked out by index.  The quads stay inside the buffer: DBuf allocations end at least 256 B past the bytes asked for.
__device__ __forceinline__ bool names_contain(const int32_t* __restrict__ names, int32_t off, int32_t n, int32_t rid) {
    const int lead = off & 3;
    const int4* q = reinterpret_cast<const int4*>(names + (off - lead));
    const int end = lead + n;   // the slice is ints [lead, end) of the quads from q on
    bool found = false;
    for (int b = 0; b < end && !found; b += 8) {
        const int4 x = __ldg(q + (b >> 2));
        const int4 y = b + 4 < end ? __ldg(q + (b >> 2) + 1) : make_int4(0, 0, 0, 0);
        const int32_t v[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
#pragma unroll
        for (int k = 0; k < 8; k++) found |= v[k] == rid && b + k >= lead && b + k < end;
    }
    return found;
}

// One (read, window) test of assign_gt / overlap_cover: a primary read covers window [s,e] iff
// start <= s and end >= e (cuteSV_genotype.py:100-138); DR counts covering reads that are not
// supporting reads (:161-173).  RS/RE are linear coordinates.
__device__ __forceinline__ void test_pair(const GenoJob& G, uint64_t RS, uint64_t RE, int32_t rid, uint32_t w) {
    const uint32_t ent = G.win_list[w];
    const csv_cand c = G.cand[ent >> 1];
    const uint64_t coff = G.ct.off[c.chrom];
    int64_t s, e;
    window_of(c, (int)(ent & 1u), G.gp, &s, &e);
    if (!(RS <= coff + (uint64_t)s && RE >= coff + (uint64_t)e)) return;
    if (ent & 1u) {  // union of the two breakpoint covers (resolveDUP.py:155-157): count once
        int64_t s0, e0;
        window_of(c, 0, G.gp, &s0, &e0);
        if (RS <= coff + (uint64_t)s0 && RE >= coff + (uint64_t)e0) return;
    }
    if (!names_contain(G.names, c.names_off, c.names_cnt, rid)) atomicAdd(&G.dr[ent >> 1], 1u);   // supporting reads are not counted
}

// the same test on a WinRec (32-bit linear coordinates): one 32 B gather instead of the candidate record, its contig
// offset and the window arithmetic
__device__ __forceinline__ void test_pair32(const GenoJob& G, uint32_t RS, uint32_t RE, int32_t rid, uint32_t w) {
    const uint4 lo = __ldg(reinterpret_cast<const uint4*>(&G.win_rec[w])), hi = __ldg(reinterpret_cast<const uint4*>(&G.win_rec[w]) + 1);
    if (!(RS <= lo.x && RE >= lo.y)) return;
    if (hi.w && RS <= lo.z && RE >= lo.w) return;   // union of the two breakpoint covers (resolveDUP.py:155-157): count once
    if (!names_contain(G.names, (int32_t)hi.x, (int32_t)hi.y, rid)) atomicAdd(&G.dr[hi.z], 1u);
}

// ONE streaming pass over the reads table (replaces overlap_cover's event sort + sweep,
// cuteSV_genotype.py:95-159).  A read can only cover windows whose start lies in a bin it
// overlaps; most reads overlap no occupied bin (bit test on an L1-resident map).  The few
// (read, window) pairs that remain are compacted (warp-aggregated append) and tested by a second,
// dense kernel so that the streaming pass keeps all 32 lanes busy.
// LIN32 (linear coordinate < 2^32): a pair is 16 B (read start, read end, read id, window slot), so the dense kernel
// needs no gather into the reads table; otherwise 8 B (read row, window slot).
struct PairBuf { uint2* pairs; uint4* pairs4; uint32_t cap; uint32_t* count; };

template <bool LIN32>
__global__ void __launch_bounds__(256) k_reads_pass(GenoJob G, PairBuf PB, const int32_t* __restrict__ r_chrom,
                                                    const int32_t* __restrict__ r_start, const int32_t* __restrict__ r_end,
                                                    const int32_t* __restrict__ r_id, const uint8_t* __restrict__ r_prim,
                                                    int64_t n_reads, uint32_t* status) {
    // LIN32: linear coordinates and contig offsets in 32 bits (every offset < 2^32 - 4096, so ~0 stays a free marker)
    using Lin = typename std::conditional<LIN32, uint32_t, uint64_t>::type;
    pdl_launch_dependents(); pdl_wait();   // programmatic dependent launch: resident early, starts when the previous kernel has finished
    constexpr int ITEMS = 4;             // four consecutive rows per thread: one 128-bit load per column
    constexpr int TAB = 1024;            // contigs whose (offset, validity) live in shared memory
    constexpr Lin NO_OFF = ~(Lin)0;
    __shared__ uint32_t s_warp[17];
    __shared__ Lin s_off[TAB];           // linear offset, NO_OFF for a contig outside the shard
    __shared__ uint32_t s_lim[TAB];      // len + pad - 1: where a row's end is cut (the contig's linear range ends there)
    __shared__ uint8_t s_seen[TAB];
    const int n_tab = G.ct.n < TAB ? G.ct.n : TAB;
    for (int i = threadIdx.x; i < n_tab; i += 256) {
        s_off[i] = G.ct.len[i] < 0 ? NO_OFF : (Lin)G.ct.off[i];
        s_lim[i] = (uint32_t)(G.ct.off[i + 1] - G.ct.off[i] - 1);
        s_seen[i] = 0;
    }
    __syncthreads();
    const bool aligned = ((((uintptr_t)r_chrom) | ((uintptr_t)r_start) | ((uintptr_t)r_end) | ((uintptr_t)r_id)) & 15) == 0 &&
                         (((uintptr_t)r_prim) & 3) == 0;
    const int64_t n_tiles = (n_reads + 256 * ITEMS - 1) / (256 * ITEMS);
    // the columns of the thread's rows in the next tile: loaded one tile ahead, so that a tile's HBM latency overlaps the
    // probe, the reservation and the pair stores of the tile before it
    int32_t ch[ITEMS], st[ITEMS], en[ITEMS], id[ITEMS];
    uint32_t pr = 0;
    auto load = [&](int64_t tile) {
        const int64_t r0 = tile * 256 * ITEMS + (int64_t)threadIdx.x * ITEMS;
        if (aligned && r0 + ITEMS <= n_reads) {
            const int4 c4 = __ldcs(reinterpret_cast<const int4*>(r_chrom + r0)), s4 = __ldcs(reinterpret_cast<const int4*>(r_start + r0));
            const int4 e4 = __ldcs(reinterpret_cast<const int4*>(r_end + r0)), i4 = __ldcs(reinterpret_cast<const int4*>(r_id + r0));
            pr = __ldcs(reinterpret_cast<const uint32_t*>(r_prim + r0));
            ch[0] = c4.x; ch[1] = c4.y; ch[2] = c4.z; ch[3] = c4.w;
            st[0] = s4.x; st[1] = s4.y; st[2] = s4.z; st[3] = s4.w;
            en[0] = e4.x; en[1] = e4.y; en[2] = e4.z; en[3] = e4.w;
            id[0] = i4.x; id[1] = i4.y; id[2] = i4.z; id[3] = i4.w;
        } else {
            pr = 0;
#pragma unroll
            for (int j = 0; j < ITEMS; j++) {
                const int64_t r = r0 + j;
                const bool in = r < n_reads;
                ch[j] = in ? __ldcs(r_chrom + r) : -1; st[j] = in ? __ldcs(r_start + r) : 0; en[j] = in ? __ldcs(r_end + r) : 0;
                id[j] = in ? __ldcs(r_id + r) : 0;
                pr |= (uint32_t)(in ? __ldcs(r_prim + r) : 0) << (8 * j);
            }
        }
    };
    if ((int64_t)blockIdx.x < n_tiles) load(blockIdx.x);
    int parity = 0;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, parity ^= 1) {
        const int64_t r0 = tile * 256 * ITEMS + (int64_t)threadIdx.x * ITEMS;
        int32_t cid[ITEMS];
        uint32_t b0[ITEMS], b1[ITEMS];
        Lin RS[ITEMS], RE[ITEMS];
        // a primary row's linear range and bin range; a row that ends past its contig would reach the first windows of the
        // next contig in the linear coordinate: it ends at the last linear coordinate of its own contig instead (DESIGN §3:
        // exact for INS / DEL windows, which end there at the latest).  Both paths of the pair test (pair buffer and inline)
        // use this end.  Other rows get an empty bin range: no probe, no pairs.
        auto place = [&](int j, Lin off, uint32_t lim, bool prim) {
            RS[j] = off + (Lin)(uint32_t)st[j];
            RE[j] = off + (Lin)((uint32_t)en[j] > lim ? lim : (uint32_t)en[j]);
            b0[j] = prim ? (uint32_t)(RS[j] >> G.shift) : 1u;
            b1[j] = prim ? min((uint32_t)(RE[j] >> G.shift), G.n_bins - 1) : 0u;
        };
        // common case, one vote per warp: every row of the warp exists and is valid and its contig is in the shared table
        bool ok = r0 + ITEMS <= n_reads;
#pragma unroll
        for (int j = 0; j < ITEMS; j++)
            ok = ok && (uint32_t)ch[j] < (uint32_t)n_tab && s_off[ch[j]] != NO_OFF && st[j] >= 0 && en[j] >= st[j];
        if (__all_sync(0xffffffffu, ok)) {
#pragma unroll
            for (int j = 0; j < ITEMS; j++) {
                const int32_t c = ch[j];
                cid[j] = id[j];
                // deliberate benign race (racecheck reports it): a byte that only goes 0 -> 1, every writer stores the same
                // value, read after the final __syncthreads().  The race-free variants (shared atomics) cost registers, and
                // so resident CTAs, in this latency-bound pass.
                s_seen[c] = 1;
                place(j, s_off[c], s_lim[c], ((pr >> (8 * j)) & 0xffu) != 0);
            }
        } else {
#pragma unroll
            for (int j = 0; j < ITEMS; j++) {
                const int32_t c = ch[j], s = st[j], e = en[j];
                cid[j] = id[j];
                b0[j] = 1; b1[j] = 0; RS[j] = 0; RE[j] = 0;
                if (r0 + j >= n_reads) continue;
                if (c < 0 || c >= G.ct.n) { atomicOr(status, ST_BAD_CHROM); continue; }
                Lin off;
                uint32_t lim;
                if (c < TAB) {
                    off = s_off[c];
                    lim = s_lim[c];
                    if (!s_seen[c]) s_seen[c] = 1;
                } else {
                    off = G.ct.len[c] < 0 ? NO_OFF : (Lin)G.ct.off[c];
                    lim = (uint32_t)(G.ct.off[c + 1] - G.ct.off[c] - 1);
                    if (!G.has_rows[c]) G.has_rows[c] = 1;
                }
                if (off == NO_OFF) { atomicOr(status, ST_BAD_CHROM); continue; }   // outside the shard
                if (s < 0 || e < s) { atomicOr(status, ST_BAD_POS); continue; }
                place(j, off, lim, ((pr >> (8 * j)) & 0xffu) != 0);
            }
        }
        if ((int64_t)tile + gridDim.x < n_tiles) load(tile + gridDim.x);
        // any occupied bin in [b0, b1]?  The first and last words of the bit map for every row are loaded before any is
        // tested; a read spans at most two words unless it covers more than 32 bins.
        uint32_t m[ITEMS], m1[ITEMS];
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
            m[j] = m1[j] = 0;
            if (b0[j] <= b1[j]) {
                m[j] = __ldg(&G.bin_bits[b0[j] >> 5]);
                if ((b1[j] >> 5) != (b0[j] >> 5)) m1[j] = __ldg(&G.bin_bits[b1[j] >> 5]);
            }
        }
        uint32_t lo[ITEMS], hi[ITEMS];
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
            lo[j] = hi[j] = 0;
            if (b0[j] > b1[j]) continue;
            const uint32_t w0 = b0[j] >> 5, w1 = b1[j] >> 5;
            uint32_t x = m[j] & (0xffffffffu << (b0[j] & 31));
            if (w1 == w0) x &= 0xffffffffu >> (31 - (b1[j] & 31));
            else {
                x |= m1[j] & (0xffffffffu >> (31 - (b1[j] & 31)));
                for (uint32_t wi = w0 + 1; wi < w1 && !x; wi++) x = __ldg(&G.bin_bits[wi]);
            }
            if (x) { lo[j] = G.bin_start[b0[j]]; hi[j] = G.bin_start[b1[j] + 1]; }
        }
        uint32_t total = 0;
#pragma unroll
        for (int j = 0; j < ITEMS; j++) total += hi[j] - lo[j];
        uint32_t o = block_reserve_256(total, PB.count, s_warp, parity);
#pragma unroll
        for (int j = 0; j < ITEMS; j++) {
            const uint32_t cnt = hi[j] - lo[j];
            if (!cnt) continue;
            // slots below the capacity go to the pair buffer (every reserved slot < cap MUST be written:
            // k_pairs_test consumes [0, min(count, cap))); the rest is tested inline (correct, just slower)
            uint32_t k = 0;
            for (; k < cnt && (uint64_t)o + k < PB.cap; k++) {
                if (LIN32) PB.pairs4[o + k] = make_uint4((uint32_t)RS[j], (uint32_t)RE[j], (uint32_t)cid[j], lo[j] + k);
                else PB.pairs[o + k] = make_uint2((uint32_t)(r0 + j), lo[j] + k);
            }
            for (; k < cnt; k++) {
                if (LIN32) test_pair32(G, (uint32_t)RS[j], (uint32_t)RE[j], cid[j], lo[j] + k);
                else test_pair(G, RS[j], RE[j], cid[j], lo[j] + k);
            }
            o += cnt;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n_tab; i += 256)
        if (s_seen[i] && !G.has_rows[i]) G.has_rows[i] = 1;
}

template <bool LIN32>
__global__ void __launch_bounds__(256) k_pairs_test(GenoJob G, PairBuf PB, const int32_t* __restrict__ r_chrom,
                                                    const int32_t* __restrict__ r_start, const int32_t* __restrict__ r_end,
                                                    const int32_t* __restrict__ r_id) {
    pdl_launch_dependents(); pdl_wait();   // programmatic dependent launch: resident early, starts when the previous kernel has finished
    const uint32_t n = min(*PB.count, PB.cap);
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        if (LIN32) {
            const uint4 pr = PB.pairs4[p];
            test_pair32(G, pr.x, pr.y, (int32_t)pr.z, pr.w);
        } else {
            const uint2 pr = PB.pairs[p];
            const int32_t ch = r_chrom[pr.x];
            const uint64_t off = G.ct.off[ch];
            // the row's end clamped to its contig as in k_reads_pass (the pair carries only the row index)
            const uint64_t RE = min(off + (uint64_t)(uint32_t)r_end[pr.x], G.ct.off[ch + 1] - 1);
            test_pair(G, off + (uint64_t)(uint32_t)r_start[pr.x], RE, r_id[pr.x], pr.y);
        }
    }
}

__global__ void k_finalize(GenoJob G) {
    pdl_launch_dependents(); pdl_wait();   // programmatic dependent launch: resident early, starts when the previous kernel has finished
    const uint32_t n = min(G.ctr->n_cand, G.cap_cand);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        csv_cand c = G.cand[i];
        csv_geno g;
        g.dr = -1; g.dv = c.names_cnt; g.gt = -1; g.pl[0] = g.pl[1] = g.pl[2] = 0; g.gq = 0; g.status = 1; g.qual = 0.0;
        if (G.genotype && n_windows_of(c) > 0) {
            if (!G.has_rows[c.chrom]) {
                c.flags |= CSV_F_NO_READS;
                G.cand[i].flags = c.flags;
            } else {
                const int32_t dr = (int32_t)G.dr[i];
                g = G.gl_table[gl_index(dr, c.names_cnt)];  // cal_GL(DR, DV) (cuteSV_genotype.py:171)
                g.dr = dr; g.dv = c.names_cnt;
            }
        }
        G.geno[i] = g;
    }
}

// ---- TRA genotyping from the packed all-alignments table ----
__global__ void k_aln_index(const int32_t* __restrict__ chrom, const int32_t* __restrict__ start, const int32_t* __restrict__ end, int64_t n,
                            int32_t n_contigs, int32_t* max_span, uint32_t* status) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t c = chrom[i];
        if (c < 0 || c >= n_contigs) { atomicOr(status, ST_BAD_CHROM); continue; }
        if (i > 0 && (chrom[i - 1] > c || (chrom[i - 1] == c && start[i - 1] > start[i]))) atomicOr(status, ST_UNSORTED);
        atomicMax(&max_span[c], end[i] - start[i]);
    }
}
// off[c] = first row of contig c, i.e. the lower bound of c in the contig-sorted column, for c in [0, n_contigs]:
// one thread per contig (k_aln_index rejects a column that is not sorted)
__global__ void k_aln_off(const int32_t* __restrict__ chrom, int64_t n, int32_t n_contigs, uint32_t* __restrict__ off) {
    for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c <= n_contigs; c += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo = 0, hi = n;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (chrom[mid] < c) lo = mid + 1; else hi = mid;
        }
        off[c] = (uint32_t)lo;
    }
}
// Warp-cooperative count_coverage (core.h tra_count_coverage is the scalar statement the emulator runs):
// 32 consecutive BAM-order records per step; the running counters become ballot prefix counts and the
// record that triggers an early return is the lowest lane whose inclusive counts satisfy a return test.
__device__ __forceinline__ int tra_count_coverage_warp(const AlnView& A, int32_t chr, int64_t s, int64_t e, const int32_t* sup, int n_sup,
                                                       int32_t up_bound, int32_t itround, int32_t* nset, int32_t* dr, int64_t xs, int64_t xe) {
    const int lane = threadIdx.x & 31;
    const uint32_t below = (1u << lane) - 1u, upto = below | (1u << lane);
    int64_t iteration = 0, primary = 0;
    const uint32_t lo0 = A.off[chr], hi0 = A.off[chr + 1];
    uint32_t lo = lo0, hi = hi0;
    const int64_t min_start = s - (int64_t)A.max_span[chr];
    while (lo < hi) { uint32_t mid = lo + (hi - lo) / 2; if ((int64_t)A.start[mid] < min_start) lo = mid + 1; else hi = mid; }
    for (uint32_t base = lo; base < hi0; base += 32) {
        const uint32_t i = base + lane;
        const bool valid = i < hi0;
        const int64_t st = valid ? (int64_t)A.start[i] : 0, en = valid ? (int64_t)A.end[i] : 0;
        const bool before_end = valid && st < e;                  // loop condition (starts ascend: a prefix of the lanes)
        const bool fetched = before_end && en > s;
        const bool prim = fetched && A.prim[i] != 0;
        const bool spanning = prim && st < s && en > e;
        const bool fresh = spanning && !(xs <= xe && st < xs && en > xe);
        const bool is_ref = fresh && !sorted_contains(sup, n_sup, A.rid[i]);
        const uint32_t m_f = __ballot_sync(0xffffffffu, fetched), m_p = __ballot_sync(0xffffffffu, prim);
        const uint32_t m_n = __ballot_sync(0xffffffffu, fresh), m_r = __ballot_sync(0xffffffffu, is_ref);
        const int64_t it_incl = iteration + __popc(m_f & upto), pr_incl = primary + __popc(m_p & upto);
        const int32_t ns_incl = *nset + __popc(m_n & upto), dr_incl = *dr + __popc(m_r & upto);
        const bool ret_up = spanning && ns_incl >= up_bound;       // return 1 inside the spanning block
        const bool ret_round = prim && it_incl >= itround;         // the itround test is only reached by primary records
        const uint32_t m_ret = __ballot_sync(0xffffffffu, ret_up || ret_round);
        if (m_ret) {
            const int src = __ffs(m_ret) - 1;
            int code = ret_up ? 1 : (((double)pr_incl / (double)it_incl) <= 0.2 ? 1 : -1);
            code = __shfl_sync(0xffffffffu, code, src);
            *nset = __shfl_sync(0xffffffffu, ns_incl, src);
            *dr = __shfl_sync(0xffffffffu, dr_incl, src);
            return code;
        }
        iteration += __popc(m_f); primary += __popc(m_p);
        *nset += __popc(m_n); *dr += __popc(m_r);
        if (__ballot_sync(0xffffffffu, before_end) != 0xffffffffu) break;   // a record with start >= e (or the contig end) was seen
    }
    return 0;
}
struct TraCountCoverageWarp {
    __device__ __forceinline__ int operator()(const AlnView& A, int32_t chr, int64_t s, int64_t e, const int32_t* sup, int n_sup, int32_t up_bound,
                                              int32_t itround, int32_t* nset, int32_t* dr, int64_t xs, int64_t xe) const {
        return tra_count_coverage_warp(A, chr, s, e, sup, n_sup, up_bound, itround, nset, dr, xs, xe);
    }
};
// call_gt of one breakpoint pair by one warp (core.h tra_call_gt_rules); every lane returns the same csv_geno
__device__ __forceinline__ csv_geno tra_call_gt_warp(const AlnView& A, int32_t chr1, int64_t pos1, int32_t chr2, int64_t pos2, const int32_t* sup,
                                                     int32_t n_sup, int32_t bias, int32_t gt_round, const csv_geno* gl_table) {
    return tra_call_gt_rules(TraCountCoverageWarp{}, A, chr1, pos1, chr2, pos2, sup, n_sup, bias, gt_round, gl_table);
}
// one warp per TRA candidate; the candidates are ordered by SV type, TRA last, so warp w takes candidate n-1-w
__global__ void __launch_bounds__(128) k_tra_genotype(GenoJob G, AlnView A, int32_t bias, int32_t gt_round) {
    const uint32_t n = min(G.ctr->n_cand, G.cap_cand);
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (uint32_t w = warp; w < n; w += n_warps) {
        const uint32_t i = n - 1 - w;
        const csv_cand c = G.cand[i];
        if (c.svtype != CSV_TRA) break;   // uniform across the warp
        const csv_geno g = tra_call_gt_warp(A, c.chrom, c.pos, c.aux >> 2, c.pos2, G.names + c.names_off, c.names_cnt, bias, gt_round, G.gl_table);
        if (lane == 0) {
            G.geno[i] = g;
            G.cand[i].flags = c.flags & ~CSV_F_GT_HOST;
        }
    }
}

// csv_tra_call_gt: one warp per caller-given breakpoint pair; query i's supporting ids are sup[sup_off[i], sup_off[i + 1]), ascending
__global__ void __launch_bounds__(128) k_tra_call_gt(const csv_tra_query* __restrict__ q, uint32_t n, const int64_t* __restrict__ sup_off,
                                                     const int32_t* __restrict__ sup, AlnView A, int32_t bias, int32_t gt_round,
                                                     const csv_geno* __restrict__ gl_table, csv_geno* __restrict__ out) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < n; i += n_warps) {
        const csv_tra_query x = q[i];
        const int64_t so = sup_off[i];
        const csv_geno g = tra_call_gt_warp(A, x.chr1, x.pos1, x.chr2, x.pos2, sup + so, (int32_t)(sup_off[i + 1] - so), bias, gt_round, gl_table);
        if ((threadIdx.x & 31) == 0) out[i] = g;
    }
}

// cal_GL for arbitrary (c0, c1) pairs: special cases + rescale on the device, libm part from the table
__global__ void k_cal_gl(const int32_t* c0, const int32_t* c1, int64_t n, const csv_geno* gl_table, csv_geno* out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        csv_geno g = gl_table[gl_index(c0[i], c1[i])];
        g.dr = c0[i]; g.dv = c1[i];
        out[i] = g;
    }
}

// ---- standalone overlap_cover / call_gt (csv_overlap_cover, csv_call_gt) ----
// Windows are listed in every bin they span (per-contig bin ranges from bin_base), so a row that starts inside a window
// finds it too; every (row, window) pair is taken once, in the bin of max(row start, window start) (core.h gc_*).
// A count pass, exclusive scans and a fill pass build per-window CSR lists of name ids; each segment is then sorted and
// deduplicated by one warp (short) or one CTA (pile-ups).
struct GcJob {
    const csv_window* win;
    uint32_t n_win;
    const uint32_t* bin_base;   // n_wc + 1: first bin of every window contig
    int32_t n_wc;
    uint32_t* bin_start;        // counts, then exclusive offsets (n_bins + 1)
    uint32_t* bin_fill;
    uint32_t* bin_list;         // window ids grouped by bin
    uint32_t* iter;             // overlapping rows per window
    uint32_t* prim;             // overlapping primary rows per window
    uint32_t* cov_off;          // counts, then raw segment offsets (n_win + 1)
    uint32_t* ovl_off;
    uint32_t* cov_fill;
    uint32_t* ovl_fill;
    int32_t* cov_raw;           // name ids, unordered inside a segment
    int32_t* ovl_raw;
    int want_overlap;
};
struct GcReads { const int32_t *chrom, *start, *end, *rid; const uint8_t* prim; int64_t n; };

template <int PASS>
__global__ void __launch_bounds__(256) k_gc_win_bins(GcJob J) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < J.n_win; i += gridDim.x * blockDim.x) {
        const csv_window w = J.win[i];
        const uint32_t base = J.bin_base[w.chrom];
        const uint32_t b0 = base + (uint32_t)gc_bin(w.s2), b1 = base + (uint32_t)gc_bin(w.e2 - 1);
        for (uint32_t b = b0; b <= b1; b++) {
            if (PASS == 0) atomicAdd(&J.bin_start[b], 1u);
            else J.bin_list[J.bin_start[b] + atomicAdd(&J.bin_fill[b], 1u)] = i;
        }
    }
}

// one thread per row: PASS 0 counts, PASS 1 writes the name ids of primary rows into the raw segments
template <int PASS>
__global__ void __launch_bounds__(256) k_gc_pairs(GcJob J, GcReads R, uint32_t* status) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < R.n; r += (int64_t)gridDim.x * blockDim.x) {
        const int32_t ch = R.chrom[r], st = R.start[r], en = R.end[r];
        if (ch < 0 || en < st) { if (PASS == 0) atomicOr(status, ch < 0 ? ST_BAD_CHROM : ST_BAD_POS); continue; }
        if (ch >= J.n_wc) continue;
        const uint32_t base = J.bin_base[ch], nb = J.bin_base[ch + 1] - base;
        const int64_t rs2 = 2 * (int64_t)st, re2 = 2 * (int64_t)en;
        const int64_t b0 = gc_bin(rs2);
        if ((uint64_t)b0 >= nb) continue;
        int64_t b1 = gc_bin(re2);
        if (b1 >= (int64_t)nb) b1 = nb - 1;
        const bool pr = R.prim[r] != 0;
        const int32_t rid = R.rid[r];
        for (int64_t b = b0; b <= b1; b++) {
            const uint32_t k1 = J.bin_start[base + b + 1];
            for (uint32_t k = J.bin_start[base + b]; k < k1; k++) {
                const uint32_t wi = J.bin_list[k];
                const csv_window w = J.win[wi];
                if (!gc_overlaps(rs2, re2, w.s2, w.e2) || !gc_pair_home(rs2, w.s2, b)) continue;
                const bool cov = pr && gc_covers(rs2, re2, w.s2, w.e2);
                if (PASS == 0) {
                    atomicAdd(&J.iter[wi], 1u);
                    if (pr) atomicAdd(&J.prim[wi], 1u);
                    if (pr && J.want_overlap) atomicAdd(&J.ovl_off[wi], 1u);
                    if (cov) atomicAdd(&J.cov_off[wi], 1u);
                } else {
                    if (pr && J.want_overlap) J.ovl_raw[J.ovl_off[wi] + atomicAdd(&J.ovl_fill[wi], 1u)] = rid;
                    if (cov) J.cov_raw[J.cov_off[wi] + atomicAdd(&J.cov_fill[wi], 1u)] = rid;
                }
            }
        }
    }
}

// Sort + deduplicate segments [off[k], off[k+1]) of raw into ded at the same offsets; ucnt[k] = distinct ids.
// k_gc_dedup_warp takes the segments of at most GC_WARP_SEG ids, k_gc_dedup_cta the longer ones.
static constexpr uint32_t GC_WARP_SEG = 64;
__global__ void __launch_bounds__(256) k_gc_dedup_warp(const uint32_t* __restrict__ off, const int32_t* raw, uint32_t n_seg, uint8_t* flag,
                                                       int32_t* ded, uint32_t* ucnt) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    CudaTeam<32> tm;
    for (uint32_t k = warp; k < n_seg; k += n_warps) {
        const uint32_t o = off[k], n = off[k + 1] - o;
        if (n > GC_WARP_SEG) continue;
        const int u = gc_sort_unique(tm, raw + o, (int)n, flag + o, ded + o);
        if (tm.tid() == 0) ucnt[k] = (uint32_t)u;
    }
}
__global__ void __launch_bounds__(256) k_gc_dedup_cta(const uint32_t* __restrict__ off, const int32_t* raw, uint32_t n_seg, uint8_t* flag,
                                                      int32_t* ded, uint32_t* ucnt) {
    CudaTeam<256> tm;
    for (uint32_t k = blockIdx.x; k < n_seg; k += gridDim.x) {
        const uint32_t o = off[k], n = off[k + 1] - o;
        if (n <= GC_WARP_SEG) continue;
        const int u = gc_sort_unique(tm, raw + o, (int)n, flag + o, ded + o);
        if (tm.tid() == 0) ucnt[k] = (uint32_t)u;
    }
}

// call_gt's genotype per candidate: DR from the deduplicated cover segments of its windows (per consecutive windows,
// united) minus its ascending support ids, DV = support list length, then cal_GL from the table
__global__ void __launch_bounds__(256) k_gc_call_gt(const uint32_t* __restrict__ cov_off, const uint32_t* __restrict__ cov_u,
                                                    const int32_t* __restrict__ ded, int64_t n_cand, int per,
                                                    const int64_t* __restrict__ sup_off, const int32_t* __restrict__ sup,
                                                    const csv_geno* __restrict__ gl_table, csv_geno* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_cand; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t w0 = i * per, w1 = per == 2 ? w0 + 1 : w0;
        const int n1 = per == 2 ? (int)cov_u[w1] : 0;
        const int64_t so = sup_off[i];
        const int32_t dv = (int32_t)(sup_off[i + 1] - so);
        const int32_t dr = gc_union_minus(ded + cov_off[w0], (int)cov_u[w0], ded + cov_off[w1], n1, sup + so, dv);
        csv_geno g = gl_table[gl_index(dr, dv)];
        g.dr = dr; g.dv = dv;
        out[i] = g;
    }
}

}  // namespace csv
