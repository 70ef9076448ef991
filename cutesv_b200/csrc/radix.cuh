// radix.cuh -- stable LSD radix sort of (key, u32 payload) pairs, 8 bits per pass, one kernel per
// pass ("onesweep": per-digit chained scan with decoupled look-back), plus one up-front
// histogram kernel for all passes.
//
// This is kernel (b)'s front half of the north star: it replaces the Timsort of
// process_process_sigs_type (cuteSV:764-801).  HBM-bound integer work: per pass each pair is
// read once and written once; scatter is staged through shared memory so that every digit's run
// is written with consecutive threads -> coalesced stores.
#pragma once
#include "devprims.cuh"

namespace csv {

static constexpr int RS_THREADS = 256;
static constexpr int RS_WARPS = RS_THREADS / 32;
static constexpr int RS_MAX_PASSES = 8;

// Peer mask of the lanes holding the same 8-bit digit, built from 8 warp votes.  MATCH.ANY is a
// long-latency, low-throughput instruction; eight VOTE.BALLOTs pipeline and cost less.
__device__ __forceinline__ uint32_t match_digit8(uint32_t d) {
    uint32_t ret = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < 8; b++) {
        uint32_t mask;
        asm volatile(
            "{\n"
            "  .reg .pred p;\n"
            "  and.b32 %0, %1, %2;\n"
            "  setp.ne.u32 p, %0, 0;\n"
            "  vote.sync.ballot.b32 %0, p, 0xffffffff;\n"
            "  @!p not.b32 %0, %0;\n"
            "}\n"
            : "=r"(mask)
            : "r"(d), "r"(1u << b));
        ret &= mask;
    }
    return ret;
}

template <typename K> struct RsTraits;
template <> struct RsTraits<uint32_t> { static constexpr int ITEMS = 16; };
template <> struct RsTraits<uint64_t> { static constexpr int ITEMS = 12; };

// histograms of every pass in one read of the keys: hist[p*256 + d]
template <typename K>
__global__ void __launch_bounds__(RS_THREADS) k_rs_hist(const K* __restrict__ keys, int64_t n_host, const uint32_t* n_dev,
                                                        int passes, uint32_t* __restrict__ hist) {
    __shared__ uint32_t s_hist[RS_MAX_PASSES * 256];
    const int64_t n = n_dev ? (int64_t)*n_dev : n_host;
    for (int i = threadIdx.x; i < passes * 256; i += RS_THREADS) s_hist[i] = 0;
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * RS_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * RS_THREADS) {
        const K k = keys[i];
        for (int p = 0; p < passes; p++) atomicAdd(&s_hist[p * 256 + (int)((k >> (8 * p)) & 0xff)], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < passes * 256; i += RS_THREADS) {
        const uint32_t v = s_hist[i];
        if (v) atomicAdd(&hist[i], v);
    }
}

// hist[p][*] -> exclusive digit offsets (in place). One CTA of 256 threads.
__global__ void __launch_bounds__(256) k_rs_hist_scan(uint32_t* hist, int passes) {
    __shared__ uint32_t s_warp[9];
    for (int p = 0; p < passes; p++) {
        const uint32_t v = hist[p * 256 + threadIdx.x];
        uint32_t total;
        const uint32_t e = block_excl_scan<256>(v, s_warp, &total);
        hist[p * 256 + threadIdx.x] = e;
    }
}

// One pass.  status: n_tiles * 256 generation-tagged words (never cleared), ticket: 1 word (zeroed).
// IOTA: the payload of element i is i itself (first pass; saves one column read).
template <typename K, bool IOTA>
__global__ void __launch_bounds__(RS_THREADS, 4) k_rs_onesweep(const K* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                                                            K* __restrict__ keys_out, uint32_t* __restrict__ vals_out,
                                                            int64_t n_host, const uint32_t* n_dev, int shift,
                                                            const uint32_t* __restrict__ gbase, TileSync ts) {
    constexpr int ITEMS = RsTraits<K>::ITEMS;
    constexpr int TILE = RS_THREADS * ITEMS;
    __shared__ uint32_t s_warp_hist[RS_WARPS][256];
    __shared__ uint32_t s_excl[256];      // local exclusive offset of each digit inside the tile
    __shared__ int64_t s_dst[256];        // global destination of local position 0 of each digit run
    __shared__ K s_keys[TILE];
    __shared__ uint32_t s_vals[TILE];
    __shared__ uint32_t s_scan[9];
    __shared__ uint32_t s_tile;

    const int64_t n = n_dev ? (int64_t)*n_dev : n_host;
    const uint32_t gen = ts_gen(ts);
    uint64_t* const status = ts.status;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(ts.ticket, 1u);
    for (int i = tid; i < RS_WARPS * 256; i += RS_THREADS) (&s_warp_hist[0][0])[i] = 0;
    __syncthreads();
    const int tile = (int)s_tile;
    const int64_t base = (int64_t)tile * TILE;
    if (base >= n) return;
    const int n_valid = (int)((n - base) < TILE ? (n - base) : TILE);

    // warp-striped load: position inside the tile = warp*32*ITEMS + i*32 + lane
    K k[ITEMS];
    uint32_t rank[ITEMS];
    const int wbase = warp * 32 * ITEMS;
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
        const int p = wbase + i * 32 + lane;
        k[i] = p < n_valid ? keys_in[base + p] : (K)~(K)0;
    }
    // stable rank of every key among equal digits of the same warp.  The peer masks are
    // independent of each other: issue all MATCH instructions first so their latency overlaps,
    // then run the (inherently serial) per-warp counter chain.
    uint32_t pm[ITEMS];
#pragma unroll
    for (int i = 0; i < ITEMS; i++) pm[i] = match_digit8((uint32_t)((k[i] >> shift) & 0xff));
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
        const int d = (int)((k[i] >> shift) & 0xff);
        const uint32_t peers = pm[i];
        const int leader = __ffs(peers) - 1;
        uint32_t prev = 0;
        if (lane == leader) {
            prev = s_warp_hist[warp][d];
            s_warp_hist[warp][d] = prev + __popc(peers);
        }
        prev = __shfl_sync(0xffffffffu, prev, leader);
        rank[i] = prev + __popc(peers & ((1u << lane) - 1u));
        __syncwarp();
    }
    __syncthreads();
    // digit `tid`: exclusive scan over warps, tile total, look-back, destinations
    {
        const int d = tid;
        uint32_t sum = 0;
#pragma unroll
        for (int w = 0; w < RS_WARPS; w++) {
            const uint32_t t = s_warp_hist[w][d];
            s_warp_hist[w][d] = sum;
            sum += t;
        }
        uint32_t total;
        const uint32_t excl_local = block_excl_scan<256>(sum, s_scan, &total);
        s_excl[d] = excl_local;
        // chained scan of this digit's count over tiles: thread d walks back over the tiles,
        // LB_BATCH predecessors per step (independent loads in flight), so that a wave of W
        // concurrently running tiles costs W/LB_BATCH dependent L2 round trips.
        uint64_t* st = status + d;
        uint32_t excl_tiles = 0;
        if (tile == 0) {
            lb_store(st, lb_word(gen, true, sum));
        } else {
            lb_store(st + (size_t)tile * 256, lb_word(gen, false, sum));
            constexpr int LB_BATCH = 8;
            int p = tile - 1;
            bool done = false;
            while (!done) {
                uint64_t v[LB_BATCH];
#pragma unroll
                for (int j = 0; j < LB_BATCH; j++) {
                    const int q = p - j;
                    v[j] = q >= 0 ? lb_load(st + (size_t)q * 256) : lb_word(gen, true, 0u);
                }
                int used = 0;
#pragma unroll
                for (int j = 0; j < LB_BATCH; j++) {
                    if (!done && used == j && lb_ready(v[j], gen)) {
                        excl_tiles += lb_value(v[j]);
                        used = j + 1;
                        if (lb_inclusive(v[j])) done = true;
                    }
                }
                p -= used;  // used == 0: nearest predecessor not published yet -> poll again
            }
            lb_store(st + (size_t)tile * 256, lb_word(gen, true, excl_tiles + sum));
        }
        s_dst[d] = (int64_t)gbase[d] + (int64_t)excl_tiles - (int64_t)excl_local;
    }
    __syncthreads();
    // local scatter into digit order
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
        const int p = wbase + i * 32 + lane;
        const int d = (int)((k[i] >> shift) & 0xff);
        const uint32_t pos = s_excl[d] + s_warp_hist[warp][d] + rank[i];
        s_keys[pos] = k[i];
        uint32_t v = 0;
        if (p < n_valid) v = IOTA ? (uint32_t)(base + p) : vals_in[base + p];
        s_vals[pos] = v;
    }
    __syncthreads();
    // coalesced write-out: consecutive threads write consecutive slots of each digit run.
    // Padding keys (all ones) are the last local positions, i.e. >= n_valid.
#pragma unroll
    for (int i = 0; i < ITEMS; i++) {
        const int p = i * RS_THREADS + tid;
        if (p < n_valid) {
            const K key = s_keys[p];
            const int d = (int)((key >> shift) & 0xff);
            const int64_t dst = s_dst[d] + p;
            keys_out[dst] = key;
            vals_out[dst] = s_vals[p];
        }
    }
}

}  // namespace csv
