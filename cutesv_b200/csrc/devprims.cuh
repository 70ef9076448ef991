// devprims.cuh -- device-wide building blocks: decoupled look-back, ordered select, exclusive scan.
//
// All kernels here take their element count either from the host (n_host) or from a device
// counter written by an earlier kernel (n_dev != nullptr), so that the whole pipeline can be
// enqueued without any host round trip.  Tiles are handed out by an atomic ticket, which makes
// the spin-wait of the look-back safe: every lower ticket belongs to a CTA that already runs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace csv {

// Programmatic dependent launch (sm_90+): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may
// become resident while its stream predecessor still runs; it must not touch memory before pdl_wait(), which returns once
// the predecessor grid has completed and its writes are visible.  pdl_launch_dependents() lets the NEXT kernel do the same
// with respect to this one.  Both are no-ops for a kernel launched the ordinary way.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// 1-D TMA (cp.async.bulk) into shared memory + mbarrier: a copy's completion is signalled to the barrier in transaction
// bytes.  bulk_load = the arrival that expects `bytes` + the copy; several copies on one barrier take one
// mbar_expect_tx for their sum and bulk_copy each.  Sizes and addresses are multiples of 16 B.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
                 "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    mbar_expect_tx(bar, bytes);
    bulk_copy(dst, src, bytes, bar);
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        "  .reg .pred p;\n"
        "WAIT_%=:\n"
        "  mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "  @!p bra WAIT_%=;\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}


// Status words are 64-bit: [generation:31][inclusive:1][value:32].  A word is published when its generation is the
// launch's; the value is the tile's own total (inclusive = 0) or the sum over tiles 0..tile (inclusive = 1), so a tile
// total or a prefix may take all 32 bits (sums wrap modulo 2^32, as the scans' uint32 outputs do).  Every launch that uses
// the look-back gets a fresh generation in [1, LB_GEN_LIMIT), so the status buffer never has to be cleared: words of other
// generations, and zeroed words (generation 0, never issued), read as "not published yet".
static constexpr uint32_t LB_GEN_LIMIT = 1u << 31;
__device__ __forceinline__ uint64_t lb_word(uint32_t gen, bool inclusive, uint32_t value) {
    return ((uint64_t)gen << 33) | ((uint64_t)inclusive << 32) | value;
}
__device__ __forceinline__ bool lb_ready(uint64_t v, uint32_t gen) { return (uint32_t)(v >> 33) == gen; }
__device__ __forceinline__ bool lb_inclusive(uint64_t v) { return (v >> 32) & 1u; }
__device__ __forceinline__ uint32_t lb_value(uint64_t v) { return (uint32_t)v; }
// gpu-scope relaxed accesses: coherent at L2, no L1 caching, cheaper than volatile (.sys)
__device__ __forceinline__ uint64_t lb_load(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void lb_store(uint64_t* p, uint64_t v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Publishes `local` for `tile` (one thread calls it); lookback_wait_warp later returns the tile's exclusive prefix.
// Splitting the two lets a CTA do other work while its predecessors publish.
__device__ __forceinline__ void lookback_publish(uint64_t* status, uint32_t gen, int tile, uint32_t local) {
    lb_store(status + tile, lb_word(gen, tile == 0, local));
}

// Warp-cooperative wait (all 32 lanes of ONE warp call it) after lookback_publish(status, gen, tile, local): returns
// the exclusive prefix over tiles < tile to every lane.  32 predecessors are inspected per step, so a wave of W
// concurrently running tiles costs W/32 dependent L2 round trips instead of W.
__device__ __forceinline__ uint32_t lookback_wait_warp(uint64_t* status, uint32_t gen, int tile, uint32_t local) {
    const int lane = threadIdx.x & 31;
    if (tile == 0) return 0;
    uint32_t excl = 0;
    int p = tile - 1;
    while (true) {
        const int q = p - lane;
        const uint64_t v = q >= 0 ? lb_load(status + q) : lb_word(gen, true, 0u);   // before tile 0: an inclusive zero
        const bool ready = lb_ready(v, gen);
        const uint32_t nr = __ballot_sync(0xffffffffu, !ready);
        const uint32_t inc = __ballot_sync(0xffffffffu, ready && lb_inclusive(v));
        const int first_nr = nr ? __ffs(nr) - 1 : 32;
        const int first_inc = inc ? __ffs(inc) - 1 : 32;
        const bool done = first_inc < first_nr;
        const int upto = done ? first_inc + 1 : first_nr;  // lanes [0, upto) are consumed
        uint32_t contrib = lane < upto ? lb_value(v) : 0u;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
        excl += contrib;
        if (done) break;
        p -= upto;  // upto == 0: the nearest predecessor has not published yet -> poll again
    }
    if (lane == 0) lb_store(status + tile, lb_word(gen, true, excl + local));
    return excl;
}

// Both at once: publishes `local` for `tile` and returns its exclusive prefix (all 32 lanes of ONE warp call it).
__device__ __forceinline__ uint32_t lookback_exclusive_warp(uint64_t* status, uint32_t gen, int tile, uint32_t local) {
    if ((threadIdx.x & 31) == 0) lookback_publish(status, gen, tile, local);
    return lookback_wait_warp(status, gen, tile, local);
}

// exclusive scan of one value per thread across an NT-thread CTA (NT = 64 .. 1024, a multiple of 32); returns exclusive
// prefix, *total = CTA sum.  s_warp: NT / 32 + 1 words of shared memory.
template <int NT>
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* s_warp, uint32_t* total) {
    static_assert(NT % 32 == 0 && NT >= 64 && NT <= 1024, "block_excl_scan: whole warps, at most 32");
    constexpr int NW = NT / 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += y;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < NW ? s_warp[lane] : 0;
        uint32_t wi = w;
#pragma unroll
        for (int d = 1; d < NW; d <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, wi, d);
            if (lane >= d) wi += y;
        }
        if (lane < NW) s_warp[lane] = wi - w;
        if (lane == NW - 1) s_warp[NW] = wi;
    }
    __syncthreads();
    uint32_t r = s_warp[warp] + incl - v;
    *total = s_warp[NW];
    __syncthreads();
    return r;
}

// Unordered append: every thread of a 256-thread CTA asks for `cnt` slots of a global buffer; ONE
// atomicAdd per CTA reserves the whole range (same-address returning atomics serialise at the L2
// slice, so one per warp would cost more than the scan).  Returns the thread's first slot.
// Two barriers per call: the warp totals go to the half of s_warp that `parity` selects, and a caller that calls it in a
// loop flips `parity` every call, so the next call's writes never meet this call's reads and no third barrier is needed.
__device__ __forceinline__ uint32_t block_reserve_256(uint32_t cnt, uint32_t* counter, uint32_t* s_warp /*17 words*/, int parity) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += y;
    }
    uint32_t* part = s_warp + 8 * parity;
    if (lane == 31) part[warp] = incl;
    __syncthreads();
    uint32_t before = 0, total = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const uint32_t t = part[i];
        before += i < warp ? t : 0u;
        total += t;
    }
    if (threadIdx.x == 0) s_warp[16] = total ? atomicAdd(counter, total) : 0u;
    __syncthreads();
    return s_warp[16] + before + incl - cnt;
}

static constexpr int SEL_THREADS = 256;
static constexpr int SEL_ITEMS = 8;
static constexpr int SEL_TILE = SEL_THREADS * SEL_ITEMS;

struct TileSync {
    uint32_t* ticket;        // 1 word, zero at launch
    uint64_t* status;        // >= n_tiles words, never cleared (generation-tagged)
    const uint32_t* epoch;   // device counter, bumped once per csv_cluster call (so that a captured CUDA graph of the
                             // call can be replayed: the generation is not a frozen kernel argument)
    uint32_t ordinal;        // unique per look-back launch inside one call (< LB_ORDINALS)
};
static constexpr uint32_t LB_ORDINALS = 1024;
// csv_cluster starts its device epoch over before it reaches LB_EPOCH_LIMIT, so that every generation fits 31 bits
static constexpr uint32_t LB_EPOCH_LIMIT = 1u << 21;
static_assert((uint64_t)LB_EPOCH_LIMIT * LB_ORDINALS <= LB_GEN_LIMIT, "look-back generations must fit 31 bits");
// first node of every csv_cluster call: fresh look-back generation, zeroed ticket words and counters (one launch
// instead of a kernel and two memsets)
__global__ void __launch_bounds__(256) k_begin(uint32_t* epoch, uint32_t* tickets, int n_tickets, uint32_t* counters, int n_counters,
                                               unsigned long long* cursor) {
    if (threadIdx.x == 0) { *epoch += 1u; *cursor = 0ull; }
    for (int i = threadIdx.x; i < n_tickets; i += 256) tickets[i] = 0u;
    for (int i = threadIdx.x; i < n_counters; i += 256) counters[i] = 0u;
}
__device__ __forceinline__ uint32_t ts_gen(const TileSync& ts) { return (*ts.epoch) * LB_ORDINALS + ts.ordinal; }

// Ordered select: out[k] = i for the k-th i in [0, n) with pred(i); *out_count = number selected.
// Overflowing out_cap sets `overflow_bit` in *status_word (and keeps counting).
template <class Pred>
__global__ void __launch_bounds__(SEL_THREADS) k_select(Pred pred, int64_t n_host, const uint32_t* n_dev, uint32_t* out,
                                                        uint32_t out_cap, uint32_t* out_count, TileSync ts,
                                                        uint32_t* status_word, uint32_t overflow_bit) {
    __shared__ uint32_t s_warp[9];
    __shared__ uint32_t s_tile, s_excl;
    const int64_t n = n_dev ? (int64_t)*n_dev : n_host;
    const uint32_t gen = ts_gen(ts);
    while (true) {
        if (threadIdx.x == 0) s_tile = atomicAdd(ts.ticket, 1u);
        __syncthreads();
        const uint32_t tile = s_tile;
        const int64_t base = (int64_t)tile * SEL_TILE;
        if (base >= n) break;
        const int64_t i0 = base + (int64_t)threadIdx.x * SEL_ITEMS;
        uint32_t flags = 0, cnt = 0;
#pragma unroll
        for (int j = 0; j < SEL_ITEMS; j++) {
            const int64_t i = i0 + j;
            if (i < n && pred(i)) { flags |= 1u << j; cnt++; }
        }
        uint32_t total;
        const uint32_t local = block_excl_scan<256>(cnt, s_warp, &total);
        if (threadIdx.x < 32) {
            const uint32_t ex = lookback_exclusive_warp(ts.status, gen, (int)tile, total);
            if (threadIdx.x == 0) {
                s_excl = ex;
                if (base + SEL_TILE >= n) *out_count = ex + total;
            }
        }
        __syncthreads();
        uint32_t o = s_excl + local;
#pragma unroll
        for (int j = 0; j < SEL_ITEMS; j++) {
            if (flags >> j & 1u) {
                if (o < out_cap) out[o] = (uint32_t)(i0 + j);
                else atomicOr(status_word, overflow_bit);
                o++;
            }
        }
        __syncthreads();
    }
}

// In-place exclusive scan of arr[0..n) (+ *carry_in when given); *total_out (nullable) receives carry + sum.
// ITEMS consecutive elements per thread: a tile is 256 * ITEMS elements, so large arrays take few tiles and the
// look-back chain (whose start-up costs one L2 round trip per 32 concurrently running tiles) stays short.
template <int ITEMS>
__global__ void __launch_bounds__(SEL_THREADS) k_scan_excl(uint32_t* arr, int64_t n_host, const uint32_t* n_dev, const uint32_t* carry_in,
                                                           uint32_t* total_out, TileSync ts) {
    pdl_launch_dependents(); pdl_wait();   // programmatic dependent launch: resident early, starts when the previous kernel has finished
    constexpr int TILE = SEL_THREADS * ITEMS;
    __shared__ uint32_t s_warp[9];
    __shared__ uint32_t s_tile, s_excl;
    int64_t n = n_dev ? (int64_t)*n_dev : n_host;
    if (n > n_host) n = n_host;
    const uint32_t carry = carry_in ? *carry_in : 0u;
    const uint32_t gen = ts_gen(ts);
    if (n <= 0) {
        if (total_out && blockIdx.x == 0 && threadIdx.x == 0) *total_out = carry;
        return;
    }
    while (true) {
        if (threadIdx.x == 0) s_tile = atomicAdd(ts.ticket, 1u);
        __syncthreads();
        const uint32_t tile = s_tile;
        const int64_t base = (int64_t)tile * TILE;
        if (base >= n) break;
        const int64_t i0 = base + (int64_t)threadIdx.x * ITEMS;
        uint32_t v[ITEMS], cnt = 0;
        const bool vec = ITEMS == 4 && (((uintptr_t)arr) & 15) == 0 && i0 + ITEMS <= n;   // one coalesced 128-bit access per thread
        if (vec) {
            const uint4 x = *reinterpret_cast<const uint4*>(arr + i0);
            v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
            cnt = x.x + x.y + x.z + x.w;
        } else {
#pragma unroll
            for (int j = 0; j < ITEMS; j++) {
                v[j] = (i0 + j < n) ? arr[i0 + j] : 0u;
                cnt += v[j];
            }
        }
        uint32_t total;
        const uint32_t local = block_excl_scan<256>(cnt, s_warp, &total);
        if (threadIdx.x < 32) {
            const uint32_t ex = lookback_exclusive_warp(ts.status, gen, (int)tile, total);
            if (threadIdx.x == 0) {
                s_excl = ex;
                if (total_out && base + TILE >= n) *total_out = carry + ex + total;
            }
        }
        __syncthreads();
        uint32_t run = carry + s_excl + local;
        if (vec) *reinterpret_cast<uint4*>(arr + i0) = make_uint4(run, run + v[0], run + v[0] + v[1], run + v[0] + v[1] + v[2]);
        else {
#pragma unroll
            for (int j = 0; j < ITEMS; j++) {
                if (i0 + j < n) arr[i0 + j] = run;
                run += v[j];
            }
        }
        __syncthreads();
    }
}

}  // namespace csv
