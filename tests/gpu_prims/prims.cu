// prims.cu -- test-only launchers of the library's device-wide primitives (cutesv_b200/csrc/devprims.cuh, included as it
// is), so that tests/test_gpu_lookback.py can run them on their own against numpy.  Every launcher takes device pointers
// and a stream, launches once and returns the launch's cudaError_t; the caller zeroes the ticket word before each launch.
#include "../../cutesv_b200/csrc/devprims.cuh"

using namespace csv;

namespace {

struct FlagPred {
    const uint8_t* flags;
    __device__ bool operator()(int64_t i) const { return flags[i] != 0; }
};

// Tile t (taken by ticket) publishes vals[t], then waits for its exclusive prefix and writes it to excl[t]: the split form
// k_part_filter uses.  One warp per CTA; a CTA takes tickets until they run out.
__global__ void __launch_bounds__(32) k_lb_probe(const uint32_t* vals, int n_tiles, uint32_t* excl, TileSync ts) {
    const uint32_t gen = ts_gen(ts);
    const int lane = threadIdx.x & 31;
    while (true) {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd(ts.ticket, 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if ((int)t >= n_tiles) break;
        const uint32_t local = vals[t];
        if (lane == 0) lookback_publish(ts.status, gen, (int)t, local);
        const uint32_t ex = lookback_wait_warp(ts.status, gen, (int)t, local);
        if (lane == 0) excl[t] = ex;
    }
}

TileSync make_ts(uint32_t* ticket, uint64_t* status, const uint32_t* epoch, uint32_t ordinal) {
    TileSync ts;
    ts.ticket = ticket;
    ts.status = status;
    ts.epoch = epoch;
    ts.ordinal = ordinal;
    return ts;
}

}  // namespace

extern "C" int prims_scan_excl(int items, uint32_t* arr, int64_t n_host, const uint32_t* n_dev, const uint32_t* carry_in, uint32_t* total_out,
                               uint32_t* ticket, uint64_t* status, const uint32_t* epoch, uint32_t ordinal, int grid, void* stream) {
    const TileSync ts = make_ts(ticket, status, epoch, ordinal);
    const cudaStream_t s = (cudaStream_t)stream;
    if (items == 4) k_scan_excl<4><<<grid, SEL_THREADS, 0, s>>>(arr, n_host, n_dev, carry_in, total_out, ts);
    else if (items == 8) k_scan_excl<8><<<grid, SEL_THREADS, 0, s>>>(arr, n_host, n_dev, carry_in, total_out, ts);
    else return (int)cudaErrorInvalidValue;
    return (int)cudaGetLastError();
}

extern "C" int prims_select(const uint8_t* flags, int64_t n_host, const uint32_t* n_dev, uint32_t* out, uint32_t out_cap, uint32_t* out_count,
                            uint32_t* status_word, uint32_t overflow_bit, uint32_t* ticket, uint64_t* status, const uint32_t* epoch,
                            uint32_t ordinal, int grid, void* stream) {
    const TileSync ts = make_ts(ticket, status, epoch, ordinal);
    k_select<FlagPred><<<grid, SEL_THREADS, 0, (cudaStream_t)stream>>>(FlagPred{flags}, n_host, n_dev, out, out_cap, out_count, ts, status_word,
                                                                       overflow_bit);
    return (int)cudaGetLastError();
}

extern "C" int prims_lookback_probe(const uint32_t* vals, int n_tiles, uint32_t* excl, uint32_t* ticket, uint64_t* status, const uint32_t* epoch,
                                    uint32_t ordinal, int grid, void* stream) {
    const TileSync ts = make_ts(ticket, status, epoch, ordinal);
    k_lb_probe<<<grid, 32, 0, (cudaStream_t)stream>>>(vals, n_tiles, excl, ts);
    return (int)cudaGetLastError();
}

// A launch's look-back generation is *epoch * LB_ORDINALS + ordinal
extern "C" uint32_t prims_lb_ordinals(void) { return LB_ORDINALS; }
