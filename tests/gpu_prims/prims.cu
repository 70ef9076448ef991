// prims.cu -- test-only launchers of the library's device-wide primitives (cutesv_b200/csrc/devprims.cuh and radix.cuh,
// included as they are), so that tests/test_gpu_lookback.py and tests/test_gpu_radix.py can run them on their own against
// numpy.  Every launcher takes device pointers and a stream, launches once and returns the launch's cudaError_t; the caller
// zeroes the ticket word before each launch.
#include "../../cutesv_b200/csrc/radix.cuh"

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

// ---- radix sort (radix.cuh): key_bytes 4 = uint32_t keys, 8 = uint64_t keys ----

extern "C" int prims_rs_hist(int key_bytes, const void* keys, int64_t n_host, const uint32_t* n_dev, int passes, uint32_t* hist, int grid,
                             void* stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    if (key_bytes == 4) k_rs_hist<uint32_t><<<grid, RS_THREADS, 0, s>>>((const uint32_t*)keys, n_host, n_dev, passes, hist);
    else if (key_bytes == 8) k_rs_hist<uint64_t><<<grid, RS_THREADS, 0, s>>>((const uint64_t*)keys, n_host, n_dev, passes, hist);
    else return (int)cudaErrorInvalidValue;
    return (int)cudaGetLastError();
}

extern "C" int prims_rs_hist_scan(uint32_t* hist, int passes, void* stream) {
    k_rs_hist_scan<<<1, 256, 0, (cudaStream_t)stream>>>(hist, passes);
    return (int)cudaGetLastError();
}

// One pass at bit `shift`; iota != 0: the payload of element i is i (vals_in is not read)
extern "C" int prims_rs_onesweep(int key_bytes, int iota, const void* keys_in, const uint32_t* vals_in, void* keys_out, uint32_t* vals_out,
                                 int64_t n_host, const uint32_t* n_dev, int shift, const uint32_t* gbase, uint32_t* ticket, uint64_t* status,
                                 const uint32_t* epoch, uint32_t ordinal, int grid, void* stream) {
    const TileSync ts = make_ts(ticket, status, epoch, ordinal);
    const cudaStream_t s = (cudaStream_t)stream;
    if (key_bytes == 4 && iota)
        k_rs_onesweep<uint32_t, true><<<grid, RS_THREADS, 0, s>>>((const uint32_t*)keys_in, vals_in, (uint32_t*)keys_out, vals_out, n_host, n_dev,
                                                                  shift, gbase, ts);
    else if (key_bytes == 4)
        k_rs_onesweep<uint32_t, false><<<grid, RS_THREADS, 0, s>>>((const uint32_t*)keys_in, vals_in, (uint32_t*)keys_out, vals_out, n_host, n_dev,
                                                                   shift, gbase, ts);
    else if (key_bytes == 8 && iota)
        k_rs_onesweep<uint64_t, true><<<grid, RS_THREADS, 0, s>>>((const uint64_t*)keys_in, vals_in, (uint64_t*)keys_out, vals_out, n_host, n_dev,
                                                                  shift, gbase, ts);
    else if (key_bytes == 8)
        k_rs_onesweep<uint64_t, false><<<grid, RS_THREADS, 0, s>>>((const uint64_t*)keys_in, vals_in, (uint64_t*)keys_out, vals_out, n_host, n_dev,
                                                                   shift, gbase, ts);
    else return (int)cudaErrorInvalidValue;
    return (int)cudaGetLastError();
}

// Keys per onesweep tile
extern "C" int prims_rs_tile(int key_bytes) {
    return key_bytes == 4 ? RS_THREADS * RsTraits<uint32_t>::ITEMS : key_bytes == 8 ? RS_THREADS * RsTraits<uint64_t>::ITEMS : 0;
}

// Onesweep CTAs resident per SM (the smaller of the iota and the plain instantiation); negative: the cudaError_t
extern "C" int prims_rs_resident(int key_bytes) {
    int a = 0, b = 0;
    cudaError_t e;
    if (key_bytes == 4) {
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, k_rs_onesweep<uint32_t, true>, RS_THREADS, 0);
        if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_rs_onesweep<uint32_t, false>, RS_THREADS, 0);
    } else if (key_bytes == 8) {
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, k_rs_onesweep<uint64_t, true>, RS_THREADS, 0);
        if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_rs_onesweep<uint64_t, false>, RS_THREADS, 0);
    } else {
        return -(int)cudaErrorInvalidValue;
    }
    return e == cudaSuccess ? (a < b ? a : b) : -(int)e;
}

// ---- the large one-pass u32 sort of tests/test_gpu_radix.py, built and checked on the device ----
// Tile t (T = 4096 keys, n_valid(t) of them real) holds one digit-0 key at z(t), one digit-255 key at f(t) != z(t) and
// digit-1 keys everywhere else; bits 8..31 of every key are a hash of its row, so a key that lands with the wrong payload
// shows.  The stable sort by the low byte then has a closed form: digit-0 rows by tile, digit-1 rows in row order, digit-255
// rows by tile.
namespace {
constexpr int64_t LG_T = RS_THREADS * RsTraits<uint32_t>::ITEMS;

__device__ __forceinline__ uint32_t lg_hash(uint64_t x) {
    x ^= x >> 31; x *= 0x9E3779B97F4A7C15ull; x ^= x >> 29;
    return (uint32_t)(x >> 32);
}
__device__ __forceinline__ int64_t lg_valid(int64_t n, int64_t t) { return (n - t * LG_T) < LG_T ? (n - t * LG_T) : LG_T; }
__device__ __forceinline__ int64_t lg_zero(int64_t n, int64_t t) { return lg_hash(2 * t) % lg_valid(n, t); }
__device__ __forceinline__ int64_t lg_ff(int64_t n, int64_t t) {   // needs n_valid(t) >= 2
    const int64_t v = lg_valid(n, t);
    return (lg_zero(n, t) + 1 + lg_hash(2 * t + 1) % (v - 1)) % v;
}
__device__ __forceinline__ uint32_t lg_key(uint32_t digit, int64_t row) { return (lg_hash((uint64_t)row + 12345) & 0xFFFFFF00u) | digit; }

__global__ void k_lg_keys(uint32_t* keys, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = i / LG_T, p = i - t * LG_T;
        keys[i] = lg_key(p == lg_zero(n, t) ? 0u : p == lg_ff(n, t) ? 255u : 1u, i);
    }
}

// counts the positions of [lo, lo + cnt) whose key or payload differs from the closed form; *first_bad = the lowest one
__global__ void k_lg_check(const uint32_t* keys, const uint32_t* vals, int64_t n, int64_t lo, int64_t cnt, unsigned long long* n_bad,
                           unsigned long long* first_bad) {
    const int64_t tiles = (n + LG_T - 1) / LG_T;
    for (int64_t j = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < lo + cnt; j += (int64_t)gridDim.x * blockDim.x) {
        int64_t row;
        uint32_t digit;
        if (j < tiles) {
            row = j * LG_T + lg_zero(n, j);
            digit = 0;
        } else if (j >= n - tiles) {
            const int64_t t = j - (n - tiles);
            row = t * LG_T + lg_ff(n, t);
            digit = 255;
        } else {   // the r-th digit-1 row of tile t: the r-th position that is neither z(t) nor f(t)
            const int64_t k = j - tiles, t = k / (LG_T - 2);
            int64_t p = k - t * (LG_T - 2);
            const int64_t z = lg_zero(n, t), f = lg_ff(n, t);
            const int64_t a = z < f ? z : f, b = z < f ? f : z;
            if (p >= a) p++;
            if (p >= b) p++;
            row = t * LG_T + p;
            digit = 1;
        }
        if (keys[j] != lg_key(digit, row) || vals[j] != (uint32_t)row) {
            atomicAdd(n_bad, 1ull);
            atomicMin(first_bad, (unsigned long long)j);
        }
    }
}
}  // namespace

extern "C" int prims_rs_large_keys(uint32_t* keys, int64_t n, void* stream) {
    k_lg_keys<<<132 * 16, 256, 0, (cudaStream_t)stream>>>(keys, n);
    return (int)cudaGetLastError();
}

extern "C" int prims_rs_large_check(const uint32_t* keys, const uint32_t* vals, int64_t n, int64_t lo, int64_t cnt, unsigned long long* n_bad,
                                    unsigned long long* first_bad, void* stream) {
    k_lg_check<<<132 * 16, 256, 0, (cudaStream_t)stream>>>(keys, vals, n, lo, cnt, n_bad, first_bad);
    return (int)cudaGetLastError();
}
