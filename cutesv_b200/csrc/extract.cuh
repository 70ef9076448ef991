// extract.cuh -- kernel (a): one warp per alignment record walks the packed CIGAR with a warp
// prefix scan over reference / query offsets (parse_read, cuteSV:606-655), lane 0 runs the
// streaming intra-read merge (generate_combine_sigs, cuteSV:515-575) and the split-read rule
// engine (cuteSV:50-513).  HBM-bound: 4 B per CIGAR op read once, coalesced.
#pragma once
#include "extract_core.h"
#include "names_core.h"

namespace csv {

struct ReadView {
    const int32_t *chrom, *ref_start, *ref_end, *flag, *mapq, *query_len, *read_id;
    const int64_t *cigar_off, *sa_off;
    int64_t n;
};

static constexpr int EX_THREADS = 256;
static constexpr int EX_WARPS = EX_THREADS / 32;
static constexpr int EX_ITEMS = 8;                       // consecutive CIGAR ops per lane and iteration
static constexpr int EX_TILE = 32 * EX_ITEMS;            // ops per warp iteration
#ifndef EX_CHUNK_TILES
#define EX_CHUNK_TILES 2
#endif
static constexpr int EX_CHUNK = EX_TILE * EX_CHUNK_TILES; // ops per bulk copy: thousands of warps stream their own record each, so
                                                          // a request must be large enough (4 KB) to stay inside a DRAM page or two
static constexpr int EX_RING = 2;                         // chunks in flight per warp
#ifndef EX_MIN_CTAS
#define EX_MIN_CTAS 3
#endif
static constexpr int EX_SLOT_BYTES = (EX_CHUNK + 4) * 4;  // + 4 ops: chunks start 16 B aligned, up to 3 ops before the read's first op
static constexpr int EX_SMEM_BYTES = EX_WARPS * EX_RING * EX_SLOT_BYTES;
static_assert(EX_SLOT_BYTES % 16 == 0, "bulk copies move multiples of 16 B");

// ---- 1-D TMA (cp.async.bulk) + mbarrier (devprims.cuh): the CIGAR stream of a record is staged tile by tile into a per-warp
// shared-memory ring, EX_RING tiles ahead of the scan, by ONE lane; completion is signalled through the slot's mbarrier.

// the rare per-signature work stays out of the scan loop's instruction stream (instruction cache)
__device__ __noinline__ void ex_push(const ExtractOut& O, const ReadCtx& RC, const ExtractParams& P, MergeState& S, InsPiece* open_pieces, uint32_t cg,
                                     int32_t pos, int64_t shift) {
    const int32_t len = (int32_t)(cg >> 4);
    if ((int)(cg & 15) == OP_D) push_del(O, RC, P, S, pos, len);
    else push_ins(O, RC, P, S, open_pieces, pos, len, shift - len, shift);
}
__device__ __noinline__ void ex_flush(const ExtractOut& O, const ReadCtx& RC, MergeState& S, const InsPiece* open_pieces) {
    flush_ins(O, RC, S, open_pieces);
    flush_del(O, RC, S);
}
__device__ __noinline__ void ex_split(const ExtractOut& O, const ReadCtx& RC0, const ExtractParams& P, int sig, int32_t clip_l, int32_t clip_r, int32_t qlen,
                                      int32_t ref_start, int32_t ref_end, int32_t chrom, bool mq_ok, const SaView& sa, int64_t s_lo, int64_t s_hi) {
    SplitCtx C;
    C.O = &O; C.R = RC0; C.P = P;
    C.R.base_rc = sig == 2 ? 1 : 0;
    Seg prim;
    if (sig == 1) { prim.rs = clip_l; prim.re = qlen - clip_r; }
    else { prim.rs = clip_r; prim.re = qlen - clip_l; }
    prim.fs = ref_start; prim.fe = ref_end; prim.chr = chrom; prim.strand = sig == 1 ? 0 : 1;
    organize_split_signal(C, mq_ok, prim, sa, s_lo, s_hi);
}

__global__ void __launch_bounds__(EX_THREADS, EX_MIN_CTAS) k_extract(ReadView R, const uint32_t* __restrict__ cigar, SaView sa, ExtractParams P,
                                                        ExtractOut O, int32_t rec_base, uint32_t* ticket) {
    extern __shared__ __align__(16) uint32_t s_ring_raw[];
    uint32_t (*s_ring)[EX_RING][EX_SLOT_BYTES / 4] = reinterpret_cast<uint32_t (*)[EX_RING][EX_SLOT_BYTES / 4]>(s_ring_raw);
    __shared__ __align__(8) uint64_t s_bar[EX_WARPS][EX_RING];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0)
        for (int k = 0; k < EX_RING; k++) mbar_init(&s_bar[warp][k], 1);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // make the barrier inits visible to the async (TMA) proxy
    __syncwarp();
    uint32_t phase = 0;   // bit k: parity the next wait on slot k expects
    // records are handed out one at a time (a persistent grid of resident warps + a ticket): CIGAR lengths vary by orders of
    // magnitude, a static stride leaves a long tail
    for (;;) {
        uint32_t tk = 0;
        if (lane == 0) tk = atomicAdd(ticket, 1u);
        const int64_t rec = (int64_t)__shfl_sync(0xffffffffu, tk, 0);
        if (rec >= R.n) break;
        const int32_t flag = R.flag[rec];
        if (flag == 256 || flag == 272) continue;  // single_pipe, cuteSV:711
        const int32_t mapq = R.mapq[rec], qlen = R.query_len[rec], chrom = R.chrom[rec], rid = R.read_id[rec];
        const int32_t ref_start = R.ref_start[rec], ref_end = R.ref_end[rec];
        const bool mq_ok = mapq >= P.min_mapq;
        if (mq_ok && lane == 0) {  // reads_info_list row, cuteSV:729-733
            const uint32_t k = atomicAdd(O.n_rows, 1u);
            if (k < O.cap_rows) {
                O.rr_chrom[k] = chrom; O.rr_start[k] = ref_start; O.rr_end[k] = ref_end; O.rr_id[k] = rid;
                O.rr_prim[k] = (flag == 0 || flag == 16) ? 1 : 0;
                if (O.rr_rec) O.rr_rec[k] = rec_base + (int32_t)rec;
            } else atomicOr(O.status, ST_LIST_OVERFLOW);
        }
        if (qlen < P.min_read_len) continue;  // parse_read, cuteSV:607
        ReadCtx RC;
        RC.rec = rec_base + (int32_t)rec; RC.chrom = chrom; RC.rid = rid; RC.qlen = qlen; RC.base_rc = 0;
        const int64_t c_lo = R.cigar_off[rec], c_hi = R.cigar_off[rec + 1];
        int32_t clip_l = 0, clip_r = 0;
        if (mq_ok && c_hi > c_lo) {
            const uint32_t first = cigar[c_lo], last = cigar[c_hi - 1];
            const int fop = first & 15, lop = last & 15;
            const int32_t hard_l = fop == OP_H ? (int32_t)(first >> 4) : 0;
            if (fop == OP_S || fop == OP_H) clip_l = (int32_t)(first >> 4);  // cuteSV:623-626,651-654
            if (lop == OP_S || lop == OP_H) clip_r = (int32_t)(last >> 4);
            MergeState S;
            S.reset();
            InsPiece open_pieces[MAX_OPEN_PIECES];
            int32_t ref = ref_start;
            int64_t q = -(int64_t)hard_l;
            int32_t acc_r = 0, acc_q = 0;   // this lane's advances over the tiles since the last qualifying op
            // EX_TILE ops per warp iteration: every lane owns EX_ITEMS consecutive ops, so one warp scan (5 shuffle steps per
            // offset) is amortised over 256 ops.  The stream is fetched by 1-D bulk copies of EX_CHUNK ops (4 KB), EX_RING
            // chunks ahead: ~24 resident warps per SM keep ~200 KB per SM in flight.  Chunk k holds ops
            // [a0 + k * EX_CHUNK, + EX_CHUNK + 4), a0 = c_lo rounded down to 16 B.
            const int64_t a0 = c_lo & ~(int64_t)3;
            const int d0 = (int)(c_lo - a0);
            const int64_t n_tiles = (c_hi - c_lo + EX_TILE - 1) / EX_TILE;
            const int64_t n_chunks = (n_tiles + EX_CHUNK_TILES - 1) / EX_CHUNK_TILES;
            if (lane == 0)
                for (int k = 0; k < EX_RING && k < n_chunks; k++)
                    bulk_load(&s_ring[warp][k][0], cigar + a0 + (int64_t)k * EX_CHUNK, EX_SLOT_BYTES, &s_bar[warp][k]);
            for (int64_t t = 0; t < n_tiles; t++) {
                const int64_t chunk = t / EX_CHUNK_TILES;
                const int sub = (int)(t % EX_CHUNK_TILES);
                const int slot = (int)(chunk % EX_RING);
                if (sub == 0) {
                    mbar_wait(&s_bar[warp][slot], (phase >> slot) & 1u);
                    phase ^= 1u << slot;
                }
                // ops left for this lane in the record (the tail of the last tile is padding)
                const int64_t left64 = c_hi - (c_lo + t * EX_TILE) - lane * EX_ITEMS;
                const int left = left64 > EX_ITEMS ? EX_ITEMS : (int)left64;
                // the lane's 8 ops start d0 (0..3, uniform for the record) words past a 16 B boundary: three aligned 128-bit loads
                // (2-way bank conflicts instead of the 8-way ones of eight strided 32-bit loads) + a uniform select
                uint32_t cur[EX_ITEMS];
                {
                    const uint4* src = reinterpret_cast<const uint4*>(&s_ring[warp][slot][sub * EX_TILE + lane * EX_ITEMS]);
                    const uint4 w0 = src[0], w1 = src[1], w2 = src[2];
                    const uint32_t w[12] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w, w2.x, w2.y, w2.z, w2.w};
#pragma unroll
                    for (int j = 0; j < EX_ITEMS; j++) {
                        const uint32_t v = d0 == 0 ? w[j] : d0 == 1 ? w[j + 1] : d0 == 2 ? w[j + 2] : w[j + 3];
                        cur[j] = j < left ? v : (uint32_t)OP_P;
                    }
                }
                if (sub == EX_CHUNK_TILES - 1 || t == n_tiles - 1) {
                    __syncwarp();   // every lane has read the slot: it can be refilled
                    if (lane == 0 && chunk + EX_RING < n_chunks)
                        bulk_load(&s_ring[warp][slot][0], cigar + a0 + (chunk + EX_RING) * EX_CHUNK, EX_SLOT_BYTES, &s_bar[warp][slot]);
                }
                int32_t radv[EX_ITEMS], qadv[EX_ITEMS];
                int32_t r_tot = 0, q_tot = 0;
                uint32_t qmask = 0;
                // op classes as bit masks over the 4-bit op code: M D N = X advance the reference (cuteSV:633-643), everything
                // but D advances the query cursor (cuteSV:631-632), I and D can be signatures
                constexpr uint32_t REF_OPS = (1u << OP_M) | (1u << OP_D) | (1u << OP_N) | (1u << OP_EQ) | (1u << OP_X);
                constexpr uint32_t SIG_OPS = (1u << OP_I) | (1u << OP_D);
#pragma unroll
                for (int j = 0; j < EX_ITEMS; j++) {
                    const uint32_t op = cur[j] & 15u;
                    const int32_t len = (int32_t)(cur[j] >> 4);
                    radv[j] = len & -(int32_t)((REF_OPS >> op) & 1u);
                    qadv[j] = op != (uint32_t)OP_D ? len : 0;
                    r_tot += radv[j];
                    q_tot += qadv[j];
                    if (len >= P.min_siglength && ((SIG_OPS >> op) & 1u)) qmask |= 1u << j;   // (padding ops are OP_P)
                }
                // Offsets are only needed where a qualifying op sits (~2 per record): tiles without one just add to the lane's
                // private totals (no shuffles); a tile with one first folds the private totals of all lanes into the record's
                // running offsets, then scans.
                uint32_t lanes = __ballot_sync(0xffffffffu, qmask != 0);
                if (lanes) {
                    int32_t ar = acc_r, aq = acc_q;
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) { ar += __shfl_xor_sync(0xffffffffu, ar, o); aq += __shfl_xor_sync(0xffffffffu, aq, o); }
                    ref += ar; q += aq;
                    acc_r = 0; acc_q = 0;
                    int32_t ir = r_tot, iq = q_tot;
#pragma unroll
                    for (int d = 1; d < 32; d <<= 1) {
                        const int32_t yr = __shfl_up_sync(0xffffffffu, ir, d);
                        const int32_t yq = __shfl_up_sync(0xffffffffu, iq, d);
                        if (lane >= d) { ir += yr; iq += yq; }
                    }
                    int32_t sig_start[EX_ITEMS];
                    int64_t shift_after[EX_ITEMS];
                    int32_t run_r = ref + ir - r_tot;
                    int64_t run_q = q + iq - q_tot;
#pragma unroll
                    for (int j = 0; j < EX_ITEMS; j++) {
                        sig_start[j] = run_r;
                        run_r += radv[j];
                        run_q += qadv[j];
                        shift_after[j] = run_q;
                    }
                    while (lanes) {   // serial hand-over to lane 0, in read order
                        const int L = __ffs(lanes) - 1;
                        lanes &= lanes - 1;
                        const uint32_t m8 = __shfl_sync(0xffffffffu, qmask, L);
#pragma unroll
                        for (int j = 0; j < EX_ITEMS; j++) {
                            if (!(m8 >> j & 1u)) continue;
                            const uint32_t v_cg = __shfl_sync(0xffffffffu, cur[j], L);
                            const int32_t v_pos = __shfl_sync(0xffffffffu, sig_start[j], L);
                            const int64_t v_shift = __shfl_sync(0xffffffffu, shift_after[j], L);
                            if (lane == 0) ex_push(O, RC, P, S, open_pieces, v_cg, v_pos, v_shift);
                        }
                    }
                    ref += __shfl_sync(0xffffffffu, ir, 31);
                    q += __shfl_sync(0xffffffffu, iq, 31);
                } else {
                    acc_r += r_tot; acc_q += q_tot;
                }
            }
            if (lane == 0) ex_flush(O, RC, S, open_pieces);
        }
        const int sig = detect_flag(flag);
        const int64_t s_lo = R.sa_off[rec], s_hi = R.sa_off[rec + 1];
        if ((sig == 1 || sig == 2) && s_hi > s_lo && lane == 0)   // cuteSV:660-680
            ex_split(O, RC, P, sig, clip_l, clip_r, qlen, ref_start, ref_end, chrom, mq_ok, sa, s_lo, s_hi);
        __syncwarp();
    }
}

// ---- packets from device memory: offsets are checked on the device before any kernel reads through them ----
enum { PK_BAD_CIGAR = 1u, PK_BAD_SA = 2u, PK_BAD_SEQ = 4u, PK_BAD_QLEN = 8u, PK_BAD_NAME = 16u, PK_LONG_NAME = 32u };
struct PacketCheck {
    const int64_t* off[4];   // cigar_off, sa_off, seq_off, name_off (n + 1 entries each; seq_off and name_off may be null)
    int64_t bound[4];        // n_cigar, sa->n, seq->n_bytes, names->n_bytes
    const int32_t* query_len;
    int64_t n;
};
// *bad |= PK_BAD_* of every column whose offsets do not start at >= 0, never decrease and end at <= its bound, or that has a
// negative query_len; PK_LONG_NAME for a name longer than NAME_MAX_BYTES
__global__ void __launch_bounds__(256) k_check_packet(PacketCheck C, uint32_t* bad) {
    uint32_t b = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= C.n; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int64_t* o = C.off[k];
            if (!o) continue;
            const int64_t v = o[i];
            const uint32_t bit = k < 3 ? 1u << k : PK_BAD_NAME;
            if ((i == 0 && v < 0) || (i == C.n && v > C.bound[k]) || (i < C.n && o[i + 1] < v)) b |= bit;
            if (k == 3 && i < C.n && o[i + 1] - v > NAME_MAX_BYTES) b |= PK_LONG_NAME;
        }
        if (i < C.n && C.query_len[i] < 0) b |= PK_BAD_QLEN;
    }
    b = __reduce_or_sync(0xffffffffu, b);
    if (b && (threadIdx.x & 31) == 0) atomicOr(bad, b);
}

// ---- INS sequences of one packet's new INS rows [first_row, first_row + m), built from the packed bases ----
struct InsSeqJob {
    const int32_t* piece_off; const int32_t* piece_cnt; const InsPiece* pieces;
    int64_t first_row; int64_t m;
    int32_t rec_base;                     // record index of the packet's first record (pieces hold global record indices)
    const int64_t* seq_off; const uint8_t* seq4; const int32_t* query_len;
    const uint32_t* cigar; const int64_t* cigar_off; const int32_t* ref_start;   // marker pieces: the record's CIGAR walk
    int32_t min_siglength, merge_ins_threshold;
};
__device__ __forceinline__ SeqRec seq_rec(const InsSeqJob& J, int64_t rec) {
    SeqRec s;
    s.qlen = J.query_len[rec];
    s.have = J.seq_off[rec + 1] - J.seq_off[rec] >= ((int64_t)s.qlen + 1) / 2;
    s.seq4 = J.seq4 + J.seq_off[rec];
    return s;
}
// arguments by value: a reference to the kernel parameter would give every thread of the common path a stack frame
__device__ __noinline__ int64_t ins_marker(SeqRec s, const uint32_t* cigar, int64_t c0, int64_t c1, int32_t ref_start, int32_t pos,
                                           int32_t min_siglength, int32_t merge_ins_threshold, uint8_t* out) {
    return ins_marker_bytes(s, cigar + c0, c1 - c0, ref_start, pos, min_siglength, merge_ins_threshold, out);
}
__device__ __forceinline__ int64_t ins_marker(const InsSeqJob& J, const SeqRec& s, int64_t rec, int32_t pos, uint8_t* out) {
    return ins_marker(s, J.cigar, J.cigar_off[rec], J.cigar_off[rec + 1], J.ref_start[rec], pos, J.min_siglength, J.merge_ins_threshold, out);
}
// len[k] = bytes of row first_row + k; *total64 += all of them (a 64-bit sum beside the 32-bit scan)
__global__ void __launch_bounds__(256) k_ins_len(InsSeqJob J, uint32_t* len, unsigned long long* total64, uint32_t* status) {
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < J.m; base += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k = base + threadIdx.x;
        int64_t w = 0;
        if (k < J.m) {
            const int64_t row = J.first_row + k;
            const int32_t po = J.piece_off[row], pc = J.piece_cnt[row];
            for (int32_t p = po; p < po + pc; p++) {
                const InsPiece ip = J.pieces[p];
                const int64_t rec = (int64_t)ip.rec - J.rec_base;
                const SeqRec s = seq_rec(J, rec);
                if (ip.rc == 2) {   // the length-only walk is inlined: a call here would make the loop spill across it
                    const int64_t c0 = J.cigar_off[rec];
                    const int64_t v = ins_marker_bytes(s, J.cigar + c0, J.cigar_off[rec + 1] - c0, J.ref_start[rec], ip.start, J.min_siglength,
                                                       J.merge_ins_threshold, nullptr);
                    if (v < 0) atomicOr(status, ST_INTERNAL);
                    else w += v;
                } else w += ins_piece_bytes(s, ip.start, ip.stop, ip.rc, nullptr, 0, 1);
            }
            len[k] = (uint32_t)w;
        }
        unsigned long long t = (unsigned long long)w;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if ((threadIdx.x & 31) == 0 && t) atomicAdd(total64, t);
    }
}
// one warp per row: start[first_row + k] = arena_base + excl[k], the row's bytes at that offset
__global__ void __launch_bounds__(256) k_ins_fill(InsSeqJob J, const uint32_t* excl, const uint32_t* len, int64_t arena_base, uint8_t* bytes,
                                                  int64_t* start, int32_t* row_len) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t k = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < J.m; k += warps) {
        const int64_t row = J.first_row + k, o = arena_base + excl[k];
        if (lane == 0) { start[row] = o; row_len[row] = (int32_t)len[k]; }
        uint8_t* out = bytes + o;
        const int32_t po = J.piece_off[row], pc = J.piece_cnt[row];
        for (int32_t p = po; p < po + pc; p++) {
            const InsPiece ip = J.pieces[p];
            const int64_t rec = (int64_t)ip.rec - J.rec_base;
            const SeqRec s = seq_rec(J, rec);
            int64_t w;
            if (ip.rc == 2) {   // rare: chains of more than MAX_OPEN_PIECES merged insertions, walked by one lane
                int64_t v = 0;
                if (lane == 0) v = ins_marker(J, s, rec, ip.start, out);
                w = __shfl_sync(0xffffffffu, v, 0);
                if (w < 0) w = 0;
            } else w = ins_piece_bytes(s, ip.start, ip.stop, ip.rc, out, lane, 32);
            out += w;
        }
    }
}
// csv_fetch_ins_seqs: one warp per requested row, out + off[i] <- the row's bytes
__global__ void __launch_bounds__(256) k_ins_gather(const int64_t* rows, int64_t n, const int64_t* off, const uint8_t* bytes, const int64_t* start,
                                                    const int32_t* row_len, uint8_t* out) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < n; i += warps) {
        const int64_t r = rows[i];
        const uint8_t* src = bytes + start[r];
        uint8_t* dst = out + off[i];
        for (int32_t j = lane; j < row_len[r]; j += 32) dst[j] = src[j];
    }
}
__global__ void k_ins_sel_len(const int64_t* rows, int64_t n, const int32_t* row_len, int32_t* len) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) len[i] = row_len[rows[i]];
}

}  // namespace csv
