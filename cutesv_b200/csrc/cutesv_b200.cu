// cutesv_b200.cu -- C-ABI (include/cutesv_b200.h) and host orchestration of the sm_90a (H100) kernels.
//
// One translation unit: nvcc -gencode arch=compute_90a,code=sm_90a -fmad=false -lineinfo.
// There is deliberately no host compute path in this library: without a usable GPU csv_create
// fails (CSV_E_NODEVICE) and every other entry point needs a ctx.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <string>
#include <vector>

#include "../../include/cutesv_b200.h"
#include "core.h"
#include "devprims.cuh"
#include "host_tables.h"
#include "kernels.cuh"
#include "radix.cuh"
#include "extract.cuh"
#include "scan_core.h"
#include "sa_core.h"

using namespace csv;

// ------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
static int set_err(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CU(call)                                                                                               \
    do {                                                                                                       \
        cudaError_t e__ = (call);                                                                              \
        if (e__ != cudaSuccess)                                                                                \
            return set_err(CSV_E_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)

extern "C" const char* csv_last_error(void) { return g_err; }
struct csv_ctx;
static void comm_destroy(csv_ctx* c);
extern "C" int csv_version(void) { return 100; }

// ------------------------------------------------------------------------------------------
// device buffers
// ------------------------------------------------------------------------------------------
// Every (re)allocation bumps this counter: a captured CUDA graph holds raw device pointers, so a graph is only
// replayed while the counter still has the value it had at capture time.
static std::atomic<uint64_t> g_alloc_epoch{1};

// Owns its allocation: freed when the buffer is destroyed (the ctx's buffers by `delete c`, on the ctx's device) or moved over.
struct DBuf {
    void* p = nullptr;
    size_t cap = 0;
    DBuf() = default;
    DBuf(const DBuf&) = delete;
    DBuf& operator=(const DBuf&) = delete;
    DBuf(DBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    DBuf& operator=(DBuf&& o) noexcept { if (this != &o) { release(); std::swap(p, o.p); std::swap(cap, o.cap); } return *this; }
    ~DBuf() { release(); }
    cudaError_t ensure(size_t bytes, bool zero_new = false) {
        if (bytes <= cap) return cudaSuccess;
        g_alloc_epoch.fetch_add(1);
        if (p) { cudaError_t e = cudaFree(p); if (e != cudaSuccess) return e; p = nullptr; cap = 0; }
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) return e;
        cap = want;
        if (zero_new) {   // visible to every (non-blocking) stream before ensure() returns
            e = cudaMemset(p, 0, want);
            if (e != cudaSuccess) return e;
            return cudaDeviceSynchronize();
        }
        return cudaSuccess;
    }
    // capacity for `bytes`, keeping the first keep_bytes of the present contents (append mode: copied on s, which is then
    // synchronised)
    cudaError_t grow(size_t bytes, size_t keep_bytes, cudaStream_t s) {
        if (bytes <= cap) return cudaSuccess;
        if (keep_bytes == 0 || !p) return ensure(bytes);
        DBuf nb;
        cudaError_t e = nb.ensure(bytes + bytes / 2);   // geometric growth: a run appends many packets
        if (e == cudaSuccess) e = cudaMemcpyAsync(nb.p, p, keep_bytes, cudaMemcpyDeviceToDevice, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e == cudaSuccess) *this = std::move(nb);   // frees the old buffer
        return e;
    }
    // D2H of bytes [off, off + bytes), when the caller asked for them (dst not null)
    cudaError_t fetch(void* dst, size_t off, size_t bytes, cudaStream_t s) const {
        return dst && bytes ? cudaMemcpyAsync(dst, (const char*)p + off, bytes, cudaMemcpyDeviceToHost, s) : cudaSuccess;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() const { return (T*)p; }
};

// ------------------------------------------------------------------------------------------
// input tables: the only place that knows their columns; callers size, grow, fill, check and fetch whole tables
// ------------------------------------------------------------------------------------------
static int check_dev_col(const csv_ctx* c, const void* p, const char* name);

// the pending and installed alignment rows of a scanned accumulation (k_scan_aln, k_scan_aln_gather)
struct AlnCols {
    int32_t *chrom, *start, *end, *id;
    uint8_t* prim;
};
// csv_sort_sigs' columns of one type (sigsort_api.inl)
struct SsCols {
    const int32_t *chrom, *a, *b, *rid, *c;
    int type;
};

// The signatures of one SV type: contig, a, b, read id and (INS / INV / TRA) c, 4 B per row each
struct SigTable {
    int64_t n = 0;
    bool has_c = false;
    DBuf chrom, a, b, rid, c;
    // capacity for `rows` rows of every column but c, which copy_in sizes when the source carries it
    int size(int64_t rows) {
        const size_t bytes = (size_t)rows * 4;
        for (DBuf* col : {&chrom, &a, &b, &rid}) CU(col->ensure(bytes));
        return CSV_OK;
    }
    // capacity for `rows` rows of all five columns, keeping the first keep_rows (append mode)
    int grow(int64_t rows, int64_t keep_rows, cudaStream_t s) {
        for (DBuf* col : {&chrom, &a, &b, &rid, &c}) CU(col->grow((size_t)rows * 4, (size_t)keep_rows * 4, s));
        return CSV_OK;
    }
    // the caller's h.n rows; without chrom for a grouped upload (k_expand_contigs writes it)
    int copy_in(const csv_sig_cols& h, bool with_chrom, cudaMemcpyKind kind, cudaStream_t s) {
        const size_t bytes = (size_t)h.n * 4;
        if (with_chrom) CU(cudaMemcpyAsync(chrom.p, h.chrom, bytes, kind, s));
        CU(cudaMemcpyAsync(a.p, h.a, bytes, kind, s));
        CU(cudaMemcpyAsync(b.p, h.b, bytes, kind, s));
        CU(cudaMemcpyAsync(rid.p, h.read_id, bytes, kind, s));
        if (h.c) { CU(c.ensure(bytes)); CU(cudaMemcpyAsync(c.p, h.c, bytes, kind, s)); }
        return CSV_OK;
    }
    // device uploads: every non-null column of h is device memory of the ctx's device
    static int check_dev(const csv_ctx* ctx, const csv_sig_cols& h, bool with_chrom) {
        const void* col[5] = {with_chrom ? h.chrom : nullptr, h.a, h.b, h.read_id, h.c};
        static const char* const nm[5] = {"chrom", "a", "b", "read_id", "c"};
        for (int k = 0; k < 5; k++) { int rc = check_dev_col(ctx, col[k], nm[k]); if (rc) return rc; }
        return CSV_OK;
    }
    // rows [first, first + count) into the host columns that are not null (c only when the table has it); not synchronised
    int fetch(int64_t first, int64_t count, int32_t* h_chrom, int32_t* h_a, int32_t* h_b, int32_t* h_rid, int32_t* h_c, cudaStream_t s) const {
        const size_t bytes = (size_t)count * 4, o = (size_t)first * 4;
        CU(chrom.fetch(h_chrom, o, bytes, s)); CU(a.fetch(h_a, o, bytes, s)); CU(b.fetch(h_b, o, bytes, s)); CU(rid.fetch(h_rid, o, bytes, s));
        if (has_c) CU(c.fetch(h_c, o, bytes, s));
        return CSV_OK;
    }
    // chrom, a, b, rid, c: the order of ExtractOut::col[t], TieCols::col and k_swap_rows
    void cols(int32_t* col[5]) const {
        col[0] = chrom.as<int32_t>(); col[1] = a.as<int32_t>(); col[2] = b.as<int32_t>(); col[3] = rid.as<int32_t>(); col[4] = c.as<int32_t>();
    }
    SsCols sort_cols(int type) const {
        return SsCols{chrom.as<int32_t>(), a.as<int32_t>(), b.as<int32_t>(), rid.as<int32_t>(), has_c ? c.as<int32_t>() : nullptr, type};
    }
};

// Rows shaped like the reads table: contig, start, end, read id (4 B each) and is_primary (1 B unless sized wider)
struct RowTable {
    int64_t n = 0;
    DBuf chrom, start, end, rid, prim;
    // capacity for `rows` rows; prim_size: bytes per is_primary entry
    int size(int64_t rows, size_t prim_size = 1) {
        const size_t bytes = (size_t)rows * 4;
        for (DBuf* col : {&chrom, &start, &end, &rid}) CU(col->ensure(bytes));
        CU(prim.ensure((size_t)rows * prim_size));
        return CSV_OK;
    }
    // capacity for `rows` rows, keeping the first keep_rows (append mode)
    int grow(int64_t rows, int64_t keep_rows, cudaStream_t s) {
        for (DBuf* col : {&chrom, &start, &end, &rid}) CU(col->grow((size_t)rows * 4, (size_t)keep_rows * 4, s));
        CU(prim.grow((size_t)rows, (size_t)keep_rows, s));
        return CSV_OK;
    }
    // h has every column the copy needs (a grouped upload has no chrom)
    static bool has_cols(const csv_reads_cols& h, bool with_chrom) {
        return (!with_chrom || h.chrom) && h.start && h.end && h.read_id && h.is_primary;
    }
    // the caller's h.n rows; without chrom for a grouped upload (k_expand_contigs writes it)
    int copy_in(const csv_reads_cols& h, bool with_chrom, cudaMemcpyKind kind, cudaStream_t s) {
        if (h.n == 0) return CSV_OK;
        const size_t bytes = (size_t)h.n * 4;
        if (with_chrom) CU(cudaMemcpyAsync(chrom.p, h.chrom, bytes, kind, s));
        CU(cudaMemcpyAsync(start.p, h.start, bytes, kind, s));
        CU(cudaMemcpyAsync(end.p, h.end, bytes, kind, s));
        CU(cudaMemcpyAsync(rid.p, h.read_id, bytes, kind, s));
        CU(cudaMemcpyAsync(prim.p, h.is_primary, (size_t)h.n, kind, s));
        return CSV_OK;
    }
    // device uploads: every non-null column of h is device memory of the ctx's device
    static int check_dev(const csv_ctx* ctx, const csv_reads_cols& h, bool with_chrom) {
        const void* col[5] = {with_chrom ? h.chrom : nullptr, h.start, h.end, h.read_id, h.is_primary};
        static const char* const nm[5] = {"chrom", "start", "end", "read_id", "is_primary"};
        for (int k = 0; k < 5; k++) { int rc = check_dev_col(ctx, col[k], nm[k]); if (rc) return rc; }
        return CSV_OK;
    }
    // rows [first, first + count) into the host columns that are not null; not synchronised
    int fetch(int64_t first, int64_t count, int32_t* h_chrom, int32_t* h_start, int32_t* h_end, int32_t* h_rid, uint8_t* h_prim,
              cudaStream_t s) const {
        const size_t bytes = (size_t)count * 4, o = (size_t)first * 4;
        CU(chrom.fetch(h_chrom, o, bytes, s)); CU(start.fetch(h_start, o, bytes, s)); CU(end.fetch(h_end, o, bytes, s));
        CU(rid.fetch(h_rid, o, bytes, s)); CU(prim.fetch(h_prim, (size_t)first, (size_t)count, s));
        return CSV_OK;
    }
    AlnCols cols() const { return AlnCols{chrom.as<int32_t>(), start.as<int32_t>(), end.as<int32_t>(), rid.as<int32_t>(), prim.as<uint8_t>()}; }
    GcReads gc_reads() const { return GcReads{chrom.as<int32_t>(), start.as<int32_t>(), end.as<int32_t>(), rid.as<int32_t>(), prim.as<uint8_t>(), n}; }
    // k_extract's reads-row outputs
    void extract_out(ExtractOut& O) const {
        O.rr_chrom = chrom.as<int32_t>(); O.rr_start = start.as<int32_t>(); O.rr_end = end.as<int32_t>(); O.rr_id = rid.as<int32_t>();
        O.rr_prim = prim.as<uint8_t>();
    }
};

// An alignment table (BAM order) and its contig index of aln_index: first row (off) and longest row (span) per contig
struct AlnTable : RowTable {
    DBuf off, span;
    int size_index(int32_t n_contigs) {
        const size_t bytes = ((size_t)n_contigs + 2) * 4;
        CU(off.ensure(bytes)); CU(span.ensure(bytes));
        return CSV_OK;
    }
    AlnView view(const int64_t* contig_len) const {
        return AlnView{chrom.as<int32_t>(), start.as<int32_t>(), end.as<int32_t>(), rid.as<int32_t>(), prim.as<uint8_t>(), off.as<uint32_t>(),
                       span.as<int32_t>(), contig_len};
    }
};

struct SmallWork {  // DUP / INV / TRA
    DBuf k_rid, k_b, k_prim, perm_a, perm_b, sel, u_chrom, u_a, u_b, u_rid, u_c;
};

// What the packets of an accumulation are; every packet of one accumulation is of one kind.  Named: the records carry read
// names instead of read ids (csv_extract*_named_device); scanned: every decoded record of a BAM packet
// (csv_scan_append_named_device, always named), with or without the alignment rows.
enum class PacketKind { PLAIN, NAMED, SCANNED, SCANNED_ALN };
static inline bool kind_named(PacketKind k) { return k != PacketKind::PLAIN; }
static inline bool kind_scanned(PacketKind k) { return k == PacketKind::SCANNED || k == PacketKind::SCANNED_ALN; }

// Upload state of one input slot: the signatures of an SV type, or the reads table
struct UploadSlot {
    cudaEvent_t ev = nullptr;   // end of the slot's last upload on the copy stream
    bool pending = false;       // ... not yet waited for
    bool device = false;        // the pending upload copies device memory
    bool checked = false;       // the slot's offsets were checked on the device
    DBuf goff;                  // contig row offsets of a grouped upload
};

// Pinned staging of the extraction stage's small copies, one field per use
struct ExStaging {
    uint32_t out[16];        // k_extract's counters, read back
    uint32_t base[16];       // the counters at the start of a packet, H2D (a rerun must not race the previous copy)
    uint32_t seq[8];         // the sequence builder's words [0, 8), read back
    uint32_t bad;            // k_check_packet's error word
    int64_t name_span[2];    // a named packet's name_off[0] and name_off[n]
};

// Words of ExtractState::seq_words (the sequence builder, seq_scan and k_check_packet; zeroed before each use)
enum : int { SW_TICKET = 0, SW_TOTAL = 1, SW_STATUS = 2, SW_TOTAL64 = 4, SW_EPOCH = 8, SW_WORDS = 16 };

struct ExtractState {
    DBuf r[7], cigar_off, sa_off, cigar, s[7], piece_off, piece_cnt, pieces, counters;
    DBuf rec[CSV_NTYPES + 1];        // record index of every extracted signature per type / reads row (last)
    bool rec_on = false;             // csv_extract_records: store the record column (off: no allocation, no stores)
    bool rec_valid = false;          // the device-resident rows are csv_extract* output with the column stored for all of them
    ExStaging* h = nullptr;          // pinned
    uint32_t n_pieces = 0;
    uint32_t n_records = 0;          // alignment records of all packets of the accumulation (record index base of INS pieces)
    uint32_t n_skipped = 0;
    bool appending = false;
    // INS sequence arena (csv_extract*_device with bases): ASCII bytes, start and length per INS row
    DBuf ins_bytes, ins_start, ins_len, seq_tmp, seq_lb, seq_words, fetch_rows, fetch_off, fetch_out;
    bool seq_valid = false;          // every packet of the accumulation carried bases
    int64_t ins_nbytes = 0;
    // read-name arena (csv_extract*_named_device): the names of all records of the accumulation, name i at bytes
    // [name_off[i], name_off[i + 1]); the records' provisional read ids are their indices.  csv_rank_names adds the tables
    // record -> dense rank and rank -> (start, length).
    DBuf name_bytes, name_off, pid, name_rank, name_tab_start, name_tab_len, name_words;
    PacketKind kind = PacketKind::PLAIN;
    bool ranked = false;             // csv_rank_names has turned the provisional ids into ranks
    int64_t name_nbytes = 0, n_names = 0;
    // scanned accumulation (csv_scan_append_named_device, scan_api.inl): every decoded record of each packet.  scan_flag is the
    // packet's flag column with 256 on every record the reference would not extract; pending the alignment rows (BAM order,
    // provisional ids) that csv_rank_names installs; rg_* the region table of csv_set_scan_regions.
    DBuf scan_flag, scan_excl;
    RowTable pending;
    DBuf rg_win_off, rg_win_start, rg_reg_off, rg_reg;
    int32_t rg_n_contigs = 0;        // 0: no region table
    double per_record[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // largest yield of a packet so far: signatures per type [0..4], pieces [5] per alignment record
};

// SA:Z text reduced on the device (sa_api.inl): csv_set_contig_names' table (names sorted bytewise, their contig ids) and the
// outputs of csv_reduce_sa_device in two sets, so that a call that fails leaves the previous outputs as they were
struct SaState {
    DBuf name_bytes, name_off, name_id, cnt;
    int64_t n_names = 0;             // 0: no table
    DBuf off[2], col[2][7];          // sa_off and the seven csv_sa_cols columns of each set
    int cur = 0;                     // the set of the last successful call
};

// Lanes: SV types are independent until the `order` stage, so their kernel chains run concurrently on
// separate streams, one lane per SV type (lane t runs type t; lane 0's stream is the ctx stream).  With lanes off every type
// runs on lane 0.  A lane owns its stream's launch state and the scratch its chain mutates; the chain's functions take it as
// an argument.
struct Lane {
    cudaStream_t stream = nullptr;
    cudaEvent_t ev_join = nullptr;
    bool used = false;                  // forked from ev_fork in the call being enqueued
    bool prev_is_chain_kernel = false;  // the launch being enqueued directly follows a chain kernel on this stream
    int mark = -1;                      // lane_marks: index of the open back-end interval in kivs
    DBuf keys_a, keys_b, vals_a, vals_b, hist, lb_status, big_list, giant_list, giant_arena;
    DBuf boff, rec_a, recc_a, rest_list;   // partitioned INS/DEL front end (edge counts | page table), k_cluster_small's rest list
    SmallWork small;
};
static constexpr int N_LANES = CSV_NTYPES;

// Look-back ticket words of one family of calls, zeroed at the start of every call.  A TileSync's generation is
// *epoch * LB_ORDINALS + ordinal; where the epoch stays 0, ordinals start at ord0 = 1 so that none equals a cleared status word.
struct LbPool {
    uint32_t* tickets = nullptr;
    const uint32_t* epoch = nullptr;
    uint32_t ord0 = 0;
    int next = 0, cap = 0;
};

// scratch of csv_overlap_cover / csv_call_gt / csv_tra_call_gt (genotype_api.inl): separate from everything csv_cluster uses.
// The host tables of the calls are copied into aln: the drop-ins' reads table (rows only), csv_tra_call_gt's alignment table.
struct GcWork {
    DBuf win, bin_base, bin_start, bin_fill, bin_list, iter, prim, cov_off, ovl_off, cov_fill, ovl_fill, cov_u, ovl_u, lb, words;
    DBuf cov_raw, ovl_raw, cov_ded, ovl_ded, cov_flag, ovl_flag, sup_off, sup, geno;
    DBuf tra_q;
    AlnTable aln;
    uint32_t n_cov = 0, n_ovl = 0;   // raw ids of the last call
};

// scratch of csv_sort_sigs (sigsort_api.inl): separate from everything csv_cluster uses
struct SsWork {
    DBuf keys_a, keys_b, vals_a, vals_b, keep, tie, kchrom, order, off, hist, lb, words;
};

struct csv_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    // uploads run on their own stream so that the H2D copy of the next SV type / the reads table
    // overlaps the kernels of the previous type (e2e is PCIe-bound)
    cudaStream_t copy_stream = nullptr;
    UploadSlot up[CSV_NTYPES + 1];   // last: reads table
    DBuf up_status;                  // one word per slot: k_check_contig_off's result, folded into the next csv_cluster's status
    cudaEvent_t ev_prod = nullptr;   // device uploads: end of the caller's work on its producer stream
    cudaEvent_t ev_done = nullptr;   // end of the last csv_cluster on the compute stream
    bool done_pending = false;
    int n_sm = 132;
    csv_params P;
    bool have_params = false;
    // contigs
    int32_t n_contigs = 0;
    std::vector<int64_t> contig_len;
    std::vector<uint64_t> contig_off;
    int64_t off_pad = 0;
    std::vector<uint8_t> owned;     // csv_set_shard: contigs this ctx works on (empty = all)
    DBuf d_off, d_len, d_len_eff;   // d_len_eff: -1 for contigs outside the shard (input validation)
    // inputs
    SigTable sig[CSV_NTYPES];
    RowTable reads;
    AlnTable aln;
    DBuf tickets, scan_carry, emit_cursor;
    DBuf d_epoch;                    // look-back generation base, bumped by the first kernel of every csv_cluster
    LbPool lb;                       // csv_cluster's look-back tickets, shared by its lanes (ordinals stay unique per call)
    uint32_t epoch_host = 0;
    bool small_chain[CSV_NTYPES] = {false, false, false, false, false};   // chained-sorts fallback after ST_BIG_RUN
    bool prefilter_enabled = true;
    bool records_enabled = true;
    bool small_path_enabled = true;
    int64_t pair_cap_override = 0;
    Lane lanes[N_LANES];           // lanes[0].stream is `stream`
    cudaEvent_t ev_fork = nullptr;
    cudaStream_t side_stream[2] = {nullptr, nullptr};   // DEL / INS: the general cluster kernels beside the register kernel
    cudaEvent_t ev_side_fork[2] = {nullptr, nullptr}, ev_side_join[2] = {nullptr, nullptr};
    cudaStream_t aux_stream = nullptr;   // resets of the genotype stage's scratch run beside the lanes
    cudaEvent_t ev_aux = nullptr;
    bool lanes_enabled = true;
    // segment / cluster
    DBuf kept[CSV_NTYPES], cnt;
    uint32_t kept_cap[CSV_NTYPES] = {0, 0, 0, 0, 0};
    // results
    DBuf cand_tmp, cand, geno, names, counters;
    uint32_t cap_cand = 0, cap_names = 0;
    Counters* h_counters = nullptr;  // pinned
    // genotype
    DBuf bin_start, bin_fill, bin_bits, win_list, win_rec, dr, has_rows, gl_table, pow_half, pairs;
    uint32_t pow_n = 0;
    // state
    bool ran = false, counts_valid = false;
    int64_t launches = 0;
    // profiling: CUDA-event intervals on the launching streams; a stage may be entered once per SV type
    bool profiling = false;
    // csv_set_profiling(c, 2): no per-launch events (programmatic launches, the side streams and the lanes run as they do
    // unprofiled; no graph replay), only one interval per INS / DEL lane from the end of the density filter to the lane's end
    // and one ("tail") from the lane join to the end of the chain
    bool lane_marks = false;
    struct Interval { int st; cudaEvent_t a, b; int64_t bytes; };
    std::vector<Interval> ivs;
    std::vector<cudaEvent_t> ev_pool;
    size_t ev_next = 0;
    bool ivs_consumed = false;
    struct KInterval { const char* name; cudaEvent_t a, b; };
    std::vector<KInterval> kivs;
    struct KTotal { std::string name; int64_t launches; double ms; };
    std::vector<KTotal> ktotals;
    float stage_ms[CSV_ST_COUNT];
    float sort_ms = 0.f;
    int64_t sort_bytes = 0;
    int32_t sort_launches = 0;
    uint32_t last_mask = 0x1f;
    // extraction
    ExtractState ex;
    SaState sa;
    // CUDA graph of one csv_cluster call (kernel chain of all lanes), keyed by everything the enqueue depends on
    struct GraphKey {
        uint32_t mask; int64_t n[CSV_NTYPES]; int64_t n_reads, n_aln; csv_params P; int lanes; uint64_t alloc_epoch; uint64_t cfg_epoch;
        bool small_chain[CSV_NTYPES];
        bool up_checked[CSV_NTYPES + 1];   // the chain folds these slots' device-side offset checks into its status
    };
    struct GraphSlot { bool valid = false; GraphKey key; cudaGraphExec_t exec = nullptr; int64_t launches = 0; uint64_t used = 0; };
    static constexpr int N_GRAPHS = 4;
    GraphSlot graphs[N_GRAPHS];
    GraphKey last_key;
    bool last_key_valid = false;
    bool graphs_enabled = true;
    uint64_t cfg_epoch = 1, graph_clock = 0;   // cfg_epoch: bumped by csv_set_contigs / csv_set_shard
    int64_t graph_replays = 0;
    // multi-GPU (csv_comm_init / csv_allgather)
    struct P2PState {
        bool ready = false, failed = false;
        void* box = nullptr;              // this rank's mail box: 2 buffers x world slots, then 2 x world arrival flags
        int64_t slot_bytes = 0;
        size_t flags_off = 0;
        std::vector<void*> peer;          // every rank's box as mapped here (CUDA IPC)
        DBuf d_tab;                       // device tables of slot / flag pointers + the push kernel's done counter
        unsigned long long epoch = 0;
    } p2p;
    bool p2p_enabled = true;
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1;
    DBuf g_send, g_recv, g_cand, g_geno, g_names, g_scratch, g_tab;
    bool pdl_enabled = true;            // programmatic dependent launches along the kernel chain (CUTESV_B200_PDL=0: off)
    bool pdl_now = false;               // ... for the call being enqueued: only with <= 2 SV-type lanes.  A dependent that is resident
                                        // early holds SM slots while it waits; with 5 lanes sharing the GPU those slots are what the
                                        // other lanes' kernels need
    DBuf cal_in0, cal_in1, cal_out, aln_flag;   // csv_cal_gl / csv_upload_alignments scratch (no per-call cudaMalloc)
    GcWork gc;                                  // csv_overlap_cover / csv_call_gt
    SsWork ss;                                  // csv_sort_sigs
    int64_t pad_cand = 0, pad_names = 0;
    int64_t* h_gather = nullptr;    // pinned: per-rank headers after the gather
    int64_t g_n_cand = 0, g_n_names = 0;
    bool gathered = false;
};

static void kprof_begin(csv_ctx* c, cudaStream_t s, const char* name);
static void kprof_end(csv_ctx* c, cudaStream_t s);
// with profiling on, every launch sits between its own pair of CUDA events on the launching stream `s`
#define LAUNCH_NAMED(ctx, s, name, kernel, grid, block, smem, ...)                    \
    do {                                                                               \
        if ((ctx)->profiling) kprof_begin((ctx), (s), (name));                         \
        kernel<<<(grid), (block), (smem), (s)>>>(__VA_ARGS__);                         \
        if ((ctx)->profiling) kprof_end((ctx), (s));                                   \
        (ctx)->launches++;                                                             \
    } while (0)
#define LAUNCH(ctx, s, kernel, grid, block, smem, ...) LAUNCH_NAMED(ctx, s, #kernel, kernel, grid, block, smem, __VA_ARGS__)
// A kernel that directly follows another kernel of the chain on the same stream (no copy, memset or join in between) and that
// begins with pdl_wait(): launched as a programmatic dependent, so its launch latency and its CTAs' start-up overlap the tail
// of its predecessor.  Captured into the CUDA graph as a programmatic edge.  Off when profiling (events sit between launches).
#define LAUNCH_PDL_NAMED(ctx, s, name, kernel, grid, block, smem, ...)                                       \
    do {                                                                                                      \
        if ((ctx)->pdl_now && !(ctx)->profiling) {                                                            \
            cudaLaunchConfig_t cfg_;                                                                          \
            memset(&cfg_, 0, sizeof(cfg_));                                                                   \
            cfg_.gridDim = dim3((unsigned)(grid)); cfg_.blockDim = dim3((unsigned)(block));                   \
            cfg_.dynamicSmemBytes = (smem); cfg_.stream = (s);                                                \
            cudaLaunchAttribute at_[1];                                                                       \
            at_[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                   \
            at_[0].val.programmaticStreamSerializationAllowed = 1;                                            \
            cfg_.attrs = at_; cfg_.numAttrs = 1;                                                              \
            cudaLaunchKernelEx(&cfg_, kernel, __VA_ARGS__);                                                   \
            (ctx)->launches++;                                                                                \
        } else LAUNCH_NAMED(ctx, s, name, kernel, grid, block, smem, __VA_ARGS__);                            \
    } while (0)
#define LAUNCH_PDL(ctx, s, kernel, grid, block, smem, ...) LAUNCH_PDL_NAMED(ctx, s, #kernel, kernel, grid, block, smem, __VA_ARGS__)

// KIND: the per-type routine of the warp kernel (0 INS/DEL generic, 1 DUP, 2 INV, 3 TRA, 4-7 INS/DEL specialisations, see
// run_cluster); the CTA kernel (rare big clusters) always uses the generic routine BKIND in 0..3
template <int KIND, int BKIND>
static void launch_cluster_kind(csv_ctx* c, cudaStream_t s, const TypeJob& J, const Emit& E, Counters* ctr, uint32_t* work, size_t smem_warp) {
    static const char* const nm_w[8] = {"k_cluster_warp<INDEL>", "k_cluster_warp<DUP>", "k_cluster_warp<INV>", "k_cluster_warp<TRA>",
                                        "k_cluster_warp<DEL>", "k_cluster_warp<INS>", "k_cluster_warp<DEL,keep-all>", "k_cluster_warp<INS,keep-all>"};
    static const char* const nm_b[4] = {"k_cluster_block<INDEL>", "k_cluster_block<DUP>", "k_cluster_block<INV>", "k_cluster_block<TRA>"};
    LAUNCH_NAMED(c, s, nm_w[KIND], (k_cluster_warp<KIND>), c->n_sm * 3, CL_THREADS, smem_warp, J, E, ctr, work);
    LAUNCH_PDL_NAMED(c, s, nm_b[BKIND], (k_cluster_block<BKIND>), c->n_sm, CL_THREADS, (size_t)BLOCK_M * ARENA_PER_MAX, J, E, ctr);
}

static int grid_for(const csv_ctx* c, int64_t n, int block, int per_sm = 8) {
    int64_t g = (n + block - 1) / block;
    int64_t cap = (int64_t)c->n_sm * per_sm;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

// CTAs that are resident at once: the grid of a kernel whose CTAs stride over tiles (a partial second wave would start
// late and finish last)
template <typename K>
static int resident_grid(const csv_ctx* c, K kernel, int block, size_t smem) {
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, smem) != cudaSuccess) { cudaGetLastError(); per_sm = 1; }
    return c->n_sm * std::max(per_sm, 1);
}

static int bits_for(uint64_t max_value) {
    int b = 0;
    while (b < 64 && (max_value >> b) != 0) b++;
    return b < 1 ? 1 : b;
}

// ------------------------------------------------------------------------------------------
// profiling helpers
// ------------------------------------------------------------------------------------------
static constexpr int ST_SORT_PASS = CSV_ST_COUNT;  // pseudo stage: one onesweep launch
static cudaEvent_t pool_event(csv_ctx* c) {
    if (c->ev_next == c->ev_pool.size()) {
        cudaEvent_t e;
        cudaEventCreate(&e);
        c->ev_pool.push_back(e);
    }
    return c->ev_pool[c->ev_next++];
}
static void stage_reset_if_consumed(csv_ctx* c) {
    if (c->ivs_consumed) { c->ivs.clear(); c->kivs.clear(); c->ev_next = 0; c->ivs_consumed = false; }
}
static void kprof_begin(csv_ctx* c, cudaStream_t s, const char* name) {
    stage_reset_if_consumed(c);
    csv_ctx::KInterval k;
    k.name = name; k.a = pool_event(c); k.b = pool_event(c);
    cudaEventRecord(k.a, s);
    c->kivs.push_back(k);
}
static void kprof_end(csv_ctx* c, cudaStream_t s) { cudaEventRecord(c->kivs.back().b, s); }
static void stage_begin(csv_ctx* c, cudaStream_t s, int st, int64_t bytes = 0) {
    if (!c->profiling) return;
    stage_reset_if_consumed(c);
    csv_ctx::Interval iv;
    iv.st = st; iv.a = pool_event(c); iv.b = pool_event(c); iv.bytes = bytes;
    cudaEventRecord(iv.a, s);
    c->ivs.push_back(iv);
}
static void stage_end(csv_ctx* c, cudaStream_t s, int st) {
    if (!c->profiling) return;
    for (size_t i = c->ivs.size(); i-- > 0;)
        if (c->ivs[i].st == st) { cudaEventRecord(c->ivs[i].b, s); return; }
}
static void stage_collect(csv_ctx* c) {  // after a stream synchronize
    for (int s = 0; s < CSV_ST_COUNT; s++) c->stage_ms[s] = 0.f;
    c->sort_ms = 0.f; c->sort_bytes = 0; c->sort_launches = 0;
    for (const csv_ctx::Interval& iv : c->ivs) {
        float t = 0.f;
        if (cudaEventElapsedTime(&t, iv.a, iv.b) != cudaSuccess) { cudaGetLastError(); continue; }
        if (iv.st == ST_SORT_PASS) { c->sort_ms += t; c->sort_bytes += iv.bytes; c->sort_launches++; }
        else c->stage_ms[iv.st] += t;
    }
    c->ktotals.clear();
    for (const csv_ctx::KInterval& k : c->kivs) {
        float t = 0.f;
        if (cudaEventElapsedTime(&t, k.a, k.b) != cudaSuccess) { cudaGetLastError(); continue; }
        std::string nm(k.name);
        if (!nm.empty() && nm.front() == '(' && nm.back() == ')') nm = nm.substr(1, nm.size() - 2);   // "(k_x<..>)" macro argument
        bool found = false;
        for (auto& kt : c->ktotals) if (kt.name == nm) { kt.launches++; kt.ms += t; found = true; break; }
        if (!found) c->ktotals.push_back({nm, 1, (double)t});
    }
    c->ivs_consumed = true;
}

// ------------------------------------------------------------------------------------------
// create / destroy / params
// ------------------------------------------------------------------------------------------
extern "C" int csv_default_params(csv_params* p) {
    if (!p) return set_err(CSV_E_INVALID, "null params");
    memset(p, 0, sizeof(*p));
    p->min_support = 10; p->min_support_allele = 5; p->min_size = 30; p->max_size = 100000;
    p->bias_del = 200; p->bias_ins = 100; p->bias_inv = 500; p->bias_dup = 500; p->bias_tra = 50;
    p->genotype = 0; p->gt_round = 500; p->gt_bias_ins = 1000;
    p->ratio_del = 0.5; p->ratio_ins = 0.3; p->ratio_tra = 0.6; p->remain_reads_ratio = 1.0;
    p->min_mapq = 20; p->max_split_parts = 7; p->min_read_len = 500; p->min_siglength = 10;
    p->merge_del_threshold = 0; p->merge_ins_threshold = 100;
    return CSV_OK;
}

static int upload_tables(csv_ctx* c, uint32_t pow_n) {
    std::vector<csv_geno> gl = build_gl_table();
    CU(c->gl_table.ensure(gl.size() * sizeof(csv_geno)));
    CU(cudaMemcpy(c->gl_table.p, gl.data(), gl.size() * sizeof(csv_geno), cudaMemcpyHostToDevice));
    std::vector<double> ph = build_pow_half(pow_n);
    CU(c->pow_half.ensure(ph.size() * sizeof(double)));
    CU(cudaMemcpy(c->pow_half.p, ph.data(), ph.size() * sizeof(double), cudaMemcpyHostToDevice));
    c->pow_n = pow_n;
    return CSV_OK;
}

extern "C" int csv_create(int device, void* stream, csv_ctx** out) {
    if (!out) return set_err(CSV_E_INVALID, "null out");
    int n_dev = 0;
    cudaError_t e = cudaGetDeviceCount(&n_dev);
    if (e != cudaSuccess || n_dev == 0)
        return set_err(CSV_E_NODEVICE, "no CUDA device (%s): cutesv_b200 has no CPU fallback",
                       e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    if (device < 0 || device >= n_dev) return set_err(CSV_E_INVALID, "device %d out of range (%d devices)", device, n_dev);
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)   // sm_90a code loads on compute capability 9.0 only
        return set_err(CSV_E_NODEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
    CU(cudaSetDevice(device));
    csv_ctx* c = new csv_ctx();
    c->device = device;
    c->n_sm = prop.multiProcessorCount;
    if (stream) { c->stream = (cudaStream_t)stream; c->own_stream = false; }
    else {
        cudaError_t e2 = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
        if (e2 != cudaSuccess) { delete c; return set_err(CSV_E_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e2)); }
        c->own_stream = true;
    }
    c->lanes[0].stream = c->stream;
    {
        cudaError_t e4 = cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking);
        for (UploadSlot& u : c->up) if (e4 == cudaSuccess) e4 = cudaEventCreateWithFlags(&u.ev, cudaEventDisableTiming);
        if (e4 == cudaSuccess) e4 = cudaEventCreateWithFlags(&c->ev_done, cudaEventDisableTiming);
        if (e4 == cudaSuccess) e4 = cudaEventCreateWithFlags(&c->ev_prod, cudaEventDisableTiming);
        if (e4 == cudaSuccess) e4 = cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming);
        if (e4 == cudaSuccess) e4 = cudaStreamCreateWithFlags(&c->aux_stream, cudaStreamNonBlocking);
        if (e4 == cudaSuccess) e4 = cudaEventCreateWithFlags(&c->ev_aux, cudaEventDisableTiming);
        for (int k = 0; k < 2 && e4 == cudaSuccess; k++) {
            e4 = cudaStreamCreateWithFlags(&c->side_stream[k], cudaStreamNonBlocking);
            if (e4 == cudaSuccess) e4 = cudaEventCreateWithFlags(&c->ev_side_fork[k], cudaEventDisableTiming);
            if (e4 == cudaSuccess) e4 = cudaEventCreateWithFlags(&c->ev_side_join[k], cudaEventDisableTiming);
        }
        for (int l = 1; l < N_LANES && e4 == cudaSuccess; l++) {   // lane 0 never joins: it is the ctx stream
            e4 = cudaStreamCreateWithFlags(&c->lanes[l].stream, cudaStreamNonBlocking);
            if (e4 == cudaSuccess) e4 = cudaEventCreateWithFlags(&c->lanes[l].ev_join, cudaEventDisableTiming);
        }
        if (e4 != cudaSuccess) { delete c; return set_err(CSV_E_CUDA, "copy stream / lanes: %s", cudaGetErrorString(e4)); }
    }
    csv_default_params(&c->P);
    if (const char* e = getenv("CUTESV_B200_PAIR_CAP")) c->pair_cap_override = atoll(e);
    if (const char* e = getenv("CUTESV_B200_NO_PREFILTER")) c->prefilter_enabled = atoi(e) == 0;
    if (const char* e = getenv("CUTESV_B200_LANES")) c->lanes_enabled = atoi(e) != 0;
    if (const char* e = getenv("CUTESV_B200_GRAPHS")) c->graphs_enabled = atoi(e) != 0;
    if (const char* e = getenv("CUTESV_B200_PDL")) c->pdl_enabled = atoi(e) != 0;
    if (const char* e = getenv("CUTESV_B200_GATHER")) c->p2p_enabled = strcmp(e, "nccl") != 0;
    if (const char* e = getenv("CUTESV_B200_RECORDS")) c->records_enabled = atoi(e) != 0;
    if (const char* e = getenv("CUTESV_B200_SMALL_PATH")) c->small_path_enabled = atoi(e) != 0;
    if (const char* e = getenv("CUTESV_B200_SMALL_CHAIN")) for (int t = 0; t < CSV_NTYPES; t++) c->small_chain[t] = atoi(e) != 0;
    for (int s = 0; s < CSV_ST_COUNT; s++) c->stage_ms[s] = 0.f;
    cudaError_t e3 = cudaMallocHost((void**)&c->h_counters, sizeof(Counters));
    if (e3 != cudaSuccess) { delete c; return set_err(CSV_E_CUDA, "cudaMallocHost: %s", cudaGetErrorString(e3)); }
    int rc = upload_tables(c, 1u << 16);
    if (rc != CSV_OK) { delete c; return rc; }
    CU(c->d_epoch.ensure(64, true));
    CU(c->emit_cursor.ensure(256, true));
    CU(c->up_status.ensure((CSV_NTYPES + 1) * 4, true));
    // opt in to large dynamic shared memory for the cluster kernels
    const int smem_warp = (CL_THREADS / 32) * WARP_M * ARENA_PER_MAX + (CL_THREADS / 32) * 40 * 8;
    CU(cudaFuncSetAttribute(k_cluster_warp<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_warp));
    CU(cudaFuncSetAttribute(k_cluster_warp<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_warp));
    CU(cudaFuncSetAttribute(k_cluster_warp<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_warp));
    CU(cudaFuncSetAttribute(k_cluster_warp<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_warp));
    CU(cudaFuncSetAttribute(k_cluster_warp<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_warp));
    CU(cudaFuncSetAttribute(k_cluster_warp<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_warp));
    CU(cudaFuncSetAttribute(k_cluster_warp<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_warp));
    CU(cudaFuncSetAttribute(k_cluster_warp<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_warp));
    CU(cudaFuncSetAttribute(k_cluster_block<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, BLOCK_M * ARENA_PER_MAX));
    CU(cudaFuncSetAttribute(k_cluster_block<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, BLOCK_M * ARENA_PER_MAX));
    CU(cudaFuncSetAttribute(k_cluster_block<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, BLOCK_M * ARENA_PER_MAX));
    CU(cudaFuncSetAttribute(k_cluster_block<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, BLOCK_M * ARENA_PER_MAX));
    CU(cudaFuncSetAttribute(k_part_filter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pf_smem_bytes(PART_W_MAX)));
    CU(cudaFuncSetAttribute(k_part_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ps_smem_bytes()));
    *out = c;
    return CSV_OK;
}

extern "C" int csv_destroy(csv_ctx* c) {
    if (!c) return CSV_OK;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    for (auto& g : c->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
    if (c->comm) comm_destroy(c);
    if (c->h_gather) cudaFreeHost(c->h_gather);
    for (int l = 1; l < N_LANES; l++) {
        Lane& L = c->lanes[l];
        if (L.stream) { cudaStreamSynchronize(L.stream); cudaStreamDestroy(L.stream); }
        if (L.ev_join) cudaEventDestroy(L.ev_join);
    }
    if (c->ev_fork) cudaEventDestroy(c->ev_fork);
    if (c->aux_stream) { cudaStreamSynchronize(c->aux_stream); cudaStreamDestroy(c->aux_stream); }
    if (c->ev_aux) cudaEventDestroy(c->ev_aux);
    for (int k = 0; k < 2; k++) {
        if (c->side_stream[k]) { cudaStreamSynchronize(c->side_stream[k]); cudaStreamDestroy(c->side_stream[k]); }
        if (c->ev_side_fork[k]) cudaEventDestroy(c->ev_side_fork[k]);
        if (c->ev_side_join[k]) cudaEventDestroy(c->ev_side_join[k]);
    }
    if (c->ex.h) cudaFreeHost(c->ex.h);
    for (cudaEvent_t e : c->ev_pool) cudaEventDestroy(e);
    if (c->h_counters) cudaFreeHost(c->h_counters);
    if (c->copy_stream) { cudaStreamSynchronize(c->copy_stream); cudaStreamDestroy(c->copy_stream); }
    for (UploadSlot& u : c->up) if (u.ev) cudaEventDestroy(u.ev);
    if (c->ev_done) cudaEventDestroy(c->ev_done);
    if (c->ev_prod) cudaEventDestroy(c->ev_prod);
    if (c->own_stream) cudaStreamDestroy(c->stream);
    delete c;   // frees every device buffer (DBuf), on c->device
    return CSV_OK;
}

extern "C" int csv_set_params(csv_ctx* c, const csv_params* p) {
    if (!c || !p) return set_err(CSV_E_INVALID, "null argument");
    if (p->min_support < 1) return set_err(CSV_E_INVALID, "min_support must be >= 1");
    if (p->bias_del < 1 || p->bias_ins < 1 || p->bias_inv < 1 || p->bias_dup < 1 || p->bias_tra < 1 || p->gt_bias_ins < 1)
        return set_err(CSV_E_INVALID, "max_cluster_bias_* must be >= 1");
    const int64_t old_pad = c->off_pad;
    c->P = *p;
    c->have_params = true;
    c->counts_valid = false;
    // the linear coordinate pads every contig by more than the largest bias
    int64_t pad = std::max<int64_t>({p->bias_del, p->bias_ins, p->bias_inv, p->bias_dup, p->bias_tra, p->gt_bias_ins}) + 1;
    if (pad != old_pad && c->n_contigs > 0) {
        std::vector<int64_t> lens = c->contig_len;
        c->off_pad = pad;
        return csv_set_contigs(c, (int32_t)lens.size(), lens.data());
    }
    c->off_pad = pad;
    return CSV_OK;
}

extern "C" int csv_set_contigs(csv_ctx* c, int32_t n, const int64_t* lens) {
    if (!c || n < 1 || !lens) return set_err(CSV_E_INVALID, "bad contig table");
    // TRA signatures and candidates carry chr2*4+type in int32
    if (n >= (1 << 29)) return set_err(CSV_E_INVALID, "%d contigs: at most 2^29 - 1 are supported", n);
    CU(cudaSetDevice(c->device));
    if (c->off_pad == 0) csv_set_params(c, &c->P);
    if ((int32_t)c->owned.size() != n) c->owned.clear();   // a new table drops the shard mask
    if (c->sa.n_names != n) c->sa.n_names = 0;             // ... and the contig names
    std::vector<int64_t> keep(lens, lens + n);   // (lens may alias c->contig_len)
    c->n_contigs = n;
    c->contig_len = keep;
    c->contig_off.resize(n + 1);
    std::vector<int64_t> eff(n);
    uint64_t run = 0;
    for (int i = 0; i < n; i++) {
        if (keep[i] < 0 || keep[i] >= (1ll << 31)) return set_err(CSV_E_INVALID, "contig %d length %lld out of range", i, (long long)keep[i]);
        const bool mine = c->owned.empty() || c->owned[i];
        c->contig_off[i] = run;
        // contigs outside the shard take no room in the linear coordinate (the bucket / bin tables scale with the shard)
        run += mine ? (uint64_t)keep[i] + (uint64_t)c->off_pad : 0ull;
        eff[i] = mine ? keep[i] : -1;
    }
    c->contig_off[n] = run;
    CU(c->d_off.ensure((n + 1) * sizeof(uint64_t)));
    CU(c->d_len.ensure(n * sizeof(int64_t)));
    CU(c->d_len_eff.ensure(n * sizeof(int64_t)));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaMemcpy(c->d_off.p, c->contig_off.data(), (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(c->d_len.p, c->contig_len.data(), n * sizeof(int64_t), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(c->d_len_eff.p, eff.data(), n * sizeof(int64_t), cudaMemcpyHostToDevice));
    c->counts_valid = false;
    c->cfg_epoch++;
    return CSV_OK;
}

extern "C" int csv_set_shard(csv_ctx* c, const uint8_t* owned) {
    if (!c) return set_err(CSV_E_INVALID, "null ctx");
    if (c->n_contigs == 0) return set_err(CSV_E_STATE, "csv_set_contigs has not been called");
    if (owned) c->owned.assign(owned, owned + c->n_contigs); else c->owned.clear();
    std::vector<int64_t> lens = c->contig_len;
    return csv_set_contigs(c, (int32_t)lens.size(), lens.data());
}

extern "C" int csv_host_alloc(void** p, size_t bytes) {
    if (!p) return set_err(CSV_E_INVALID, "null");
    CU(cudaMallocHost(p, bytes ? bytes : 1));
    return CSV_OK;
}
extern "C" int csv_host_free(void* p) { if (p) CU(cudaFreeHost(p)); return CSV_OK; }
extern "C" int csv_host_register(void* p, size_t bytes) { CU(cudaHostRegister(p, bytes, cudaHostRegisterDefault)); return CSV_OK; }
extern "C" int csv_host_unregister(void* p) { CU(cudaHostUnregister(p)); return CSV_OK; }

extern "C" int csv_set_lanes(csv_ctx* c, int on) {
    if (!c) return set_err(CSV_E_INVALID, "null ctx");
    c->lanes_enabled = on != 0;
    return CSV_OK;
}

extern "C" int csv_set_profiling(csv_ctx* c, int on) {
    if (!c) return set_err(CSV_E_INVALID, "null ctx");
    CU(cudaSetDevice(c->device));
    c->profiling = on == 1;
    c->lane_marks = on == 2;
    return CSV_OK;
}

// ------------------------------------------------------------------------------------------
// uploads
// ------------------------------------------------------------------------------------------
// Where the columns of one upload live.  Host columns (csv_upload_*) are H2D copies; device columns (csv_upload_*_device) are
// device-to-device copies ordered after the work the caller enqueued on its producer stream, and that stream in turn waits for the
// copies, so the caller may overwrite or free its buffers in stream order as soon as the call returns.  Either way the ctx owns
// its inputs: csv_remap_read_ids / csv_swap_ins_rows rewrite them and captured graphs hold their addresses.
struct UpSrc {
    bool device;
    cudaStream_t producer;   // device: the caller's stream (0 = the legacy default stream)
    cudaMemcpyKind kind() const { return device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice; }
};
static const UpSrc HOST_SRC = {false, nullptr};

// Device calls: every non-null column must be device (or managed) memory of the ctx's device.
static int check_dev_col(const csv_ctx* c, const void* p, const char* name) {
    if (!p) return CSV_OK;
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return set_err(CSV_E_INVALID, "column %s: not a CUDA pointer (%s)", name, cudaGetErrorString(e));
    }
    if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged)
        return set_err(CSV_E_INVALID, "column %s is not device memory (host pointers go to the calls without _device)", name);
    if (a.device != c->device) return set_err(CSV_E_INVALID, "column %s is on device %d, the ctx on device %d", name, a.device, c->device);
    return CSV_OK;
}

// The copy stream must not overwrite inputs that kernels of the previous csv_cluster still read, nor read device columns before
// the caller's producer stream wrote them.
static int upload_begin(csv_ctx* c, const UpSrc& src) {
    if (c->done_pending) {
        CU(cudaStreamWaitEvent(c->copy_stream, c->ev_done, 0));
        c->done_pending = false;
    }
    if (src.device) {
        CU(cudaEventRecord(c->ev_prod, src.producer));
        CU(cudaStreamWaitEvent(c->copy_stream, c->ev_prod, 0));
    }
    return CSV_OK;
}
static int upload_end(csv_ctx* c, int slot, const UpSrc& src) {
    UploadSlot& u = c->up[slot];
    CU(cudaEventRecord(u.ev, c->copy_stream));
    if (src.device) CU(cudaStreamWaitEvent(src.producer, u.ev, 0));
    u.pending = true;
    u.device = src.device;
    return CSV_OK;
}
static int wait_upload(csv_ctx* c, cudaStream_t s, int slot) {
    UploadSlot& u = c->up[slot];
    if (u.pending) {
        CU(cudaStreamWaitEvent(s, u.ev, 0));
        u.pending = false;
    }
    return CSV_OK;
}
// Grouped uploads: rows grouped by contig id (ascending) + n_contigs+1 row offsets instead of the 4-byte contig
// column; the column is rebuilt on the device behind the copies (k_expand_contigs on the copy stream).  Host offsets are checked
// here; device offsets are checked on the device (reading them here would need a synchronisation), and a failure is reported by
// the next csv_cluster as CSV_E_INPUT.
static int stage_group_offsets(csv_ctx* c, int slot, const int64_t* off, int64_t n, int32_t* chrom_dev, const UpSrc& src) {
    if (c->n_contigs == 0) return set_err(CSV_E_STATE, "csv_set_contigs has not been called");
    if (!src.device) {
        if (off[0] != 0 || off[c->n_contigs] != n) return set_err(CSV_E_INVALID, "contig_off must start at 0 and end at n");
        for (int k = 0; k < c->n_contigs; k++)
            if (off[k + 1] < off[k]) return set_err(CSV_E_INVALID, "contig_off must be non-decreasing");
    }
    UploadSlot& u = c->up[slot];
    CU(u.goff.ensure(((size_t)c->n_contigs + 1) * 8));
    CU(cudaMemcpyAsync(u.goff.p, off, ((size_t)c->n_contigs + 1) * 8, src.kind(), c->copy_stream));
    uint32_t* bad = nullptr;
    if (src.device) {
        bad = c->up_status.as<uint32_t>() + slot;
        CU(cudaMemsetAsync(bad, 0, 4, c->copy_stream));
        k_check_contig_off<<<grid_for(c, (int64_t)c->n_contigs + 1, 256), 256, 0, c->copy_stream>>>(u.goff.as<int64_t>(), c->n_contigs, n, bad);
        c->launches++;
        u.checked = true;
    }
    k_expand_contigs<<<grid_for(c, n, 256 * 4), 256, 0, c->copy_stream>>>(u.goff.as<int64_t>(), c->n_contigs, n, chrom_dev, bad);
    c->launches++;
    return CSV_OK;
}

// An upload replaced the device-resident inputs of one slot (an SV type, or the reads table): the rows no longer come from the
// accumulation, which otherwise stays as it is
static void inputs_replaced(csv_ctx* c, int slot) {
    c->counts_valid = false;
    c->ex.rec_valid = false;
    c->ex.seq_valid = false;
    c->ex.kind = PacketKind::PLAIN; c->ex.ranked = false;
    c->ex.pending.n = 0;
    c->up[slot].checked = false;
}

static int upload_sigs_impl(csv_ctx* c, int t, const csv_sig_cols* h, const int64_t* contig_off, const UpSrc& src) {
    if (!c || t < 0 || t >= CSV_NTYPES || !h) return set_err(CSV_E_INVALID, "bad argument");
    if (h->n < 0 || h->n >= (1ll << 30)) return set_err(CSV_E_INVALID, "signature count %lld out of range", (long long)h->n);
    CU(cudaSetDevice(c->device));
    SigTable& s = c->sig[t];
    s.n = h->n;
    s.has_c = h->c != nullptr;
    inputs_replaced(c, t);
    if (h->n == 0) return CSV_OK;
    if ((!contig_off && !h->chrom) || !h->a || !h->b || !h->read_id) return set_err(CSV_E_INVALID, "null column");
    if ((t == CSV_INS || t == CSV_INV || t == CSV_TRA) && !h->c) return set_err(CSV_E_INVALID, "column c is required for INS/INV/TRA");
    int rc;
    if (src.device && ((rc = SigTable::check_dev(c, *h, !contig_off)) || (rc = check_dev_col(c, contig_off, "contig_off")))) return rc;
    if ((rc = upload_begin(c, src)) || (rc = s.size(h->n))) return rc;
    if (contig_off && (rc = stage_group_offsets(c, t, contig_off, h->n, s.chrom.as<int32_t>(), src))) return rc;
    if ((rc = s.copy_in(*h, !contig_off, src.kind(), c->copy_stream))) return rc;
    return upload_end(c, t, src);
}
extern "C" int csv_upload_sigs(csv_ctx* c, int t, const csv_sig_cols* h) { return upload_sigs_impl(c, t, h, nullptr, HOST_SRC); }
extern "C" int csv_upload_sigs_grouped(csv_ctx* c, int t, const csv_sig_cols* h, const int64_t* contig_off) {
    if (!contig_off) return set_err(CSV_E_INVALID, "null contig_off");
    return upload_sigs_impl(c, t, h, contig_off, HOST_SRC);
}
extern "C" int csv_upload_sigs_device(csv_ctx* c, int t, const csv_sig_cols* d, void* stream) {
    return upload_sigs_impl(c, t, d, nullptr, UpSrc{true, (cudaStream_t)stream});
}
extern "C" int csv_upload_sigs_grouped_device(csv_ctx* c, int t, const csv_sig_cols* d, const int64_t* contig_off, void* stream) {
    if (!contig_off) return set_err(CSV_E_INVALID, "null contig_off");
    return upload_sigs_impl(c, t, d, contig_off, UpSrc{true, (cudaStream_t)stream});
}

static int upload_reads_impl(csv_ctx* c, const csv_reads_cols* h, const int64_t* contig_off, const UpSrc& src) {
    if (!c || !h) return set_err(CSV_E_INVALID, "bad argument");
    if (h->n < 0 || h->n >= (1ll << 31)) return set_err(CSV_E_INVALID, "read count out of range");
    CU(cudaSetDevice(c->device));
    RowTable& r = c->reads;
    r.n = h->n;
    inputs_replaced(c, CSV_NTYPES);
    if (h->n == 0) return CSV_OK;
    if (!RowTable::has_cols(*h, !contig_off)) return set_err(CSV_E_INVALID, "null column");
    int rc;
    if (src.device && ((rc = RowTable::check_dev(c, *h, !contig_off)) || (rc = check_dev_col(c, contig_off, "contig_off")))) return rc;
    if ((rc = upload_begin(c, src)) || (rc = r.size(h->n))) return rc;
    if (contig_off && (rc = stage_group_offsets(c, CSV_NTYPES, contig_off, h->n, r.chrom.as<int32_t>(), src))) return rc;
    if ((rc = r.copy_in(*h, !contig_off, src.kind(), c->copy_stream))) return rc;
    return upload_end(c, CSV_NTYPES, src);
}

extern "C" int csv_upload_reads(csv_ctx* c, const csv_reads_cols* h) { return upload_reads_impl(c, h, nullptr, HOST_SRC); }
extern "C" int csv_upload_reads_grouped(csv_ctx* c, const csv_reads_cols* h, const int64_t* contig_off) {
    if (!contig_off) return set_err(CSV_E_INVALID, "null contig_off");
    return upload_reads_impl(c, h, contig_off, HOST_SRC);
}
extern "C" int csv_upload_reads_device(csv_ctx* c, const csv_reads_cols* d, void* stream) {
    return upload_reads_impl(c, d, nullptr, UpSrc{true, (cudaStream_t)stream});
}
extern "C" int csv_upload_reads_grouped_device(csv_ctx* c, const csv_reads_cols* d, const int64_t* contig_off, void* stream) {
    if (!contig_off) return set_err(CSV_E_INVALID, "null contig_off");
    return upload_reads_impl(c, d, contig_off, UpSrc{true, (cudaStream_t)stream});
}

// Contig index (off, span: n_contigs + 2 entries) + sortedness check of the rows of an alignment table (BAM order is a
// precondition of the early-exit scan); one synchronisation.  A failure leaves the table empty.
static int aln_index(csv_ctx* c, AlnTable& t) {
    CU(c->aln_flag.ensure(64));
    uint32_t* flag = c->aln_flag.as<uint32_t>();
    CU(cudaMemsetAsync(flag, 0, 4, c->stream));
    CU(cudaMemsetAsync(t.span.p, 0, ((size_t)c->n_contigs + 2) * 4, c->stream));
    LAUNCH(c, c->stream, k_aln_index, grid_for(c, t.n, 256), 256, 0, t.chrom.as<int32_t>(), t.start.as<int32_t>(), t.end.as<int32_t>(), t.n,
           c->n_contigs, t.span.as<int32_t>(), flag);
    LAUNCH(c, c->stream, k_aln_off, grid_for(c, (int64_t)c->n_contigs + 1, 256), 256, 0, t.chrom.as<int32_t>(), t.n, c->n_contigs, t.off.as<uint32_t>());
    uint32_t hflag = 0;
    CU(cudaMemcpyAsync(&hflag, flag, 4, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (hflag) {
        t.n = 0;
        return set_err(CSV_E_INPUT, "alignment table: %s", (hflag & ST_UNSORTED) ? "not coordinate-sorted (BAM order required)" : "contig id out of range");
    }
    return CSV_OK;
}

// The alignment table is copied on the ctx stream and its order is checked before the call returns (one synchronisation, for host
// and device columns alike), so a device source's buffers are free again on return.
static int upload_alignments_impl(csv_ctx* c, const csv_reads_cols* h, const UpSrc& src) {
    if (!c || !h) return set_err(CSV_E_INVALID, "bad argument");
    if (c->n_contigs == 0) return set_err(CSV_E_STATE, "csv_set_contigs has not been called");
    if (h->n < 0 || h->n >= (1ll << 31)) return set_err(CSV_E_INVALID, "alignment count out of range");
    CU(cudaSetDevice(c->device));
    AlnTable& A = c->aln;
    A.n = h->n;
    c->counts_valid = false;
    if (kind_scanned(c->ex.kind)) c->ex.kind = PacketKind::NAMED;   // the table no longer comes from a scanned accumulation
    c->ex.pending.n = 0;
    if (h->n == 0) return CSV_OK;
    if (!RowTable::has_cols(*h, true)) return set_err(CSV_E_INVALID, "null column");
    int rc;
    if (src.device && (rc = RowTable::check_dev(c, *h, true))) return rc;
    if ((rc = A.size(h->n)) || (rc = A.size_index(c->n_contigs))) return rc;
    CU(c->counters.ensure(sizeof(Counters)));
    if (src.device) {
        CU(cudaEventRecord(c->ev_prod, src.producer));
        CU(cudaStreamWaitEvent(c->stream, c->ev_prod, 0));
    }
    if ((rc = A.copy_in(*h, true, src.kind(), c->stream))) return rc;
    return aln_index(c, A);
}
extern "C" int csv_upload_alignments(csv_ctx* c, const csv_reads_cols* h) { return upload_alignments_impl(c, h, HOST_SRC); }
extern "C" int csv_upload_alignments_device(csv_ctx* c, const csv_reads_cols* d, void* stream) {
    return upload_alignments_impl(c, d, UpSrc{true, (cudaStream_t)stream});
}

// ------------------------------------------------------------------------------------------
// look-back sync objects
// ------------------------------------------------------------------------------------------
// One ticket word of the pool, zero at the start of the call (a TileSync's, or a counter of a kernel chain)
static int take_ticket(LbPool& lb, uint32_t** word) {
    if (lb.next >= lb.cap) return set_err(CSV_E_STATE, "look-back ticket pool exhausted");
    *word = lb.tickets + lb.next++;
    return CSV_OK;
}
// A TileSync over `status`, which must hold status_words words.  A status buffer that is too small grows, zero-filled, once
// the work enqueued on `s` (which may still use it) is done.
static int make_sync(LbPool& lb, DBuf& status, cudaStream_t s, size_t status_words, TileSync* ts) {
    if (lb.next >= lb.cap) return set_err(CSV_E_STATE, "look-back ticket pool exhausted");
    if (status.cap < status_words * 8) {
        CU(cudaStreamSynchronize(s));
        CU(status.ensure(status_words * 8, true));
    }
    ts->ordinal = lb.ord0 + (uint32_t)lb.next;
    ts->status = status.as<uint64_t>();
    ts->epoch = lb.epoch;
    return take_ticket(lb, &ts->ticket);
}

// ------------------------------------------------------------------------------------------
// radix sort driver: sorts (keys_a, vals_a) using (keys_b, vals_b) as the ping-pong partner, on stream s with the
// histogram buffer `hist` and look-back syncs from (lb, status).  iota: the payload of the first pass is the index.
// probe: each pass is a csv_sort_probe interval.  Outputs point at the final buffers.
// ------------------------------------------------------------------------------------------
template <typename K>
static int radix_sort(csv_ctx* c, cudaStream_t s, DBuf& hist, LbPool& lb, DBuf& status, bool probe, K* keys_a, uint32_t* vals_a,
                      K* keys_b, uint32_t* vals_b, bool iota, int64_t n, int bits, K** keys_out, uint32_t** vals_out) {
    const uint32_t* n_dev = nullptr;   // every sort's size is known on the host
    const int passes = std::max(1, (bits + 7) / 8);
    if (passes > RS_MAX_PASSES) return set_err(CSV_E_INVALID, "radix sort: %d bits", bits);
    constexpr int TILE = RS_THREADS * RsTraits<K>::ITEMS;
    const int64_t n_tiles = (n + TILE - 1) / TILE;
    CU(hist.ensure(RS_MAX_PASSES * 256 * 4));
    CU(cudaMemsetAsync(hist.p, 0, RS_MAX_PASSES * 256 * 4, s));
    LAUNCH(c, s, (k_rs_hist<K>), grid_for(c, n, RS_THREADS * 16, 4), RS_THREADS, 0, keys_a, n, n_dev, passes, hist.as<uint32_t>());
    LAUNCH(c, s, k_rs_hist_scan, 1, 256, 0, hist.as<uint32_t>(), passes);
    K* ki = keys_a; K* ko = keys_b;
    uint32_t* vi = vals_a; uint32_t* vo = vals_b;
    for (int p = 0; p < passes; p++) {
        TileSync ts;
        int rc = make_sync(lb, status, s, (size_t)n_tiles * 256, &ts);
        if (rc) return rc;
        const int64_t per_elem = (int64_t)(sizeof(K) + ((p == 0 && iota) ? 0 : 4) + sizeof(K) + 4);
        if (probe) stage_begin(c, s, ST_SORT_PASS, n * per_elem);
        if (p == 0 && iota)
            LAUNCH(c, s, (k_rs_onesweep<K, true>), (int)n_tiles, RS_THREADS, 0, ki, (const uint32_t*)nullptr, ko, vo, n, n_dev, 8 * p,
                   hist.as<uint32_t>() + p * 256, ts);
        else
            LAUNCH(c, s, (k_rs_onesweep<K, false>), (int)n_tiles, RS_THREADS, 0, ki, vi, ko, vo, n, n_dev, 8 * p,
                   hist.as<uint32_t>() + p * 256, ts);
        if (probe) stage_end(c, s, ST_SORT_PASS);
        std::swap(ki, ko);
        std::swap(vi, vo);
    }
    *keys_out = ki;
    *vals_out = vi;
    return CSV_OK;
}
// csv_cluster's sorts: on lane L's stream and buffers, with the call's shared ticket pool
template <typename K>
static int lane_sort(csv_ctx* c, Lane& L, bool iota, int64_t n, int bits, K** keys_out, uint32_t** vals_out) {
    return radix_sort<K>(c, L.stream, L.hist, c->lb, L.lb_status, true, L.keys_a.as<K>(), L.vals_a.as<uint32_t>(), L.keys_b.as<K>(),
                         L.vals_b.as<uint32_t>(), iota, n, bits, keys_out, vals_out);
}

// ------------------------------------------------------------------------------------------
// the pipeline
// ------------------------------------------------------------------------------------------
static ClusterParams cluster_params(const csv_params& P, int t) {
    ClusterParams C;
    C.min_support = P.min_support;
    C.min_support_allele = P.min_support_allele;
    C.min_size = P.min_size;
    C.max_size = P.max_size;
    C.bias = t == CSV_DEL ? P.bias_del : t == CSV_INS ? P.bias_ins : t == CSV_INV ? P.bias_inv : t == CSV_DUP ? P.bias_dup : P.bias_tra;
    C.ratio = t == CSV_DEL ? P.ratio_del : t == CSV_INS ? P.ratio_ins : P.ratio_tra;
    C.keep = P.remain_reads_ratio > 1 ? 1 : P.remain_reads_ratio;
    C.genotype = P.genotype;
    return C;
}

static Emit make_emit(csv_ctx* c) {
    Emit E;
    E.cand = c->cand_tmp.as<csv_cand>();
    E.names = c->names.as<int32_t>();
    E.cnt = c->cnt.as<uint32_t>();
    E.ctr = c->counters.as<Counters>();
    E.pow_half = c->pow_half.as<double>();
    E.lim.cap_cand = c->cap_cand;
    E.lim.cap_names = c->cap_names;
    E.lim.pow_n = c->pow_n;
    E.cursor = c->emit_cursor.as<unsigned long long>();
    return E;
}

static int run_segment_and_cluster(csv_ctx* c, Lane& L, TypeJob& J, int t, uint32_t kslot_base) {
    Counters* ctr = c->counters.as<Counters>();
    const cudaStream_t s = L.stream;
    // ---- segment: kept chain clusters, in order ----
    stage_begin(c, s, CSV_ST_SEGMENT);
    J.kslot_base = kslot_base;
    J.kept_start = c->kept[t].as<uint32_t>();
    J.big_list = L.big_list.as<uint32_t>();
    J.giant_list = L.giant_list.as<uint32_t>();
    J.giant_arena = L.giant_arena.as<char>();
    J.big_cap = (uint32_t)(L.big_list.cap / 4);
    J.giant_cap = (uint32_t)(L.giant_list.cap / 4);
    TileSync ts;
    int rc = make_sync(c->lb, L.lb_status, s, (size_t)(J.n_host / SEL_TILE + 2), &ts);
    if (rc) return rc;
    if ((J.cp.min_support + 31) / 32 + 1 <= HEAD_MAX_NEED_WORDS) {
        MemberRec MR;
        memset(&MR, 0, sizeof(MR));
        J.small_list = nullptr; J.n_small = nullptr; J.rest_list = nullptr; J.n_rest = nullptr; J.n_rest_lo = nullptr;
        if ((t == CSV_DEL || t == CSV_INS) && J.iv.rec) {
            MR.rec = const_cast<IndelRec*>(J.iv.rec); MR.recc = const_cast<int32_t*>(J.iv.recc);
            MR.a = J.iv.a; MR.b = J.iv.b; MR.rid = J.iv.rid; MR.c = J.iv.recc ? J.iv.c : nullptr; MR.sidx = J.iv.sidx;
            if (t == CSV_DEL && J.keys32) { MR.del_off = c->d_off.as<uint64_t>(); MR.n_contigs = c->n_contigs; }
            if (J.cp.keep >= 1.0 && J.small_path) {   // the walk also sorts the kept clusters into the two lists of the cluster kernels
                CU(L.rest_list.ensure((size_t)c->kept_cap[t] * 12 + 64));
                MR.rest_list = L.rest_list.as<uint32_t>();
                MR.small_list = (uint2*)(L.rest_list.as<uint32_t>() + c->kept_cap[t] + (c->kept_cap[t] & 1u));
                if ((rc = take_ticket(c->lb, &MR.n_small)) || (rc = take_ticket(c->lb, &MR.n_rest)) || (rc = take_ticket(c->lb, &MR.n_rest_lo)))
                    return rc;
                MR.rest_cap = c->kept_cap[t];
                J.small_list = MR.small_list; J.n_small = MR.n_small; J.rest_list = MR.rest_list; J.n_rest = MR.n_rest;
                J.n_rest_lo = MR.n_rest_lo; J.rest_cap = MR.rest_cap;
            }
        }
        // every CTA that fits at once: the tiles' look-backs and member gathers are latency chains, so a CTA that waits
        // should have others beside it (the survivors of the density filter are about a quarter of the bound n_host)
        const int sel_grid = std::min(grid_for(c, J.n_host, SEL_TILE, 64), resident_grid(c, k_select_heads, SEL_THREADS, 0));
        if (L.prev_is_chain_kernel)   // directly behind k_part_filter on this stream
            LAUNCH_PDL(c, s, k_select_heads, sel_grid, SEL_THREADS, 0, J, c->kept[t].as<uint32_t>(), c->kept_cap[t],
                       &ctr->n_kept[t], ts, &ctr->status, (uint32_t)ST_LIST_OVERFLOW, MR);
        else
            LAUNCH(c, s, k_select_heads, sel_grid, SEL_THREADS, 0, J, c->kept[t].as<uint32_t>(), c->kept_cap[t],
                   &ctr->n_kept[t], ts, &ctr->status, (uint32_t)ST_LIST_OVERFLOW, MR);
    } else {
        J.iv.rec = nullptr; J.iv.recc = nullptr;   // generic path: members are gathered by the cluster kernels
        HeadPred hp{J};
        LAUNCH(c, s, (k_select<HeadPred>), grid_for(c, J.n_host, SEL_TILE, 4), SEL_THREADS, 0, hp, J.n_host, J.n_dev,
               c->kept[t].as<uint32_t>(), c->kept_cap[t], &ctr->n_kept[t], ts, &ctr->status, (uint32_t)ST_LIST_OVERFLOW);
    }
    stage_end(c, s, CSV_ST_SEGMENT);
    // ---- cluster ----
    stage_begin(c, s, CSV_ST_CLUSTER);
    Emit E = make_emit(c);
    const size_t smem_warp = (size_t)(CL_THREADS / 32) * WARP_M * ARENA_PER_MAX + (CL_THREADS / 32) * 40 * 8;
    uint32_t* work = nullptr;   // zeroed per call
    if ((rc = take_ticket(c->lb, &work))) return rc;
    const bool keep_all = J.cp.keep >= 1.0;
    const int side_k = t == CSV_INS ? 1 : 0;
    cudaStream_t gs = s;   // the general kernels' stream: a side stream while the register kernel runs on the lane's own
    if (kind_of(t) == 0 && keep_all && J.small_path) {
        uint32_t* work_s = nullptr;
        if ((rc = take_ticket(c->lb, &work_s))) return rc;
        TypeJob JS = J;
        uint32_t* n_rest = nullptr;
        if (!J.small_list) {   // gather mode: the register kernel sizes the clusters itself and lists the larger ones
            CU(L.rest_list.ensure((size_t)c->kept_cap[t] * 12 + 64));
            if ((rc = take_ticket(c->lb, &n_rest))) return rc;
            JS.rest_list = L.rest_list.as<uint32_t>();
            JS.n_rest = n_rest;
        } else if (!c->profiling) {
            // both lists exist already: fork, the general kernels run beside the register kernel
            gs = c->side_stream[side_k];
            CU(cudaEventRecord(c->ev_side_fork[side_k], s));
            CU(cudaStreamWaitEvent(gs, c->ev_side_fork[side_k], 0));
        }
        if (t == CSV_INS) LAUNCH_PDL_NAMED(c, s, "k_cluster_small<INS>", (k_cluster_small<true>), c->n_sm * 6, 256, 0, JS, E, ctr, work_s, n_rest);
        else LAUNCH_PDL_NAMED(c, s, "k_cluster_small<DEL>", (k_cluster_small<false>), c->n_sm * 6, 256, 0, JS, E, ctr, work_s, n_rest);
        if (!J.small_list) { J.rest_list = JS.rest_list; J.n_rest = n_rest; }
    } else { J.small_list = nullptr; J.n_small = nullptr; J.rest_list = nullptr; J.n_rest = nullptr; J.n_rest_lo = nullptr; }
    switch (kind_of(t)) {   // one per-type routine per kernel instantiation (instruction-cache footprint)
        case 0:
            if (t == CSV_DEL) { if (keep_all) launch_cluster_kind<6, 0>(c, gs, J, E, ctr, work, smem_warp); else launch_cluster_kind<4, 0>(c, gs, J, E, ctr, work, smem_warp); }
            else { if (keep_all) launch_cluster_kind<7, 0>(c, gs, J, E, ctr, work, smem_warp); else launch_cluster_kind<5, 0>(c, gs, J, E, ctr, work, smem_warp); }
            break;
        case 1: launch_cluster_kind<1, 1>(c, gs, J, E, ctr, work, smem_warp); break;
        case 2: launch_cluster_kind<2, 2>(c, gs, J, E, ctr, work, smem_warp); break;
        default: launch_cluster_kind<3, 3>(c, gs, J, E, ctr, work, smem_warp); break;
    }
    if (gs != s) {
        CU(cudaEventRecord(c->ev_side_join[side_k], gs));
        CU(cudaStreamWaitEvent(s, c->ev_side_join[side_k], 0));
    }
    stage_end(c, s, CSV_ST_CLUSTER);
    if (L.mark >= 0) { CU(cudaEventRecord(c->kivs[L.mark].b, s)); L.mark = -1; }
    return CSV_OK;
}

static int run_indel(csv_ctx* c, Lane& L, int t, uint32_t kslot_base) {
    SigTable& s = c->sig[t];
    const cudaStream_t st = L.stream;
    const int64_t n = s.n;
    const uint64_t total = c->contig_off[c->n_contigs];
    const int bits = bits_for(total);
    const bool k64 = bits > 32;
    ContigTab ct{c->d_off.as<uint64_t>(), c->d_len_eff.as<int64_t>(), c->n_contigs};
    Counters* ctr = c->counters.as<Counters>();
    TypeJob J;
    memset(&J, 0, sizeof(J));
    J.svtype = t; J.n_host = n; J.n_dev = nullptr;
    J.cp = cluster_params(c->P, t);
    // density pre-filter: worthwhile when the expected neighbourhood count is below min_support
    const uint32_t radius = (uint32_t)std::min<int64_t>((int64_t)(J.cp.min_support - 1) * J.cp.bias, 1 << 24);
    const double lambda = (double)n * (2.0 * radius + 2.0 * (1 << BKT_SHIFT)) / (double)std::max<uint64_t>(total, 1);
    const int rb = (int)((radius + (1u << BKT_SHIFT) - 1) >> BKT_SHIFT);  // neighbourhood radius in buckets (conservative)
    const bool prefilter = !k64 && c->prefilter_enabled && J.cp.min_support >= 3 && lambda < 0.8 * J.cp.min_support &&
                           n >= (1 << 16) && rb <= BKT_PAD;
    J.iv.rec = nullptr; J.iv.recc = nullptr;
    uint32_t* sidx = nullptr;
    int rc;
    if (prefilter) {
        // filter-first front end, partitioned by genome range: scatter of (key, index) by partition into each partition's
        // pages of a pool -> per partition, in shared memory, over its pages: bucket histogram, density flags, survivors in
        // key order.  W: the widest partitions (at most 2^22 bp) that still give every SM about two of them.
        int W = PART_W_MAX;
        while (W > PART_W_MIN && (int64_t)(total >> W) + 1 < 2 * (int64_t)c->n_sm) W--;
        const int P = (int)(total >> W) + 1;
        const int n_chunks = (int)((n + PART_ROUND - 1) / PART_ROUND);
        const uint32_t ptw = (uint32_t)((n + PART_PAGE - 1) / PART_PAGE) + 1;   // page-table row: every page of n pairs, + 1
        // edge counts at a fixed size in front, so that the fill counters and page table behind them, all zero between
        // calls, stay zero whatever P and n the next call has
        const size_t edge_words = (size_t)PART_MAX * 2 * BKT_PAD, tab_words = PART_MAX + (size_t)P * ptw;
        stage_begin(c, st, CSV_ST_KEYS);
        CU(L.boff.ensure((edge_words + tab_words) * 4, true));   // edges | fill[PART_MAX] | pt[P][ptw]
        uint32_t* edge = L.boff.as<uint32_t>();
        uint32_t* fill = edge + edge_words;
        uint32_t* pt = fill + PART_MAX;
        CU(L.keys_a.ensure(((size_t)ptw - 1 + P) * PART_PAGE * 8));   // the page pool
        uint2* pool = (uint2*)L.keys_a.p;
        // the spill area of partitions whose survivors exceed the shared-memory stage; the member records use it later
        CU(L.rec_a.ensure((size_t)n * sizeof(IndelRec)));
        CU(cudaMemsetAsync(edge, 0, (size_t)P * 2 * BKT_PAD * 4, st));
        const int is_ins = t == CSV_INS ? 1 : 0;
        if ((((uintptr_t)s.chrom.p) | ((uintptr_t)s.a.p)) & 15)   // k_part_scatter loads both columns 16 B at a time
            return set_err(CSV_E_STATE, "signature columns are not 16 B aligned");
        // Everything that can fail on the host is done before the scatter: once it is enqueued, its filter is enqueued
        // right behind it, and the filter resets the fill counters and page-table entries the scatter set.
        uint32_t* pool_next = nullptr;   // zeroed by k_begin
        TileSync ts;
        if ((rc = take_ticket(c->lb, &pool_next)) || (rc = make_sync(c->lb, L.lb_status, st, (size_t)P, &ts))) return rc;
        const size_t smem = pf_smem_bytes(W);
        const int g = std::min(P, resident_grid(c, k_part_filter, PF_THREADS, smem));
        LAUNCH(c, st, k_part_scatter, n_chunks, PS_THREADS, ps_smem_bytes(), s.chrom.as<int32_t>(), s.a.as<int32_t>(), n, is_ins, ct, W, P,
               rb, pool, fill, pt, ptw, pool_next, edge, &ctr->status);
        stage_end(c, st, CSV_ST_KEYS);
        stage_begin(c, st, CSV_ST_SORT);
        uint32_t* n_pass = &ctr->n_dom[t];
        LAUNCH_PDL(c, st, k_part_filter, g, PF_THREADS, smem, (const uint2*)pool, fill, pt, ptw, P, W, rb, (uint32_t)J.cp.min_support,
                   (const uint32_t*)edge, L.keys_b.as<uint32_t>(), L.vals_b.as<uint32_t>(), (uint2*)L.rec_a.p, n_pass, ts);
        stage_end(c, st, CSV_ST_SORT);
        if (c->lane_marks) {
            kprof_begin(c, st, t == CSV_DEL ? "back end<DEL>" : "back end<INS>");
            L.mark = (int)c->kivs.size() - 1;
        }
        J.n_dev = n_pass;
        J.keys32 = L.keys_b.as<uint32_t>();
        sidx = L.vals_b.as<uint32_t>();
    } else {
        stage_begin(c, st, CSV_ST_KEYS);
        if (!k64)
            LAUNCH(c, st, (k_indel_keys<uint32_t>), grid_for(c, n, 256), 256, 0, s.chrom.as<int32_t>(), s.a.as<int32_t>(), s.b.as<int32_t>(),
                   s.rid.as<int32_t>(), n, t == CSV_INS ? 1 : 0, ct, L.keys_a.as<uint32_t>(), &ctr->status);
        else
            LAUNCH(c, st, (k_indel_keys<uint64_t>), grid_for(c, n, 256), 256, 0, s.chrom.as<int32_t>(), s.a.as<int32_t>(), s.b.as<int32_t>(),
                   s.rid.as<int32_t>(), n, t == CSV_INS ? 1 : 0, ct, L.keys_a.as<uint64_t>(), &ctr->status);
        stage_end(c, st, CSV_ST_KEYS);
        stage_begin(c, st, CSV_ST_SORT);
        if (!k64) {
            uint32_t* ko = nullptr;
            rc = lane_sort<uint32_t>(c, L, true, n, bits, &ko, &sidx);
            J.keys32 = ko;
        } else {
            uint64_t* ko = nullptr;
            rc = lane_sort<uint64_t>(c, L, true, n, bits, &ko, &sidx);
            J.keys64 = ko;
        }
        if (rc) return rc;
        stage_end(c, st, CSV_ST_SORT);
    }
    J.iv.chrom = s.chrom.as<int32_t>(); J.iv.a = s.a.as<int32_t>(); J.iv.b = s.b.as<int32_t>(); J.iv.rid = s.rid.as<int32_t>();
    J.iv.c = s.has_c ? s.c.as<int32_t>() : nullptr;
    J.iv.sidx = sidx;
    if (!k64 && c->records_enabled && (J.cp.min_support + 31) / 32 + 1 <= HEAD_MAX_NEED_WORDS) {
        // record mode: k_select_heads gathers one contiguous 16 B record (+ c of INS) per member of a kept chain cluster
        const bool with_c = t == CSV_INS && s.has_c;
        CU(L.rec_a.ensure((size_t)n * sizeof(IndelRec)));
        if (with_c) CU(L.recc_a.ensure((size_t)n * 4));
        J.iv.rec = L.rec_a.as<IndelRec>();
        J.iv.recc = with_c ? L.recc_a.as<int32_t>() : nullptr;
    }
    J.iv.is_ins = t == CSV_INS ? 1 : 0;
    J.small_path = c->small_path_enabled ? 1 : 0;
    L.prev_is_chain_kernel = prefilter;
    rc = run_segment_and_cluster(c, L, J, t, kslot_base);
    L.prev_is_chain_kernel = false;
    return rc;
}

static int run_other(csv_ctx* c, Lane& L, int t, uint32_t kslot_base) {
    SigTable& s = c->sig[t];
    const cudaStream_t st = L.stream;
    const int64_t n = s.n;
    SmallWork& w = L.small;
    ContigTab ct{c->d_off.as<uint64_t>(), c->d_len_eff.as<int64_t>(), c->n_contigs};
    Counters* ctr = c->counters.as<Counters>();
    // primary key = (chr, a) | (chr, strand, a) | (chr1, chr2*4+type, a): value range sized from the contig count
    const uint64_t hi_max = t == CSV_DUP ? (uint64_t)c->n_contigs : t == CSV_INV ? 2ull * c->n_contigs : 4ull * c->n_contigs * c->n_contigs;
    // The packed TRA key needs 2*ceil(log2 n_contigs) + 33 bits.  On more than 32768 contigs (chr1, chr2*4+type) is
    // replaced by its dense rank among the pairs present, which is below the signature count, so the key stays (rank, a)
    // in 31 + bits_for(n) bits
    const int clog = c->n_contigs > 1 ? bits_for((uint64_t)c->n_contigs - 1) : 0;   // ceil(log2 n_contigs)
    const bool compact = t == CSV_TRA && 2 * clog + 33 > 64;
    const int prim_bits = 31 + bits_for(compact ? (uint64_t)n : hi_max);
    const int32_t* col_c = s.has_c ? s.c.as<int32_t>() : nullptr;
    const bool chain = c->small_chain[t];
    uint64_t* k_prim = chain ? w.k_prim.as<uint64_t>() : L.keys_a.as<uint64_t>();
    int rc;
    stage_begin(c, st, CSV_ST_KEYS);
    if (!compact) {
        LAUNCH(c, st, (k_other_keys<false>), grid_for(c, n, 256), 256, 0, s.chrom.as<int32_t>(), s.a.as<int32_t>(), s.b.as<int32_t>(),
               s.rid.as<int32_t>(), col_c, n, t, ct, chain ? w.k_rid.as<uint32_t>() : (uint32_t*)nullptr, w.k_b.as<uint32_t>(), k_prim,
               &ctr->status);
    } else {
        // pair words -> sort -> flags at pair changes -> exclusive scan = ranks -> (rank, a) scattered back to input order
        LAUNCH(c, st, (k_other_keys<true>), grid_for(c, n, 256), 256, 0, s.chrom.as<int32_t>(), s.a.as<int32_t>(), s.b.as<int32_t>(),
               s.rid.as<int32_t>(), col_c, n, t, ct, chain ? w.k_rid.as<uint32_t>() : (uint32_t*)nullptr, w.k_b.as<uint32_t>(),
               L.keys_a.as<uint64_t>(), &ctr->status);
        uint64_t* pair_sorted = nullptr;
        uint32_t* pair_perm = nullptr;
        rc = lane_sort<uint64_t>(c, L, true, n, bits_for(hi_max), &pair_sorted, &pair_perm);
        if (rc) return rc;
        uint32_t* rank = w.sel.as<uint32_t>();   // free until the de-duplication below
        LAUNCH(c, st, k_tra_pair_flags, grid_for(c, n, 256), 256, 0, (const uint64_t*)pair_sorted, n, rank);
        TileSync ts;
        rc = make_sync(c->lb, L.lb_status, st, (size_t)(n / (SEL_THREADS * 4) + 2), &ts);
        if (rc) return rc;
        LAUNCH(c, st, (k_scan_excl<4>), grid_for(c, n, SEL_THREADS * 4, 4), SEL_THREADS, 0, rank, n, (const uint32_t*)nullptr,
               (const uint32_t*)nullptr, (uint32_t*)nullptr, ts);
        // k_prim may alias pair_sorted (keys_a), which is no longer read; pair_perm is a value buffer
        LAUNCH(c, st, k_tra_compact_key, grid_for(c, n, 256), 256, 0, (const uint32_t*)pair_perm, (const uint32_t*)rank, s.a.as<int32_t>(), n,
               k_prim);
    }
    stage_end(c, st, CSV_ST_KEYS);
    stage_begin(c, st, CSV_ST_SORT);
    if (!chain) {
        // ONE sort on the primary key (<= 8 passes instead of 16), then (b, name) order inside runs of equal primary keys
        uint64_t* k64o = nullptr;
        uint32_t* perm = nullptr;
        rc = lane_sort<uint64_t>(c, L, true, n, prim_bits, &k64o, &perm);
        if (rc) return rc;
        LAUNCH(c, st, k_run_fixup, grid_for(c, n, 256), 256, 0, k64o, perm, n, s.b.as<int32_t>(), s.rid.as<int32_t>(), w.perm_b.as<uint32_t>(),
               &ctr->status);
    } else {
        // LSD over the fields of the reference's tuple sort key: name, then second coordinate, then primary
        // (fallback after ST_BIG_RUN: a run of equal primary keys too long for the ranking kernel)
        uint32_t *k32o = nullptr, *perm = nullptr;
        LAUNCH(c, st, (k_gather_keys<uint32_t>), grid_for(c, n, 256), 256, 0, w.k_rid.as<uint32_t>(), (const uint32_t*)nullptr, n, L.keys_a.as<uint32_t>());
        rc = lane_sort<uint32_t>(c, L, true, n, 31, &k32o, &perm);
        if (rc) return rc;
        CU(cudaMemcpyAsync(w.perm_a.p, perm, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
        LAUNCH(c, st, (k_gather_keys<uint32_t>), grid_for(c, n, 256), 256, 0, w.k_b.as<uint32_t>(), w.perm_a.as<uint32_t>(), n, L.keys_a.as<uint32_t>());
        CU(cudaMemcpyAsync(L.vals_a.p, w.perm_a.p, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
        rc = lane_sort<uint32_t>(c, L, false, n, 31, &k32o, &perm);
        if (rc) return rc;
        CU(cudaMemcpyAsync(w.perm_a.p, perm, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
        LAUNCH(c, st, (k_gather_keys<uint64_t>), grid_for(c, n, 256), 256, 0, w.k_prim.as<uint64_t>(), w.perm_a.as<uint32_t>(), n, L.keys_a.as<uint64_t>());
        CU(cudaMemcpyAsync(L.vals_a.p, w.perm_a.p, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
        uint64_t* k64o = nullptr;
        rc = lane_sort<uint64_t>(c, L, false, n, prim_bits, &k64o, &perm);
        if (rc) return rc;
        CU(cudaMemcpyAsync(w.perm_b.p, perm, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
    }
    stage_end(c, st, CSV_ST_SORT);
    // exact-duplicate removal + materialise the sorted columns
    stage_begin(c, st, CSV_ST_SEGMENT);
    uint32_t* n_u = &ctr->n_dom[t];  // device-side size of the de-duplicated domain
    TileSync ts;
    rc = make_sync(c->lb, L.lb_status, st, (size_t)(n / SEL_TILE + 2), &ts);
    if (rc) return rc;
    DedupPred dp{s.chrom.as<int32_t>(), s.a.as<int32_t>(), s.b.as<int32_t>(), s.rid.as<int32_t>(), col_c, w.perm_b.as<uint32_t>()};
    LAUNCH(c, st, (k_select<DedupPred>), grid_for(c, n, SEL_TILE, 4), SEL_THREADS, 0, dp, n, (const uint32_t*)nullptr, w.sel.as<uint32_t>(),
           (uint32_t)n, n_u, ts, &ctr->status, (uint32_t)ST_INTERNAL);
    LAUNCH(c, st, k_other_gather, grid_for(c, n, 256), 256, 0, s.chrom.as<int32_t>(), s.a.as<int32_t>(), s.b.as<int32_t>(), s.rid.as<int32_t>(),
           col_c, w.perm_b.as<uint32_t>(), w.sel.as<uint32_t>(), n_u, w.u_chrom.as<int32_t>(), w.u_a.as<int32_t>(), w.u_b.as<int32_t>(),
           w.u_rid.as<int32_t>(), w.u_c.as<int32_t>());
    stage_end(c, st, CSV_ST_SEGMENT);
    TypeJob J;
    memset(&J, 0, sizeof(J));
    J.svtype = t; J.n_host = n; J.n_dev = n_u;
    J.cp = cluster_params(c->P, t);
    J.sv.chrom = w.u_chrom.as<int32_t>(); J.sv.a = w.u_a.as<int32_t>(); J.sv.b = w.u_b.as<int32_t>();
    J.sv.rid = w.u_rid.as<int32_t>(); J.sv.c = w.u_c.as<int32_t>();
    return run_segment_and_cluster(c, L, J, t, kslot_base);
}

// lane L's DUP / INV / TRA scratch, for chains over at most ns signatures
static int ensure_small(Lane& L, size_t ns) {
    SmallWork& w = L.small;
    CU(w.k_rid.ensure(ns * 4)); CU(w.k_b.ensure(ns * 4)); CU(w.k_prim.ensure(ns * 8)); CU(w.perm_a.ensure(ns * 4)); CU(w.perm_b.ensure(ns * 4));
    CU(w.sel.ensure(ns * 4)); CU(w.u_chrom.ensure(ns * 4)); CU(w.u_a.ensure(ns * 4)); CU(w.u_b.ensure(ns * 4)); CU(w.u_rid.ensure(ns * 4));
    CU(w.u_c.ensure(ns * 4));
    return CSV_OK;
}
// lane L's sort and cluster scratch, for chains over at most nm signatures
static int ensure_lane_scratch(Lane& L, size_t nm) {
    CU(L.keys_a.ensure(nm * 8)); CU(L.keys_b.ensure(nm * 8)); CU(L.vals_a.ensure(nm * 4)); CU(L.vals_b.ensure(nm * 4));
    CU(L.big_list.ensure((nm / WARP_M + 2) * 4));
    CU(L.giant_list.ensure((nm / BLOCK_M + 2) * 4));
    CU(L.giant_arena.ensure(nm * 2 * ARENA_PER_MAX + 256));
    return CSV_OK;
}

static int ensure_workspace(csv_ctx* c, uint32_t type_mask) {
    int64_t n_max = 0, n_total = 0, n_small_max = 0;
    for (int t = 0; t < CSV_NTYPES; t++) {
        if (!(type_mask >> t & 1)) continue;
        n_max = std::max(n_max, c->sig[t].n);
        n_total += c->sig[t].n;
        if (t >= CSV_INV) n_small_max = std::max(n_small_max, c->sig[t].n);
    }
    const size_t nm = (size_t)std::max<int64_t>(n_max, 1);
    int rc = ensure_lane_scratch(c->lanes[0], nm);   // lane 0 can run every type (lanes disabled)
    if (rc) return rc;
    if (c->lanes_enabled) {
        for (int t = 1; t < CSV_NTYPES; t++) {   // lane t runs type t
            const int64_t nl = (type_mask >> t & 1) ? c->sig[t].n : 0;
            if (nl == 0) continue;
            if ((rc = ensure_lane_scratch(c->lanes[t], (size_t)nl))) return rc;
            if (t >= CSV_INV && (rc = ensure_small(c->lanes[t], (size_t)nl))) return rc;
        }
    }
    CU(c->tickets.ensure(LB_ORDINALS * 4));
    CU(c->counters.ensure(sizeof(Counters)));
    if ((rc = ensure_small(c->lanes[0], (size_t)std::max<int64_t>(n_small_max, 1)))) return rc;
    uint64_t kept_total = 0;
    const int ms = std::max(1, c->P.min_support);
    for (int t = 0; t < CSV_NTYPES; t++) {
        if (!(type_mask >> t & 1)) continue;
        c->kept_cap[t] = (uint32_t)(c->sig[t].n / ms + 1);
        CU(c->kept[t].ensure((size_t)c->kept_cap[t] * 4));
        kept_total += c->kept_cap[t];
    }
    CU(c->cnt.ensure((size_t)kept_total * 4 + 4));
    const int ms_a = std::max(1, std::min(c->P.min_support, std::max(1, c->P.min_support_allele)));
    c->cap_cand = (uint32_t)(2 * (n_total / ms_a) + 16);  // TRA can emit two rows per chain cluster (resolveTRA.py:133-209)
    c->cap_names = (uint32_t)(n_total + 16);
    CU(c->cand_tmp.ensure((size_t)c->cap_cand * sizeof(csv_cand)));
    CU(c->cand.ensure((size_t)c->cap_cand * sizeof(csv_cand)));
    CU(c->geno.ensure((size_t)c->cap_cand * sizeof(csv_geno)));
    CU(c->names.ensure((size_t)c->cap_names * 4));
    CU(c->dr.ensure((size_t)c->cap_cand * 4));
    CU(c->win_list.ensure((size_t)c->cap_cand * 2 * 4));
    CU(c->win_rec.ensure((size_t)c->cap_cand * 2 * sizeof(WinRec)));
    CU(c->has_rows.ensure((size_t)c->n_contigs + 16));
    return CSV_OK;
}

static int join_lanes(csv_ctx* c) {
    for (int l = 1; l < N_LANES; l++) {
        Lane& L = c->lanes[l];
        if (!L.used) continue;
        CU(cudaEventRecord(L.ev_join, L.stream));
        CU(cudaStreamWaitEvent(c->stream, L.ev_join, 0));
        L.used = false;
    }
    return CSV_OK;
}

// Enqueues the whole kernel chain of one csv_cluster call (all lanes).  Pure enqueue when every buffer already has
// its size: that is what csv_cluster() captures into a CUDA graph.
static int enqueue_cluster(csv_ctx* c, uint32_t type_mask) {
    int rc;
    stage_reset_if_consumed(c);
    c->last_mask = type_mask;
    c->lb = LbPool{c->tickets.as<uint32_t>(), c->d_epoch.as<uint32_t>(), 0, 0, (int)LB_ORDINALS};   // k_begin zeroes the tickets
    {
        int n_lanes = 0;
        for (int t = 0; t < CSV_NTYPES; t++) n_lanes += ((type_mask >> t & 1) && c->sig[t].n > 0) ? 1 : 0;
        c->pdl_now = c->pdl_enabled && n_lanes <= 2;
    }
    // fresh look-back generation, zeroed tickets and counters.  (The per-cluster row counts `cnt` need no clearing: every
    // kept-cluster slot below n_kept[t] is written by a cluster kernel and the order scans stop at n_kept[t].)
    LAUNCH(c, c->stream, k_begin, 1, 256, 0, c->d_epoch.as<uint32_t>(), c->tickets.as<uint32_t>(), (int)LB_ORDINALS, c->counters.as<uint32_t>(),
           (int)(sizeof(Counters) / 4), c->emit_cursor.as<unsigned long long>());
    Counters* ctr = c->counters.as<Counters>();
    uint32_t kslot_base = 0;
    // fork: every lane's chain starts after the resets above; join before `order`
    const bool lanes = c->lanes_enabled;
    if (lanes) CU(cudaEventRecord(c->ev_fork, c->stream));
    for (Lane& L : c->lanes) L.used = false;
    // genotype-stage scratch (bin tables of the linear coordinate): sized and cleared now, beside the lanes
    const uint64_t total_len = c->contig_off[c->n_contigs];
    int geno_shift = 10;
    while ((total_len >> geno_shift) > (1u << 20)) geno_shift++;
    const uint32_t geno_bins = (uint32_t)(total_len >> geno_shift) + 2;
    bool aux_used = false;
    if (c->P.genotype) {
        CU(c->bin_start.ensure(((size_t)geno_bins + 1) * 4));
        CU(c->bin_fill.ensure((size_t)geno_bins * 4));
        CU(c->bin_bits.ensure(((size_t)geno_bins / 32 + 2) * 4));
        cudaStream_t rs = lanes ? c->aux_stream : c->stream;
        if (lanes) CU(cudaStreamWaitEvent(rs, c->ev_fork, 0));
        CU(cudaMemsetAsync(c->bin_start.p, 0, ((size_t)geno_bins + 1) * 4, rs));
        CU(cudaMemsetAsync(c->bin_fill.p, 0, (size_t)geno_bins * 4, rs));
        CU(cudaMemsetAsync(c->bin_bits.p, 0, ((size_t)geno_bins / 32 + 2) * 4, rs));
        CU(cudaMemsetAsync(c->has_rows.p, 0, (size_t)c->n_contigs, rs));
        if (lanes) { CU(cudaEventRecord(c->ev_aux, rs)); aux_used = true; }
    }
    for (int t = 0; t < CSV_NTYPES; t++) {
        if (!(type_mask >> t & 1) || c->sig[t].n == 0) continue;
        Lane& L = c->lanes[lanes ? t : 0];
        if (&L != &c->lanes[0] && !L.used) { CU(cudaStreamWaitEvent(L.stream, c->ev_fork, 0)); L.used = true; }
        rc = wait_upload(c, L.stream, t);
        if (!rc && c->up[t].checked) LAUNCH(c, L.stream, k_fold_status, 1, 32, 0, c->up_status.as<uint32_t>() + t, &ctr->status);
        if (!rc) rc = (t == CSV_DEL || t == CSV_INS) ? run_indel(c, L, t, kslot_base) : run_other(c, L, t, kslot_base);
        if (rc) {   // the ctx stream must not run ahead of work already forked
            join_lanes(c);
            if (aux_used) cudaStreamWaitEvent(c->stream, c->ev_aux, 0);
            return rc;
        }
        kslot_base += c->kept_cap[t];
    }
    rc = join_lanes(c);
    if (rc) return rc;
    if (aux_used) CU(cudaStreamWaitEvent(c->stream, c->ev_aux, 0));
    int tail_mark = -1;   // lane_marks: the serial tail, from the lane join to the end of the call's chain
    if (c->lane_marks) { kprof_begin(c, c->stream, "tail"); tail_mark = (int)c->kivs.size() - 1; }
    GenoJob G;
    memset(&G, 0, sizeof(G));
    G.cand = c->cand.as<csv_cand>(); G.geno = c->geno.as<csv_geno>(); G.names = c->names.as<int32_t>(); G.ctr = ctr;
    G.cap_cand = c->cap_cand;
    G.ct = ContigTab{c->d_off.as<uint64_t>(), c->d_len_eff.as<int64_t>(), c->n_contigs};
    G.gp = GtParams{c->P.bias_del, c->P.gt_bias_ins, c->P.bias_dup, c->P.bias_inv};
    G.shift = geno_shift;
    G.n_bins = geno_bins;
    G.bin_start = c->bin_start.as<uint32_t>(); G.bin_fill = c->bin_fill.as<uint32_t>(); G.bin_bits = c->bin_bits.as<uint32_t>();
    G.win_list = c->win_list.as<uint32_t>(); G.win_cap = c->cap_cand * 2;
    G.lin32 = (total_len + 4096) < (1ull << 32) ? 1 : 0;   // (window ends may pass the last contig by a bias)
    G.win_rec = c->win_rec.as<WinRec>();
    G.dr = c->dr.as<uint32_t>(); G.has_rows = c->has_rows.as<uint8_t>();
    G.gl_table = c->gl_table.as<csv_geno>();
    G.genotype = c->P.genotype;
    // ---- order ----
    stage_begin(c, c->stream, CSV_ST_ORDER);
    {
        // exclusive scan of the per-cluster row counts, one short scan per SV type over the slots actually used
        // (n_kept[t] of kept_cap[t]), chained through a carry word
        CU(c->scan_carry.ensure(64));
        uint32_t* carry = c->scan_carry.as<uint32_t>();
        uint32_t kb = 0;
        int prev = -1;
        for (int t = 0; t < CSV_NTYPES; t++) {
            if (!(type_mask >> t & 1) || c->sig[t].n == 0) continue;
            TileSync ts;
            rc = make_sync(c->lb, c->lanes[0].lb_status, c->stream, (size_t)(c->kept_cap[t] / SEL_TILE + 2), &ts);
            if (rc) return rc;
            if (prev >= 0)
                LAUNCH_PDL(c, c->stream, (k_scan_excl<8>), grid_for(c, std::max<int64_t>(c->kept_cap[t], 1), SEL_TILE, 2), SEL_THREADS, 0, c->cnt.as<uint32_t>() + kb,
                           (int64_t)c->kept_cap[t], (const uint32_t*)&ctr->n_kept[t], (const uint32_t*)(carry + prev), carry + t, ts);
            else
                LAUNCH(c, c->stream, (k_scan_excl<8>), grid_for(c, std::max<int64_t>(c->kept_cap[t], 1), SEL_TILE, 2), SEL_THREADS, 0, c->cnt.as<uint32_t>() + kb,
                       (int64_t)c->kept_cap[t], (const uint32_t*)&ctr->n_kept[t], (const uint32_t*)nullptr, carry + t, ts);
            kb += c->kept_cap[t];
            prev = t;
        }
        // final order; the same pass counts the genotype windows per bin
        LAUNCH_PDL(c, c->stream, k_permute, grid_for(c, c->cap_cand, 256, 4), 256, 0, c->cand_tmp.as<csv_cand>(), c->cnt.as<uint32_t>(), ctr, c->cap_cand,
               c->cand.as<csv_cand>(), G, c->emit_cursor.as<unsigned long long>());
    }
    stage_end(c, c->stream, CSV_ST_ORDER);
    // ---- genotype ----
    rc = wait_upload(c, c->stream, CSV_NTYPES);
    if (rc) return rc;
    if (c->up[CSV_NTYPES].checked && c->reads.n > 0)
        LAUNCH(c, c->stream, k_fold_status, 1, 32, 0, c->up_status.as<uint32_t>() + CSV_NTYPES, &ctr->status);
    stage_begin(c, c->stream, CSV_ST_GENOTYPE);
    {
        if (c->P.genotype) {
            TileSync ts;
            // 1024-bin tiles, one 128-bit access per thread: the scan of the (at most 2^20 + 2) bins is a latency chain,
            // many small tiles on all SMs finish it sooner than few wide ones
            rc = make_sync(c->lb, c->lanes[0].lb_status, c->stream, (size_t)((G.n_bins + 1) / (SEL_THREADS * 4) + 2), &ts);
            if (rc) return rc;
            LAUNCH_PDL(c, c->stream, (k_scan_excl<4>), grid_for(c, G.n_bins + 1, SEL_THREADS * 4, 4), SEL_THREADS, 0, G.bin_start, (int64_t)G.n_bins + 1,
                   (const uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, ts);
            LAUNCH_PDL(c, c->stream, (k_windows<1>), grid_for(c, c->cap_cand, 256, 4), 256, 0, G);
            if (c->reads.n > 0) {
                const GcReads R = c->reads.gc_reads();
                PairBuf PB;
                PB.cap = (uint32_t)std::min<int64_t>(4 * R.n + (1 << 20), (int64_t)1 << 30);
                if (c->pair_cap_override > 0) PB.cap = (uint32_t)c->pair_cap_override;  // tests: force the overflow path
                CU(c->pairs.ensure((size_t)PB.cap * (G.lin32 ? sizeof(uint4) : sizeof(uint2))));
                PB.pairs = c->pairs.as<uint2>();
                PB.pairs4 = c->pairs.as<uint4>();
                PB.count = &ctr->n_windows;
                if (G.lin32) {
                    LAUNCH_PDL(c, c->stream, (k_reads_pass<true>), std::min(grid_for(c, R.n, 1024, 8), resident_grid(c, k_reads_pass<true>, 256, 0)), 256, 0, G, PB,
                               R.chrom, R.start, R.end, R.rid, R.prim, R.n, &ctr->status);
                    LAUNCH_PDL(c, c->stream, (k_pairs_test<true>), c->n_sm * 8, 256, 0, G, PB, R.chrom, R.start, R.end, R.rid);
                } else {
                    LAUNCH_PDL(c, c->stream, (k_reads_pass<false>), std::min(grid_for(c, R.n, 1024, 8), resident_grid(c, k_reads_pass<false>, 256, 0)), 256, 0, G, PB,
                               R.chrom, R.start, R.end, R.rid, R.prim, R.n, &ctr->status);
                    LAUNCH_PDL(c, c->stream, (k_pairs_test<false>), c->n_sm * 8, 256, 0, G, PB, R.chrom, R.start, R.end, R.rid);
                }
            }
        }
        LAUNCH_PDL(c, c->stream, k_finalize, grid_for(c, c->cap_cand, 256, 4), 256, 0, G);
        if (c->P.genotype && c->aln.n > 0 && (type_mask >> CSV_TRA & 1) && c->sig[CSV_TRA].n > 0) {
            const AlnView A = c->aln.view(c->d_len.as<int64_t>());
            LAUNCH(c, c->stream, k_tra_genotype, c->n_sm * 8, 128, 0, G, A, c->P.bias_tra, c->P.gt_round);   // 4 warps per CTA, one warp per TRA candidate
        }
    }
    stage_end(c, c->stream, CSV_ST_GENOTYPE);
    if (tail_mark >= 0) CU(cudaEventRecord(c->kivs[tail_mark].b, c->stream));
    return CSV_OK;
}

static bool key_equal(const csv_ctx::GraphKey& a, const csv_ctx::GraphKey& b) { return memcmp(&a, &b, sizeof(a)) == 0; }

extern "C" int csv_cluster(csv_ctx* c, uint32_t type_mask) {
    if (!c) return set_err(CSV_E_INVALID, "null ctx");
    if (c->n_contigs == 0) return set_err(CSV_E_STATE, "csv_set_contigs has not been called");
    CU(cudaSetDevice(c->device));
    int rc = ensure_workspace(c, type_mask);
    if (rc) return rc;
    c->gathered = false;
    // look-back generations are epoch * LB_ORDINALS + ordinal in 31 bits: start over before they could wrap
    if (++c->epoch_host >= LB_EPOCH_LIMIT) {
        CU(cudaDeviceSynchronize());
        CU(cudaMemset(c->d_epoch.p, 0, 64));
        for (Lane& L : c->lanes) if (L.lb_status.p) CU(cudaMemset(L.lb_status.p, 0, L.lb_status.cap));
        c->epoch_host = 1;
    }
    // A call whose inputs are already resident (no upload in flight) and that is not being profiled replays a
    // captured CUDA graph: first sighting of a key runs eagerly (buffers get their sizes), the second captures,
    // later ones replay -- ~40 launches on 6 streams become one cudaGraphLaunch.  Device-to-device uploads are waited for here,
    // before the chain (they take a fraction of the chain's time), so that a call on fresh device inputs still replays; host
    // uploads keep their per-type waits, which let the H2D copies of later types overlap the kernels of earlier ones.
    bool pending = false;
    for (int t = 0; t <= CSV_NTYPES; t++) {
        if (c->up[t].pending && c->up[t].device) { rc = wait_upload(c, c->stream, t); if (rc) return rc; }
        pending |= c->up[t].pending;
    }
    bool done = false;
    if (c->graphs_enabled && !c->profiling && !c->lane_marks && !pending) {
        csv_ctx::GraphKey key;
        memset(&key, 0, sizeof(key));
        key.mask = type_mask;
        for (int t = 0; t < CSV_NTYPES; t++) { key.n[t] = c->sig[t].n; key.small_chain[t] = c->small_chain[t]; }
        for (int t = 0; t <= CSV_NTYPES; t++) key.up_checked[t] = c->up[t].checked;
        key.n_reads = c->reads.n; key.n_aln = c->aln.n; key.P = c->P; key.lanes = c->lanes_enabled ? 1 : 0;
        key.alloc_epoch = g_alloc_epoch.load(); key.cfg_epoch = c->cfg_epoch;
        csv_ctx::GraphSlot* hit = nullptr;
        for (auto& g : c->graphs) if (g.valid && key_equal(g.key, key)) hit = &g;
        if (!hit && c->last_key_valid && key_equal(c->last_key, key)) {
            // second sighting: capture
            csv_ctx::GraphSlot* slot = &c->graphs[0];
            for (auto& g : c->graphs) { if (!g.valid) { slot = &g; break; } if (g.used < slot->used) slot = &g; }
            if (slot->exec) { cudaGraphExecDestroy(slot->exec); slot->exec = nullptr; }
            slot->valid = false;
            const int64_t l0 = c->launches;
            cudaGraph_t graph = nullptr;
            cudaError_t e = cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal);
            if (e == cudaSuccess) {
                rc = enqueue_cluster(c, type_mask);
                e = cudaStreamEndCapture(c->stream, &graph);
                const int64_t n_launch = c->launches - l0;
                c->launches = l0;
                if (rc == CSV_OK && e == cudaSuccess && graph && g_alloc_epoch.load() == key.alloc_epoch &&
                    cudaGraphInstantiate(&slot->exec, graph, 0) == cudaSuccess) {
                    slot->valid = true; slot->key = key; slot->launches = n_launch;
                    hit = slot;
                } else {
                    cudaGetLastError();
                    if (rc != CSV_OK && rc != CSV_E_CUDA) { if (graph) cudaGraphDestroy(graph); return rc; }
                }
                if (graph) cudaGraphDestroy(graph);
            } else cudaGetLastError();
        }
        if (hit) {
            CU(cudaGraphLaunch(hit->exec, c->stream));
            hit->used = ++c->graph_clock;
            c->launches += hit->launches;
            c->graph_replays++;
            c->last_mask = type_mask;
            done = true;
        } else { c->last_key = key; c->last_key_valid = true; }
    }
    if (!done) {
        rc = enqueue_cluster(c, type_mask);
        if (rc) return rc;
        if (c->last_key_valid && c->last_key.alloc_epoch != g_alloc_epoch.load()) c->last_key.alloc_epoch = g_alloc_epoch.load();
    }
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->ev_done, c->stream));
    c->done_pending = true;
    c->ran = true;
    c->counts_valid = false;
    return CSV_OK;
}

static int finish(csv_ctx* c) {
    if (!c->ran) return set_err(CSV_E_STATE, "csv_cluster has not been called");
    if (c->counts_valid) return CSV_OK;
    CU(cudaMemcpyAsync(c->h_counters, c->counters.p, sizeof(Counters), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    const uint32_t st = c->h_counters->status;
    if (st & (ST_BAD_CHROM | ST_BAD_POS | ST_NEG_FIELD | ST_BAD_GROUPS))
        return set_err(CSV_E_INPUT, "input validation failed on the device: %s%s%s%s", (st & ST_BAD_CHROM) ? "[contig id out of range] " : "",
                       (st & ST_BAD_POS) ? "[position outside its contig] " : "", (st & ST_NEG_FIELD) ? "[negative field] " : "",
                       (st & ST_BAD_GROUPS) ? "[contig_off of a grouped device upload is not 0 .. n, non-decreasing] " : "");
    if (st & ST_POW_TABLE) {
        // an allele with more supporting reads than the n**0.5 table: grow the table and rerun
        uint32_t need = c->h_counters->max_support + 1;
        uint32_t pn = c->pow_n;
        while (pn <= need) pn *= 2;
        int rc = upload_tables(c, pn);
        if (rc) return rc;
        return 1;  // rerun
    }
    if (st & ST_BIG_RUN) {
        // a DUP/INV/TRA run of equal primary keys longer than the ranking kernel handles: rerun those types with the chained sorts
        bool changed = false;
        for (int t = CSV_INV; t < CSV_NTYPES; t++) if (!c->small_chain[t]) { c->small_chain[t] = true; changed = true; }
        if (changed) return 1;
    }
    if (st) return set_err(CSV_E_CUDA, "internal pipeline error, status 0x%x (cand %u/%u names %u/%u)", st, c->h_counters->n_cand, c->cap_cand,
                           c->h_counters->n_names, c->cap_names);
    c->counts_valid = true;
    return CSV_OK;
}

extern "C" int csv_result_counts(csv_ctx* c, int64_t* n_cand, int64_t* n_names) {
    if (!c) return set_err(CSV_E_INVALID, "null ctx");
    CU(cudaSetDevice(c->device));
    int rc = finish(c);
    while (rc == 1) {  // table grown: rerun on the same device-resident inputs
        rc = csv_cluster(c, c->last_mask);
        if (rc) return rc;
        rc = finish(c);
    }
    if (rc) return rc;
    if (n_cand) *n_cand = c->h_counters->n_cand;
    if (n_names) *n_names = c->h_counters->n_names;
    return CSV_OK;
}

extern "C" int csv_fetch(csv_ctx* c, csv_cand* cands, csv_geno* genos, int64_t cap_cand, int32_t* names, int64_t cap_names) {
    int64_t nc = 0, nn = 0;
    int rc = csv_result_counts(c, &nc, &nn);
    if (rc) return rc;
    if (nc > cap_cand || nn > cap_names) return set_err(CSV_E_CAPACITY, "need %lld candidates / %lld names", (long long)nc, (long long)nn);
    stage_begin(c, c->stream, CSV_ST_D2H);
    if (nc) {
        CU(cudaMemcpyAsync(cands, c->cand.p, (size_t)nc * sizeof(csv_cand), cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(genos, c->geno.p, (size_t)nc * sizeof(csv_geno), cudaMemcpyDeviceToHost, c->stream));
    }
    if (nn) CU(cudaMemcpyAsync(names, c->names.p, (size_t)nn * 4, cudaMemcpyDeviceToHost, c->stream));
    stage_end(c, c->stream, CSV_ST_D2H);
    CU(cudaStreamSynchronize(c->stream));
    if (c->profiling || c->lane_marks) stage_collect(c);
    return CSV_OK;
}

extern "C" int csv_result_device_ptrs(csv_ctx* c, const csv_cand** cands, const csv_geno** genos, const int32_t** names) {
    if (!c || !c->ran) return set_err(CSV_E_STATE, "no results");
    if (cands) *cands = c->cand.as<csv_cand>();
    if (genos) *genos = c->geno.as<csv_geno>();
    if (names) *names = c->names.as<int32_t>();
    return CSV_OK;
}

static int cluster_host_impl(csv_ctx* c, const csv_sig_cols sigs[CSV_NTYPES], const int64_t* const* sig_off, const csv_reads_cols* reads,
                             const int64_t* reads_off, bool grouped, uint32_t type_mask, csv_cand* cands, csv_geno* genos, int64_t cap_cand,
                             int32_t* names, int64_t cap_names, int64_t* n_cand, int64_t* n_names) {
    if (!c || !sigs) return set_err(CSV_E_INVALID, "null argument");
    int rc;
    for (int t = 0; t < CSV_NTYPES; t++) {
        if (!(type_mask >> t & 1)) continue;
        if (grouped && sigs[t].n > 0 && (!sig_off || !sig_off[t])) return set_err(CSV_E_INVALID, "null contig_off");
        rc = upload_sigs_impl(c, t, &sigs[t], grouped && sigs[t].n > 0 ? sig_off[t] : nullptr, HOST_SRC);
        if (rc) return rc;
    }
    if (reads) {
        if (grouped && reads->n > 0 && !reads_off) return set_err(CSV_E_INVALID, "null contig_off");
        rc = upload_reads_impl(c, reads, grouped && reads->n > 0 ? reads_off : nullptr, HOST_SRC);
        if (rc) return rc;
    }
    rc = csv_cluster(c, type_mask);
    if (rc) return rc;
    int64_t nc = 0, nn = 0;
    rc = csv_result_counts(c, &nc, &nn);
    if (rc) return rc;
    if (n_cand) *n_cand = nc;
    if (n_names) *n_names = nn;
    return csv_fetch(c, cands, genos, cap_cand, names, cap_names);
}
extern "C" int csv_cluster_host(csv_ctx* c, const csv_sig_cols sigs[CSV_NTYPES], const csv_reads_cols* reads, uint32_t type_mask,
                                csv_cand* cands, csv_geno* genos, int64_t cap_cand, int32_t* names, int64_t cap_names, int64_t* n_cand,
                                int64_t* n_names) {
    return cluster_host_impl(c, sigs, nullptr, reads, nullptr, false, type_mask, cands, genos, cap_cand, names, cap_names, n_cand, n_names);
}
extern "C" int csv_cluster_host_grouped(csv_ctx* c, const csv_sig_cols sigs[CSV_NTYPES], const int64_t* const sig_off[CSV_NTYPES],
                                        const csv_reads_cols* reads, const int64_t* reads_off, uint32_t type_mask, csv_cand* cands,
                                        csv_geno* genos, int64_t cap_cand, int32_t* names, int64_t cap_names, int64_t* n_cand,
                                        int64_t* n_names) {
    return cluster_host_impl(c, sigs, sig_off, reads, reads_off, true, type_mask, cands, genos, cap_cand, names, cap_names, n_cand, n_names);
}

extern "C" int csv_cal_gl(csv_ctx* c, const int32_t* c0, const int32_t* c1, int64_t n, csv_geno* out) {
    if (!c || !c0 || !c1 || !out || n < 0) return set_err(CSV_E_INVALID, "bad argument");
    if (n == 0) return CSV_OK;
    CU(cudaSetDevice(c->device));
    CU(c->cal_in0.ensure((size_t)n * 4)); CU(c->cal_in1.ensure((size_t)n * 4)); CU(c->cal_out.ensure((size_t)n * sizeof(csv_geno)));
    int32_t *d0 = c->cal_in0.as<int32_t>(), *d1 = c->cal_in1.as<int32_t>();
    csv_geno* dg = c->cal_out.as<csv_geno>();
    CU(cudaMemcpyAsync(d0, c0, n * 4, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d1, c1, n * 4, cudaMemcpyHostToDevice, c->stream));
    LAUNCH(c, c->stream, k_cal_gl, grid_for(c, n, 256), 256, 0, d0, d1, n, c->gl_table.as<csv_geno>(), dg);
    CU(cudaMemcpyAsync(out, dg, n * sizeof(csv_geno), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return CSV_OK;
}

extern "C" int csv_stage_ms(csv_ctx* c, float ms[CSV_ST_COUNT]) {
    if (!c || !ms) return set_err(CSV_E_INVALID, "null argument");
    for (int s = 0; s < CSV_ST_COUNT; s++) ms[s] = c->stage_ms[s];
    return CSV_OK;
}
extern "C" int64_t csv_launch_count(csv_ctx* c) { return c ? c->launches : 0; }
extern "C" int64_t csv_graph_replays(csv_ctx* c) { return c ? c->graph_replays : 0; }
extern "C" int csv_debug_counters(csv_ctx* c, uint32_t out[32]) {
    if (!c || !out || !c->h_counters) return set_err(CSV_E_INVALID, "null argument");
    static_assert(sizeof(Counters) == 32 * 4, "Counters layout");
    memcpy(out, c->h_counters, 32 * 4);
    return CSV_OK;
}

// Per-kernel totals of the intervals collected while profiling was on (since the last collection): one line per
// kernel, "name<TAB>launches<TAB>total_ms".  Returns the text length needed (incl. NUL) when cap is too small.
extern "C" int64_t csv_kernel_times(csv_ctx* c, char* buf, int64_t cap) {
    if (!c) return 0;
    std::string out;
    char line[512];
    for (const auto& kt : c->ktotals) {
        snprintf(line, sizeof(line), "%s\t%lld\t%.6f\n", kt.name.c_str(), (long long)kt.launches, kt.ms);
        out += line;
    }
    if (buf && cap > 0) {
        const size_t k = std::min<size_t>(out.size(), (size_t)cap - 1);
        memcpy(buf, out.data(), k);
        buf[k] = 0;
    }
    return (int64_t)out.size() + 1;
}

extern "C" int csv_sort_probe(csv_ctx* c, float* ms_total, int64_t* bytes_total, int32_t* launches) {
    if (!c) return set_err(CSV_E_INVALID, "null ctx");
    if (ms_total) *ms_total = c->sort_ms;
    if (bytes_total) *bytes_total = c->sort_bytes;
    if (launches) *launches = c->sort_launches;
    return CSV_OK;
}

// scan_api.inl: the scan's per-packet step inside extract_impl and the alignment table csv_rank_names installs
static int scan_packet(csv_ctx* c, const csv_read_cols* reads, bool want_aln, int64_t* n_aln_new);
static int scan_install_alignments(csv_ctx* c, cudaStream_t st, LbPool& lb);

#include "extract_api.inl"
#include "gather_api.inl"
#include "genotype_api.inl"
#include "sigsort_api.inl"
#include "names_api.inl"
#include "scan_api.inl"
#include "sa_api.inl"
