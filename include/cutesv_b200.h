/*
 * cutesv_b200.h -- C-ABI of the H100-native cuteSV hot path
 * (signature extraction -> sort + chain-linkage clustering -> consensus -> genotype).
 *
 * The reference (tjiangHIT/cuteSV v2.1.4) is pure Python and has no FFI; every entry point
 * below cites the reference interface it replaces ("cuteSV:N" = src/cuteSV/cuteSV line N,
 * other files relative to src/cuteSV/).  The Python binding a maintainer would add is the
 * ctypes stub in cutesv_b200/_lib.py (see INTEGRATION.md).
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; csv_last_error() gives the text.
 *   - the caller owns every host buffer; the library owns all device memory inside a csv_ctx.
 *   - outputs use capacity + "needed" convention (CSV_E_CAPACITY -> retry with larger buffers).
 *   - one csv_ctx per GPU; calls on one ctx are not re-entrant; no callbacks, no exceptions.
 *   - there is NO CPU fallback: csv_create fails if no sm_90 (H100) device is usable.
 *
 * Columnar signature layout (int32 columns, one set per SV type; reference tuple types at
 * cuteSV:520-531 (INS/DEL), 235-239 (DUP), 55-60 (INV), 111-117 (TRA)):
 *
 *   type  chrom        a                  b        read_id   c
 *   DEL   contig id    pos                len      name rank -
 *   INS   contig id    2*pos (carries .5) len      name rank len(seq)
 *   INV   contig id    bp1                bp2      name rank strand: 0 "++", 1 "--"
 *   DUP   contig id    pos1               pos2     name rank -
 *   TRA   contig id 1  pos1               pos2     name rank chr2_id*4 + {A:0,B:1,C:2,D:3}
 *
 * contig id = rank of the contig name in Python string order, read_id = rank of the read name
 * in Python string order (the reference sorts tuples with string tie-breaks, cuteSV:764-801).
 *
 * INS rows that tie on (contig, int(pos), len, read_id) must come in the order of their sequence strings: the
 * reference's INS sort key is (chr, int(pos), len, name, seq) (cuteSV:774) and the library never sees the strings,
 * it breaks such ties by input order.  They need one read reporting two insertions of equal length at the same
 * position; the host converters (workdir.py, cli.py) put them in order.
 */
#ifndef CUTESV_B200_H
#define CUTESV_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Emission order of the reference's clustering phase (cuteSV:1116-1189). */
enum { CSV_DEL = 0, CSV_INS = 1, CSV_INV = 2, CSV_DUP = 3, CSV_TRA = 4, CSV_NTYPES = 5 };

enum {
    CSV_OK = 0,
    CSV_E_INVALID = -1,  /* bad argument */
    CSV_E_CUDA = -2,     /* CUDA runtime error */
    CSV_E_CAPACITY = -3, /* output buffer too small; sizes are reported back */
    CSV_E_NODEVICE = -4, /* no usable sm_90 device: the product path never falls back to CPU */
    CSV_E_INPUT = -5,    /* device-side validation of the inputs failed (see csv_last_error) */
    CSV_E_STATE = -6     /* call sequence error */
};

/* Flags of csv_cand.flags */
enum {
    CSV_F_NO_READS = 1, /* call_gt(): contig absent from the reads table -> the reference drops
                           every candidate of that contig (resolveINDEL.py:443-444) */
    CSV_F_GT_HOST = 2   /* genotype must be completed on the host (TRA: BAM-order dependent,
                           resolveTRA.py:260-309) */
};

/* POD mirror of the reference flags that reach the hot path (cuteSV_Description.py:53-263;
 * argument wiring at cuteSV:1058-1076 and 1116-1189). */
typedef struct csv_params {
    int32_t min_support;        /* -s: read_count of every resolution_* */
    int32_t min_support_allele; /* minimum_support_reads = min(min_support, 5), cuteSV:1124,1141 */
    int32_t min_size;           /* -l: sv_size */
    int32_t max_size;           /* -L: MaxSize (-1 = unlimited) */
    int32_t bias_del, bias_ins, bias_inv, bias_dup, bias_tra; /* --max_cluster_bias_* */
    int32_t genotype;           /* --genotype: "action" */
    int32_t gt_round;           /* --gt_round (TRA host genotyper only) */
    int32_t gt_bias_ins;        /* constant 1000 of resolveINDEL.py:312 */
    double ratio_del, ratio_ins; /* --diff_ratio_merging_DEL / _INS: threshold_gloab */
    double ratio_tra;            /* --diff_ratio_filtering_TRA: overlap_size */
    double remain_reads_ratio;   /* --remain_reads_ratio */
    /* extraction (cuteSV:606, 697) */
    int32_t min_mapq, max_split_parts, min_read_len, min_siglength;
    int32_t merge_del_threshold, merge_ins_threshold;
    int32_t reserved[2];
} csv_params;

/* One SV type's signature columns (host or device pointers, depending on the call). */
typedef struct csv_sig_cols {
    int64_t n;
    const int32_t* chrom;
    const int32_t* a;
    const int32_t* b;
    const int32_t* read_id;
    const int32_t* c; /* may be NULL for DEL / DUP */
} csv_sig_cols;

/* reads_info_list rows (cuteSV:729-733): (start, end, is_primary, name, chr). */
typedef struct csv_reads_cols {
    int64_t n;
    const int32_t* chrom;
    const int32_t* start;
    const int32_t* end;
    const int32_t* read_id;
    const uint8_t* is_primary;
} csv_reads_cols;

/* Candidate record, 64 B.  One per row returned by resolution_* (resolveINDEL.py:197-205,
 * 408-417; resolveDUP.py:114-118; resolveINV.py:136-143; resolveTRA.py:171-182). */
typedef struct csv_cand {
    int32_t svtype;     /* CSV_* */
    int32_t chrom;      /* contig id (TRA: chr1) */
    int32_t pos;        /* DEL/INS breakpoint, DUP bp1, INV bp1, TRA pos1 */
    int32_t len;        /* DEL: -len (as printed), INS: len, DUP: bp2-bp1, INV: inv_len, TRA: 0 */
    int32_t support;    /* RE / DV */
    int32_t cipos;      /* INDEL: x of "-x,x" */
    int32_t cilen;
    int32_t search_pos; /* INDEL: centre of the genotyping window (resolveINDEL.py:204,415) */
    int32_t pos2;       /* DUP bp2, INV bp2, TRA pos2 */
    int32_t aux;        /* INS: input index of the signature whose seq is the ALT (host slices
                           seq[:len]); INV: strand; TRA: chr2_id*4+type */
    int32_t names_off;  /* slice of the names buffer: supporting read ids in reference order */
    int32_t names_cnt;
    int32_t cluster;    /* ordinal of the chain-linkage cluster this row came from */
    int32_t flags;      /* CSV_F_* */
    int32_t reserved[2]; /* [1]: source rank of a record returned by csv_fetch_gathered */
} csv_cand;

/* assign_gt()/cal_GL() result (cuteSV_genotype.py:33-56,161-173), 40 B. */
typedef struct csv_geno {
    int32_t dr;    /* -1 when genotyping is off or deferred to the host */
    int32_t dv;
    int32_t gt;    /* 0 "0/0", 1 "0/1", 2 "1/1", -1 "./." */
    int32_t pl[3];
    int32_t gq;
    int32_t status; /* 0 filled, 1 not computed */
    double qual;
} csv_geno;

typedef struct csv_ctx csv_ctx;

/* Stages timed with CUDA events on the ctx stream when profiling is on. */
enum {
    CSV_ST_H2D = 0,
    CSV_ST_KEYS,      /* key building + validation */
    CSV_ST_SORT,      /* radix sort passes */
    CSV_ST_SEGMENT,   /* chain-linkage boundary votes + kept-cluster compaction */
    CSV_ST_CLUSTER,   /* per-cluster consensus kernels */
    CSV_ST_ORDER,     /* candidate ordering */
    CSV_ST_GENOTYPE,  /* window binning + reads pass + cal_GL */
    CSV_ST_D2H,
    CSV_ST_EXTRACT,   /* CIGAR / SA walk */
    CSV_ST_COUNT
};

const char* csv_last_error(void);
int csv_version(void);

/* Fill *p with the reference defaults (cuteSV_Description.py:78-262). */
int csv_default_params(csv_params* p);

/* device: CUDA ordinal.  stream: a cudaStream_t to run on (NULL = library-owned stream). */
int csv_create(int device, void* stream, csv_ctx** out);
int csv_destroy(csv_ctx* ctx);
int csv_set_params(csv_ctx* ctx, const csv_params* p);
/* Contig table: id = rank of the name in Python string order; lens from the BAM header
 * (cuteSV:1029).  Needed to linearise (contig, pos) into one sortable coordinate.  Up to 2^29 - 1
 * contigs (draft assemblies with 10^5-10^6 scaffolds included; TRA's chr2*4+type is int32); more are
 * CSV_E_INVALID.  Every contig must be shorter than 2^30 bp, since INS positions and genotype windows
 * are half units in int32.  That length limit is NOT validated here: lengths up to 2^31 - 1 are
 * accepted, and INS / genotyping results on a contig of 2^30 bp or more are undefined. */
int csv_set_contigs(csv_ctx* ctx, int32_t n_contigs, const int64_t* contig_len);

/* Pinned host memory helpers (caller-owned buffers stay caller-owned). */
int csv_host_alloc(void** p, size_t bytes);
int csv_host_free(void* p);
int csv_host_register(void* p, size_t bytes);
int csv_host_unregister(void* p);

/* Replaces the pickle transport <work_dir>/<TYPE>.pickle + reads.pickle (cuteSV:817-857):
 * async H2D copy of the columns onto the ctx stream.  n == 0 clears the type. */
int csv_upload_sigs(csv_ctx* ctx, int svtype, const csv_sig_cols* host_cols);
int csv_upload_reads(csv_ctx* ctx, const csv_reads_cols* host_cols);
/* The same with rows GROUPED BY CONTIG, as the reference itself holds them (one list per chromosome:
 * the <TYPE>.pickle / reads.pickle files are dicts keyed by chr, cuteSV:817-857): all rows of contig
 * id 0, then id 1, ...; host_cols->chrom is ignored (may be NULL) and contig_off[k] .. contig_off[k+1]
 * (n_contigs + 1 entries, contig_off[0] == 0, contig_off[n_contigs] == n) is the row range of contig k.
 * Saves the 4-byte contig column on the PCIe link; the column is rebuilt on the device. */
int csv_upload_sigs_grouped(csv_ctx* ctx, int svtype, const csv_sig_cols* host_cols, const int64_t* contig_off);
int csv_upload_reads_grouped(csv_ctx* ctx, const csv_reads_cols* host_cols, const int64_t* contig_off);

/* Optional input of the TRA genotyper: ALL alignment records (no mapq filter, every flag) in BAM
 * order, i.e. coordinate-sorted per contig, contigs ascending by id.  is_primary = flag in (0, 16).
 * The reference re-opens the BAM per TRA candidate and iterates bam.fetch() with an early exit
 * (call_gt resolveTRA.py:260-309, count_coverage cuteSV_genotype.py:72-93); with this table the same
 * scan runs on the device.  Without it TRA rows keep CSV_F_GT_HOST.  n == 0 clears the table.
 * The per-contig row index is built in parallel (one thread per contig), so the call stays cheap at
 * large contig counts.
 * Precondition (as for the reads table): one primary record per read name. */
int csv_upload_alignments(csv_ctx* ctx, const csv_reads_cols* aln);

/* ---- the same uploads from columns that already live in GPU memory (a PyTorch pipeline, a GPU aligner, another ctx's
 * extraction) ----
 * Every non-null column (and contig_off, n_contigs + 1 int64) must be device or managed memory on the ctx's device, as
 * cudaPointerGetAttributes reports it; anything else is CSV_E_INVALID naming the column.  Host columns keep going through the
 * calls above.  Counts limits, the "column c required for INS/INV/TRA" rule and n == 0 behave as in the host calls.
 *   - Copy, not borrow: the columns are copied device-to-device into the ctx's own buffers, which csv_remap_read_ids /
 *     csv_swap_ins_rows rewrite and captured CUDA graphs address.
 *   - Stream order both ways, no host synchronisation: stream is the caller's producer stream (NULL = the legacy default
 *     stream).  The copies wait for everything enqueued on it before the call, and it waits for the copies: the caller may
 *     overwrite or free its buffers in stream order as soon as the call returns.
 *   - Grouped calls: contig_off is read on the device only.  Offsets that do not start at 0, end at n and never decrease make
 *     the next csv_cluster return CSV_E_INPUT; the rows then get contig 0 and nothing outside the given buffers is read or
 *     written.  An upload of the same slot with valid offsets (or any other upload of it) clears the report.
 *   - csv_upload_alignments_device checks the table's order like csv_upload_alignments and, like it, blocks until that check
 *     is done (the copies are then complete too).
 * csv_cluster waits for pending device uploads before its kernel chain, so a call on fresh device inputs of unchanged sizes
 * replays its captured graph (see csv_graph_replays). */
int csv_upload_sigs_device(csv_ctx* ctx, int svtype, const csv_sig_cols* dev_cols, void* stream);
int csv_upload_reads_device(csv_ctx* ctx, const csv_reads_cols* dev_cols, void* stream);
int csv_upload_sigs_grouped_device(csv_ctx* ctx, int svtype, const csv_sig_cols* dev_cols, const int64_t* contig_off, void* stream);
int csv_upload_reads_grouped_device(csv_ctx* ctx, const csv_reads_cols* dev_cols, const int64_t* contig_off, void* stream);
int csv_upload_alignments_device(csv_ctx* ctx, const csv_reads_cols* dev_cols, void* stream);

/* Replaces process_process_sigs_type (sort + dedup, cuteSV:750-857) and the whole clustering
 * phase Pool(run_del|run_ins|run_inv|run_dup|run_tra) (cuteSV:1113-1199) including call_gt /
 * overlap_cover / assign_gt / cal_GL (cuteSV_genotype.py:33-173) for every contig at once.
 * Asynchronous on the ctx stream; operates on the device-resident inputs.
 * type_mask: bit t set = run SV type t. */
int csv_cluster(csv_ctx* ctx, uint32_t type_mask);

/* Blocks until csv_cluster finished; reports the result sizes. */
int csv_result_counts(csv_ctx* ctx, int64_t* n_cand, int64_t* n_names);
/* D2H of the results.  Order: svtype ascending (DEL, INS, INV, DUP, TRA), then contig id, then
 * the reference's emission order inside one resolution_* call. */
int csv_fetch(csv_ctx* ctx, csv_cand* cands, csv_geno* genos, int64_t cap_cand, int32_t* names,
              int64_t cap_names);
/* Device pointers of the result buffers (for an NCCL all-gather of candidate records). */
int csv_result_device_ptrs(csv_ctx* ctx, const csv_cand** cands, const csv_geno** genos,
                           const int32_t** names);

/* The reference-facing one-shot call: host columns in, host rows out (H2D + kernels + D2H).
 * sigs[t] may have n == 0.  On CSV_E_CAPACITY *n_cand / *n_names hold the needed sizes. */
int csv_cluster_host(csv_ctx* ctx, const csv_sig_cols sigs[CSV_NTYPES], const csv_reads_cols* reads,
                     uint32_t type_mask, csv_cand* cands, csv_geno* genos, int64_t cap_cand,
                     int32_t* names, int64_t cap_names, int64_t* n_cand, int64_t* n_names);

/* csv_cluster_host over grouped inputs (see csv_upload_sigs_grouped); sig_off[t] may be NULL when sigs[t].n == 0. */
int csv_cluster_host_grouped(csv_ctx* ctx, const csv_sig_cols sigs[CSV_NTYPES], const int64_t* const sig_off[CSV_NTYPES],
                             const csv_reads_cols* reads, const int64_t* reads_off, uint32_t type_mask, csv_cand* cands,
                             csv_geno* genos, int64_t cap_cand, int32_t* names, int64_t cap_names, int64_t* n_cand,
                             int64_t* n_names);

/* cal_GL(c0=DR, c1=DV) (cuteSV_genotype.py:33-56) for n pairs, evaluated on the device. */
int csv_cal_gl(csv_ctx* ctx, const int32_t* c0, const int32_t* c1, int64_t n, csv_geno* out);

/* ---- standalone genotype helpers: overlap_cover (cuteSV_genotype.py:95-159) and the call_gt of resolveINDEL.py:441,
 * resolveDUP.py:137 and resolveINV.py:208 over any window list and reads table (both may span several contigs) ----
 *
 * Coordinates are in half units, so that the x.5 windows of DUP / INV (bias/2) are exact: window [s, e] is
 * (s2, e2) = (2s, 2e), a reads-table row [start, end] is compared as (2 start, 2 end).  A row overlaps a window iff
 * start < e and end > s; it covers it iff start <= s and end >= e.  Only rows on the window's contig count.
 *
 * reads == NULL: the device-resident reads table of csv_extract* / csv_upload_reads*.  Neither call changes that table
 * nor anything csv_cluster / csv_fetch return; both block until their results are on the host.
 * Input errors (CSV_E_INPUT): a window with chrom < 0 or e2 <= s2 (the reference raises KeyError there), a reads row with
 * chrom < 0 or end < start. */
typedef struct csv_window {
    int32_t chrom;    /* contig id, the same numbering as the reads table's chrom column */
    int32_t reserved;
    int64_t s2;       /* 2 * window start */
    int64_t e2;       /* 2 * window end, > s2 */
} csv_window;

/* overlap_cover: iteration[i] = overlapping rows, primary_num[i] = overlapping rows with is_primary != 0;
 * cover / overlap: per window the distinct read ids of the primary covering / overlapping rows, ascending, as CSR
 * (cover_off / overlap_off: n_windows + 1 entries).  On CSV_E_CAPACITY *n_cover / *n_overlap hold the sizes needed.
 * overlap_ids may be NULL (with cap_overlap 0) to skip the overlap lists; overlap_off is then left alone. */
int csv_overlap_cover(csv_ctx* ctx, const csv_window* windows, int64_t n_windows, const csv_reads_cols* reads,
                      int32_t* iteration, int32_t* primary_num, int64_t* cover_off, int32_t* cover_ids, int64_t cap_cover,
                      int64_t* overlap_off, int32_t* overlap_ids, int64_t cap_overlap, int64_t* n_cover, int64_t* n_overlap);

/* call_gt + assign_gt: n_cand candidates of windows_per_cand (1: DEL / INS, 2: DUP / INV breakpoints, whose cover
 * sets are united) consecutive windows each; support_off (n_cand + 1) / support_ids: every candidate's supporting
 * read ids in any order, duplicates allowed.  DR = |cover \ support|, DV = the support list's length,
 * out[i] = cal_GL(DR, DV) with dr / dv filled. */
int csv_call_gt(csv_ctx* ctx, const csv_window* windows, int64_t n_cand, int32_t windows_per_cand, const csv_reads_cols* reads,
                const int64_t* support_off, const int32_t* support_ids, csv_geno* out);

/* ---- standalone TRA genotyper: the call_gt of resolveTRA.py:260-309 (count_coverage, cuteSV_genotype.py:72-93) for
 * caller-given breakpoint pairs over an all-alignments table in BAM order ----
 *
 * Query i scans the window [max(pos1 - bias, 0), min(pos1 + bias, len(chr1))] of chr1 and, when that scan ends without
 * an early return, the same window around pos2 on chr2; contig lengths come from csv_set_contigs.  A record is fetched by
 * a window [s, e] iff start < e and end > s.  support_off (n + 1) / support_ids: every query's supporting read ids in any
 * order, duplicates allowed; DV = the segment's length, membership is by id.
 *   - the first scan returns -1 (more than 20% primary records at gt_round): out[i] = {dr -1, dv, gt -1, status 2};
 *   - otherwise out[i] = cal_GL(DR, DV) with dr / dv filled (the second scan's status is not used, as in the reference).
 * aln: host columns (chrom, start, end, read_id, is_primary = flag in (0, 16)), copied into the call's own scratch; NULL
 * uses the table installed by csv_upload_alignments* / csv_rank_names (CSV_E_STATE when there is none).  Precondition, as
 * for that table: one primary record per read name.
 * Errors, all found before any launch except the table's order (CSV_E_INPUT), and none changing the ctx:
 *   CSV_E_INVALID  a null pointer, n outside [0, 2^29), bias < 0, support_off not starting at 0 or decreasing;
 *   CSV_E_INPUT    a contig id outside the contig table or a clamped window with start > end (pysam's fetch raises
 *                  ValueError), naming the query; a table not in BAM order or with a contig id out of range.
 * Blocks until out is on the host.  Leaves csv_cluster's inputs, results, alignment table and captured graphs alone. */
typedef struct csv_tra_query {
    int32_t chr1, chr2;   /* contig ids of the two breakpoints */
    int64_t pos1, pos2;
} csv_tra_query;
int csv_tra_call_gt(csv_ctx* ctx, const csv_tra_query* q, int64_t n, const csv_reads_cols* aln, int32_t bias, int32_t gt_round,
                    const int64_t* support_off, const int32_t* support_ids, csv_geno* out);

/* ---- standalone signature rebuild: the sort + remove_duplicates_sorted of process_process_sigs_type (cuteSV:750-857,
 * 958-969) over the device-resident columns of ONE type (svtype CSV_DEL..CSV_TRA) or of the reads table
 * (svtype CSV_SORT_READS), i.e. whatever csv_upload_sigs / csv_upload_reads (grouped or not) or csv_extract* put there ----
 *
 * Sort key, stable on input order (names and contigs are ranks), and what counts as an adjacent duplicate:
 *   DEL, DUP  chrom, a, b, read_id                        all four fields equal
 *   INV       chrom, c (strand), a, b, read_id            all five equal
 *   TRA       chrom, c>>2 (chr2), c&3 (type), a, b, read_id   all five equal
 *   INS       chrom, a>>1 (int(pos)), b, read_id          none dropped (see ins_tie)
 *   reads     chrom                                       none dropped
 * order[k] (k < *n_kept) = input row of the k-th kept row; contig_off (n_contigs + 1 entries) = row range of every contig
 * id inside order, which is what the reference's per-contig pickle index needs.  On CSV_E_CAPACITY (*n_kept > cap) nothing
 * but *n_kept is written.
 * INS: the reference's key ends with the sequence string (cuteSV:774), which the library never sees.  ins_tie[k] = 1 when
 * kept row k ties with row k - 1 on (chrom, int(pos), len, read_id); the host orders every such group by sequence
 * (stably) and drops the adjacent duplicates (equal a, b, read_id and sequence).  The groups need one read reporting two
 * equal insertions at one position, so they are rare.  ins_tie may be NULL; for other types it is zero-filled.
 * Key widths follow the data (contig count, coordinates, read count), so > 32 768 contigs and genome spans > 2^32 sort as
 * they are.  Own scratch: neither the device-resident inputs nor anything csv_cluster / csv_fetch return change.
 * Input errors (CSV_E_INPUT): a contig id outside the contig table, a negative field.  Blocks until the results are on
 * the host. */
enum { CSV_SORT_READS = 5 };
int csv_sort_sigs(csv_ctx* ctx, int svtype, int64_t* order, int64_t cap, int64_t* n_kept, int64_t* contig_off, uint8_t* ins_tie);

/* ---- signature extraction: parse_read / generate_combine_sigs / organize_split_signal /
 * analysis_split_read (cuteSV:50-681) over a packet of decoded alignment records ---- */

/* Per-record header (pysam fields the reference reads at cuteSV:606-680). */
typedef struct csv_read_cols {
    int64_t n;
    const int32_t* chrom;     /* contig id */
    const int32_t* ref_start; /* read.reference_start */
    const int32_t* ref_end;   /* read.reference_end */
    const int32_t* flag;      /* read.flag */
    const int32_t* mapq;
    const int32_t* query_len; /* read.query_length */
    const int32_t* read_id;   /* name rank */
    const int64_t* cigar_off; /* n+1 offsets into cigar[] */
    const int64_t* sa_off;    /* n+1 offsets into the SA segment table */
} csv_read_cols;

/* SA-tag entries reduced on the host with acquire_clip_pos semantics (cuteSV:466-513). */
typedef struct csv_sa_cols {
    int64_t n;
    const int32_t* chrom;      /* contig id of the SA entry */
    const int32_t* pos0;       /* int(seq[1]) - 1 */
    const int32_t* strand;     /* 0 '+', 1 '-' */
    const int32_t* mapq;
    const int32_t* first_clip; /* leading S length */
    const int32_t* last_clip;  /* trailing S length */
    const int32_t* ref_span;   /* sum of M, D, =, X */
} csv_sa_cols;

/* Extracted signatures and reads-table rows REPLACE the device-resident inputs of csv_cluster()
 * (one packet per call); counts per type are reported.  cigar[] is BAM-native u32 = len << 4 | op.
 * Replaces Pool#1 (single_pipe/parse_read per window, cuteSV:1058-1076) without the pickle files.
 * INS sequences are not materialised on the device: every INS signature carries len(seq) in
 * column c plus a list of "pieces" (Python slices of a record's query sequence, or of its
 * reverse complement) from which the host rebuilds the string when it needs it. */
int csv_extract(csv_ctx* ctx, const csv_read_cols* reads, const uint32_t* cigar, int64_t n_cigar,
                const csv_sa_cols* sa, int64_t counts[CSV_NTYPES], int64_t* n_read_rows);
/* Append mode (cuteSV:734-739: every task's signatures are appended to the per-type lists; the reference then
 * concatenates the lists of all tasks, cuteSV:750-762): like csv_extract, but the signatures, INS piece descriptors
 * and reads-table rows of this packet are APPENDED to the device-resident inputs of csv_cluster, so a BAM-to-VCF run
 * never moves a signature column across PCIe.  The record index in an INS piece is the packet-local index plus the
 * number of records of all earlier packets of the accumulation.  counts / n_read_rows report the totals so far.
 * csv_extract_reset (or a plain csv_extract / csv_upload_*) starts a new accumulation. */
int csv_extract_append(csv_ctx* ctx, const csv_read_cols* reads, const uint32_t* cigar, int64_t n_cigar,
                       const csv_sa_cols* sa, int64_t counts[CSV_NTYPES], int64_t* n_read_rows);
int csv_extract_reset(csv_ctx* ctx);

/* ---- extraction from alignment records that already live in GPU memory (a GPU aligner, a PyTorch pipeline) ----
 * Query bases in BAM's 4-bit packed form ("=ACMGRSVTWYHKDBN", high nibble first): record i's bases start at byte
 * seq_off[i] (n + 1 entries), query_len[i] bases are expected.  A record with fewer than (query_len + 1) / 2 stored bytes has
 * no stored sequence (BAM '*'): its INS slices are empty.  bamio.BamReader.next_packet produces this layout. */
typedef struct csv_seq_cols {
    int64_t n_bytes;
    const int64_t* seq_off;
    const uint8_t* seq4;
} csv_seq_cols;
/* csv_extract / csv_extract_append (same results, counters, record column and skipped-record count) on a packet whose
 * columns, CIGAR stream, SA table and bases (seq, may be NULL) are device or managed memory on the ctx's device, as
 * cudaPointerGetAttributes reports it; anything else is CSV_E_INVALID naming the column.  Device and host packets may be
 * mixed in one append accumulation.
 *   - Stream order both ways: the call's device work waits for everything enqueued on `stream` (NULL = the legacy default
 *     stream) before it, and `stream` waits for the call's last read of the caller's memory.  The call blocks the host
 *     until the output counts are known, as the host calls do.
 *   - Only the CIGAR stream is copied (into the ctx's padded buffer: the kernel's bulk copies read whole tiles); the other
 *     columns and the bases are read in place during the call.
 *   - The offsets are checked on the device before any kernel reads through them: cigar_off, sa_off and seq_off must start
 *     at >= 0, never decrease and end at <= n_cigar, sa->n and seq->n_bytes; query_len must be >= 0.  A failure is
 *     CSV_E_INPUT naming the column and changes nothing: the previous accumulation and its counters stay as they were.
 *   - With seq, the sequence of every new INS signature is built on the device into a ctx-owned arena, appended per packet:
 *     row k's string is bytes[start[k] .. start[k] + len[k]), byte-identical to what the host builds from the piece list
 *     (cutesv_b200/packing.py ins_sequence, marker pieces included).  The arena is valid while every packet of the
 *     accumulation carried seq; any other extraction, csv_extract_reset or a signature / reads upload invalidates it.
 *     csv_swap_ins_rows keeps it attached to the rows, csv_remap_read_ids leaves it alone.  The strings of one packet must
 *     stay below 4 GiB, else CSV_E_CAPACITY: an append call then leaves the accumulation as it was, a non-append call leaves
 *     it empty (as csv_extract_reset does; its kernel has already overwritten the previous rows). */
int csv_extract_device(csv_ctx* ctx, const csv_read_cols* reads, const uint32_t* cigar, int64_t n_cigar, const csv_sa_cols* sa,
                       const csv_seq_cols* seq, void* stream, int64_t counts[CSV_NTYPES], int64_t* n_read_rows);
int csv_extract_append_device(csv_ctx* ctx, const csv_read_cols* reads, const uint32_t* cigar, int64_t n_cigar, const csv_sa_cols* sa,
                              const csv_seq_cols* seq, void* stream, int64_t counts[CSV_NTYPES], int64_t* n_read_rows);
/* Device pointers of the INS sequence arena, for a caller's own CUDA code: ASCII bases, the int64 start and the int32 length
 * of every INS row (n_rows = the INS signature count).  Blocks until the arena is complete.  Valid until the next
 * extraction, upload, csv_swap_ins_rows or csv_destroy.  CSV_E_STATE when the arena is not valid. */
int csv_ins_seq_device_ptrs(csv_ctx* ctx, const uint8_t** bytes, const int64_t** start, const int32_t** len, int64_t* n_rows);
/* Strings of INS rows rows[0..n) (any order, repeats allowed) gathered on the device, one D2H copy of the strings: row rows[i]
 * is out[out_off[i] .. out_off[i + 1]) (out_off: n + 1 entries, 64-bit, so the total may exceed 4 GiB).  On CSV_E_CAPACITY
 * out_off is filled and out_off[n] is the size `out` needs.  CSV_E_STATE when the arena is not valid, CSV_E_INVALID for a row
 * outside the INS signatures. */
int csv_fetch_ins_seqs(csv_ctx* ctx, const int64_t* rows, int64_t n, uint8_t* out, int64_t cap, int64_t* out_off);

/* ---- read names of device packets, ranked on the device ----
 * The reference's sort keys break ties on the read name in Python string order (cuteSV:764-801), so every read id must be
 * the rank of its name across the whole run.  A named packet carries the names instead of ids: record i's name is
 * names[name_off[i] .. name_off[i + 1]) (name_off: n + 1 entries), without a NUL terminator, compared as bytes (for UTF-8
 * text byte order is Python str order). */
typedef struct csv_name_cols {
    int64_t n_bytes;
    const int64_t* name_off;
    const uint8_t* names;
} csv_name_cols;
/* csv_extract_device / csv_extract_append_device on a named packet (device memory, like every other column); reads->read_id
 * must be NULL (CSV_E_INVALID otherwise).
 *   - Each record gets a provisional read id: its index in the accumulation (the records of earlier packets plus the
 *     packet-local index, the numbering of csv_fetch_records).  csv_rank_names turns these into ranks.
 *   - The names are copied device to device into a ctx-owned arena, appended per packet, in the stream order of the CIGAR copy.
 *   - name_off is checked on the device with the other offsets: start >= 0, never decreasing, end <= n_bytes, every name at
 *     most 254 bytes (BAM's limit).  A failure is CSV_E_INPUT naming the column and changes nothing.
 *   - CSV_E_STATE, changing nothing: a named packet appended to an accumulation of unnamed packets or the reverse (host
 *     packets included), or any append after csv_rank_names (csv_extract_reset or a fresh extraction starts over). */
int csv_extract_named_device(csv_ctx* ctx, const csv_read_cols* reads, const uint32_t* cigar, int64_t n_cigar, const csv_sa_cols* sa,
                             const csv_seq_cols* seq, const csv_name_cols* names, void* stream, int64_t counts[CSV_NTYPES],
                             int64_t* n_read_rows);
int csv_extract_append_named_device(csv_ctx* ctx, const csv_read_cols* reads, const uint32_t* cigar, int64_t n_cigar,
                                    const csv_sa_cols* sa, const csv_seq_cols* seq, const csv_name_cols* names, void* stream,
                                    int64_t counts[CSV_NTYPES], int64_t* n_read_rows);
/* Sorts the names of a named accumulation byte-lexicographically (a proper prefix first, embedded NUL bytes included) on the
 * device, gives every record the dense rank of its name among the distinct names (*n_distinct, may be NULL) and rewrites the
 * read ids of all five signature types and of the reads table from provisional ids to ranks, with no host copy.  A second
 * call only reports the count.  CSV_E_STATE when the device-resident rows are not a named accumulation (or an upload came
 * since).  Its scratch is csv_sort_sigs' (never csv_cluster's inputs, results or captured graphs). */
int csv_rank_names(csv_ctx* ctx, int64_t* n_distinct);
/* Device pointer of the ranked accumulation's table record -> rank (int32, *n_records entries), e.g. to turn the provisional
 * ids of a caller-built alignment table (csv_upload_alignments_device) into ranks with one gather.  Blocks until the table is
 * complete; valid until the next extraction, csv_extract_reset or csv_destroy.  CSV_E_STATE before csv_rank_names. */
int csv_name_ranks_device_ptr(csv_ctx* ctx, const int32_t** rank_of_record, int64_t* n_records);
/* Names of ranks ranks[0..n) (any order, repeats allowed), gathered on the device, one D2H copy: rank ranks[i] is
 * out[out_off[i] .. out_off[i + 1]) (out_off: n + 1 entries, 64-bit).  On CSV_E_CAPACITY out_off is filled and out_off[n]
 * is the size `out` needs.  CSV_E_STATE before csv_rank_names, CSV_E_INVALID for a rank outside [0, n_distinct). */
int csv_fetch_names(csv_ctx* ctx, const int32_t* ranks, int64_t n, uint8_t* out, int64_t cap, int64_t* out_off);
/* Puts the INS rows that tie on (contig, int(pos), len, read) into the order of their sequence strings (cuteSV:774) on the
 * device, from the sequence arena: each tie group's contents, ordered by (sequence bytes, row), go onto the group's rows in
 * ascending order.  Moves everything csv_swap_ins_rows moves (and likewise invalidates the record column); the result equals
 * the host's swaps (cutesv_b200/cli.py ins_tie_swaps) applied with csv_swap_ins_rows.  *n_rows_moved (may be NULL): rows whose
 * content changed.
 *   - CSV_E_STATE without a valid sequence arena: ties then keep extraction order (as with --ignore_sequence).
 *   - The read ids must be final ranks.  For a named accumulation the call checks that csv_rank_names ran (CSV_E_STATE
 *     otherwise); for any other accumulation that is the caller's contract, met by csv_remap_read_ids. */
int csv_order_ins_ties(csv_ctx* ctx, int64_t* n_rows_moved);

/* ---- scanned packets: every decoded record, filtered on the device ----
 * A caller that decodes a BAM into GPU memory hands over every record of a packet in BAM order, with names; the library
 * applies the reference's record filter (single_pipe, cuteSV:697-733), the -include_bed test and builds the TRA genotyper's
 * all-alignments table on the device.
 *
 * Region table (the task windows and -include_bed regions of cutesv_b200/cli.py task_windows + load_bed), host arrays:
 *   - win_off: n_contigs + 1 offsets; the windows of contig id k are [win_off[k], win_off[k + 1]), their starts win_start[]
 *     (float64: the reference's bounds may be fractional, cuteSV:1026-1034) ascending;
 *   - reg_off: n_windows + 1 offsets (n_windows = win_off[n_contigs]); the padded regions of window w are the int64 (lo, hi)
 *     pairs reg[2k], reg[2k + 1] for k in [reg_off[w], reg_off[w + 1]) (lo may be negative).
 * n_contigs == 0 clears the table: no region filtering.  A record is kept iff, in its contig's last window starting at or
 * before its ref_start (compared as float64), some region has not (ref_end <= lo or ref_start >= hi).  With a table, a record
 * on a contig without a window is not extracted (the reference never fetches it).  CSV_E_INVALID for offsets that decrease or
 * starts that are not ascending; CSV_E_STATE, changing nothing, while a scanned accumulation is open (appended to and not
 * ranked). */
int csv_set_scan_regions(csv_ctx* ctx, int32_t n_contigs, const int64_t* win_off, const double* win_start, const int64_t* reg_off,
                         const int64_t* reg);
/* Appends one scanned packet: the columns of csv_extract_append_named_device (device memory, checked the same way, CSV_E_INPUT
 * changing nothing), but the packet holds every decoded record, in BAM order.
 *   - Alignment row: every record with cigar_off[i + 1] > cigar_off[i] and chrom >= 0, as (chrom, ref_start, ref_end,
 *     provisional id, is_primary = flag is 0 or 16), kept in a ctx-owned pending table, only when want_alignments != 0.
 *   - Extracted: an alignment row whose flag is neither 256 nor 272 (exact values, cuteSV:711) and that passes the region
 *     table.  The other records yield no signature and no reads row.
 *   - Every record's name joins the name arena, so csv_rank_names ranks the names of all decoded records.
 *   - Numbering: every per-record number refers to the record's index among all scanned records of the accumulation (the
 *     packets the caller holds): provisional ids, csv_name_ranks_device_ptr, csv_fetch_records and the record of an INS piece.
 *   - counts / n_read_rows as for csv_extract_append; *n_aln_rows (may be NULL): pending alignment rows so far.
 *   - CSV_E_STATE, changing nothing: a scanned packet appended to an accumulation of other packets or the reverse, packets
 *     that disagree on want_alignments, any append after csv_rank_names.  An upload of signatures, reads or alignments ends
 *     the scanned state.
 * csv_rank_names on a scanned accumulation that asked for alignments also turns the pending rows' ids into ranks, stable-sorts
 * the rows by contig id on the device and installs them as csv_cluster's alignment table, checked as csv_upload_alignments
 * checks a table: rows out of BAM order are CSV_E_INPUT, and the accumulation then stays unranked. */
int csv_scan_append_named_device(csv_ctx* ctx, const csv_read_cols* reads, const uint32_t* cigar, int64_t n_cigar, const csv_sa_cols* sa,
                                 const csv_seq_cols* seq, const csv_name_cols* names, int want_alignments, void* stream,
                                 int64_t counts[CSV_NTYPES], int64_t* n_read_rows, int64_t* n_aln_rows);
/* D2H of csv_cluster's alignment table, uploaded or installed by csv_rank_names (*n_rows: its row count, also on
 * CSV_E_CAPACITY); any column pointer may be NULL. */
int csv_fetch_alignments(csv_ctx* ctx, int64_t cap, int32_t* chrom, int32_t* start, int32_t* end, int32_t* read_id, uint8_t* is_primary,
                         int64_t* n_rows);

/* ---- SA:Z tags reduced on the device ----
 * The contig names of the csv_set_contigs table, host arrays: name k (contig id k) is names[name_off[k], name_off[k + 1]),
 * bytes without NUL.  n must equal the table's contig count; names must be non-empty and unique.  Anything else is
 * CSV_E_INVALID, changing nothing.  The library keeps them sorted bytewise on the device with their ids; a later
 * csv_set_contigs with another contig count drops them.  Ends the outputs of csv_reduce_sa_device. */
int csv_set_contig_names(csv_ctx* ctx, int32_t n, const uint8_t* names, const int64_t* name_off);

/* Record i's SA:Z value is text[text_off[i], text_off[i + 1]) (device memory): no tag prefix, no NUL terminator; an empty
 * range is a record without the tag. */
typedef struct csv_sa_text {
    int64_t n_records;
    int64_t n_bytes;
    const int64_t* text_off;   /* n_records + 1 */
    const uint8_t* text;
} csv_sa_text;
/* SA:Z text -> the SA table of a device packet: *sa_off (n_records + 1 entries, for csv_read_cols::sa_off) and *sa (the seven
 * columns, sa->n rows), ctx-owned device memory that csv_extract*_device and csv_scan_append_named_device take as they are.
 * Valid until the next csv_reduce_sa_device, csv_set_contig_names or csv_destroy; a call that fails leaves them as they were.
 * The reduction is that of the native BAM decoder (bam_reader.cpp): entries end at ';' (an entry without it is dropped with
 * everything after it), a NUL byte ends the value, entries of fewer than 5 comma-separated fields are skipped, an unknown
 * contig name gives contig -1, pos0 = atoi(pos) - 1, strand '+' -> 0 else 1, mapq = atoi(mapq), and the clips and span of
 * the CIGAR as acquire_clip_pos (cuteSV:466-481) computes them.  Ordered after the caller's work on `stream` (0: the legacy
 * default stream); the call returns when the outputs are complete.
 *   - CSV_E_STATE before csv_set_contig_names; CSV_E_INVALID for host memory or null pointers.
 *   - CSV_E_INPUT, changing nothing: text_off does not start at >= 0, decreases or ends past n_bytes (checked on the
 *     device); a position, mapq or CIGAR number (or span) whose value does not fit int32.
 *   - CSV_E_CAPACITY: 2^32 or more entries in one call. */
int csv_reduce_sa_device(csv_ctx* ctx, const csv_sa_text* text, void* stream, const int64_t** sa_off, csv_sa_cols* sa);

/* Records whose split-read analysis was skipped because they carry more than 64 qualifying segments (only reachable
 * with --max_split_parts -1; their CIGAR signatures are taken).  The reference has no such limit: a documented,
 * counted deviation instead of a failed run. */
int64_t csv_extract_skipped(csv_ctx* ctx);
/* read_id of every device-resident signature / reads-table row: id -> rank[id].  The CLI numbers read names in
 * first-seen order while it decodes and learns their ranks in Python string order at the end (cuteSV:764-801). */
int csv_remap_read_ids(csv_ctx* ctx, const int32_t* rank, int64_t n_rank);
/* Swap rows pairs[2k] <-> pairs[2k+1] of the device-resident INS signatures (columns, piece descriptors and, while it is
 * valid, the sequence arena's start and length), in
 * sequence.  INS rows that tie on (contig, int(pos), len, read) must be in the order of their sequence strings
 * (the reference's sort key ends with the sequence, cuteSV:774); the host, which owns the strings, fixes the few
 * ties of device-extracted rows with this call. */
int csv_swap_ins_rows(csv_ctx* ctx, const int64_t* pairs, int64_t n_pairs);
/* Slices [first, first + count) of the extracted columns of one type / of the piece table (append mode: the rows a
 * packet added). */
int csv_fetch_sigs_range(csv_ctx* ctx, int svtype, int64_t first, int64_t count, int32_t* chrom, int32_t* a, int32_t* b,
                         int32_t* read_id, int32_t* c, int32_t* piece_off, int32_t* piece_cnt);
int csv_fetch_pieces_range(csv_ctx* ctx, int64_t first, int64_t count, int32_t* pieces4);
/* on != 0: the following csv_extract* calls also store the record index of every row they emit, for csv_fetch_records
 * (4 B per row; default off, so an extraction that never asks for it pays nothing). */
int csv_extract_records(csv_ctx* ctx, int on);
/* Record index (position of the alignment record in the packet, plus the records of earlier packets of an append
 * accumulation) of device-resident rows [first, first + count) of one type, or of the reads table (svtype 5).  The kernel
 * hands out row slots with atomics, so rows come in no particular record order; but one thread emits all rows of a
 * record, so a stable sort of the rows by this column restores the reference's list order (records in input order,
 * inside a record the order in which parse_read appends, cuteSV:606-681, 729-733).  CSV_E_STATE when the device-resident
 * rows were not produced by csv_extract* calls made with csv_extract_records on (or an upload or csv_swap_ins_rows came
 * since). */
int csv_fetch_records(csv_ctx* ctx, int svtype, int64_t first, int64_t count, int32_t* rec);
/* D2H of the extracted signature columns of one type (parity tests, .sigs dumps, host ALT
 * strings).  piece_off / piece_cnt (INS only, may be NULL): slice of the piece table. */
int csv_fetch_sigs(csv_ctx* ctx, int svtype, int64_t cap, int32_t* chrom, int32_t* a, int32_t* b,
                   int32_t* read_id, int32_t* c, int32_t* piece_off, int32_t* piece_cnt);
/* Piece table: 4 int32 per piece = (record index, slice start, slice stop, reverse-complement flag),
 * Python slice semantics (negative indices allowed).  *n_pieces reports the table size.
 * flag == 2 marks a signature that merged more CIGAR insertions than the device buffers (64): `slice start` is then
 * the reference position of the merged group and the host rebuilds the string by walking that record's CIGAR
 * (cutesv_b200/packing.py merged_ins_from_cigar); position, length and len(seq) of the signature are complete. */
int csv_fetch_pieces(csv_ctx* ctx, int64_t cap, int32_t* pieces4, int64_t* n_pieces);
int csv_fetch_read_rows(csv_ctx* ctx, int64_t cap, int32_t* chrom, int32_t* start, int32_t* end,
                        int32_t* read_id, uint8_t* is_primary);

/* Profiling: per-stage device milliseconds of the last csv_cluster / csv_extract call.  on = 2: no per-launch events and
 * no graph replay, only one interval per INS / DEL lane that takes the density filter, from the filter's end to the
 * lane's end, reported by csv_kernel_times as "back end<DEL>" / "back end<INS>". */
int csv_set_profiling(csv_ctx* ctx, int on);
int csv_stage_ms(csv_ctx* ctx, float ms[CSV_ST_COUNT]);
/* Per-kernel totals of the last profiled call(s): with profiling on, every kernel launch sits between its own
 * pair of CUDA events on its launching stream; one text line per kernel, "name<TAB>launches<TAB>total_ms".
 * Returns the buffer size the text needs (incl. NUL). */
int64_t csv_kernel_times(csv_ctx* ctx, char* buf, int64_t cap);
/* SV types are independent until the final ordering (the reference runs them as separate Pool#3
 * tasks, cuteSV:1113-1199); by default each type's kernel chain runs on its own stream ("lane").
 * on = 0 serialises the types on the ctx stream, e.g. to time every kernel alone. */
int csv_set_lanes(csv_ctx* ctx, int on);
/* Number of kernels the library launched since the ctx was created (kernels inside a replayed CUDA graph count). */
int64_t csv_launch_count(csv_ctx* ctx);
/* csv_cluster calls served by replaying a captured CUDA graph.  A call whose inputs are already device resident
 * replays the graph of its (type_mask, sizes, params) from its third occurrence on; CUTESV_B200_GRAPHS=0 disables. */
int64_t csv_graph_replays(csv_ctx* ctx);

/* ---- multi-GPU: contigs sharded over ranks, one csv_ctx per GPU / process -------------------------------------
 * Every resolution_* call of the reference is keyed by (svtype, chr) and reads only that contig's signatures and
 * reads-table rows (cuteSV:1116-1189; resolveINDEL.py:52-54,445-447), so contigs are independent units: each rank
 * runs the whole pipeline on its contigs with no data-path collective, and ONE all-gather of the final
 * records assembles the result on every rank in the single-GPU order.  (The reference's Pool(threads).map_async
 * over (type, chr) tasks, cuteSV:1113-1199, is the CPU counterpart.) */

/* owned[k] != 0: contig k belongs to this ctx's shard (NULL = all).  Contigs outside the shard take no room in the
 * linear coordinate, so histogram / bin tables scale with the shard; a signature or reads-table row on such a
 * contig is an input error (CSV_E_INPUT).  Contig ids stay global.  Call after csv_set_contigs. */
int csv_set_shard(csv_ctx* ctx, const uint8_t* owned);
/* ncclGetUniqueId: rank 0 calls it and ships the bytes (>= 128) to the other ranks by any means. */
int csv_comm_unique_id(void* id, size_t bytes);
/* ncclCommInitRank on the ctx's device.  Collective: every rank calls it with the same id. */
int csv_comm_init(csv_ctx* ctx, const void* id, int rank, int world);
int csv_comm_destroy(csv_ctx* ctx);
/* After csv_cluster, asynchronous on the ctx stream, collective: packs this rank's records (csv_cand, csv_geno,
 * supporting read ids) into one padded message, gathers the messages of all ranks, then merges them on the device
 * into the single-GPU order (svtype, contig id, emission order).  The gather itself is either ONE ncclAllGather over
 * NVLink or (default when every rank could map every rank's mail box through CUDA IPC) ONE kernel that packs the
 * records straight into the peers' mail boxes over NVLink and releases an arrival flag (no staging copy); csv_set_gather(ctx, 0) or
 * CUTESV_B200_GATHER=nccl selects NCCL, csv_gather_mode() tells which one the last gather used (1 peer-to-peer).  csv_cand.reserved[1] of a
 * gathered record is its source rank (csv_cand.aux of an INS row indexes THAT rank's INS signatures).  The padded
 * message size is agreed once (first call: one count all-reduce) and re-agreed only when a rank outgrows it. */
int csv_allgather(csv_ctx* ctx);
int csv_set_gather(csv_ctx* ctx, int peer_to_peer);
int csv_gather_mode(csv_ctx* ctx);
/* Blocks until the gather finished; total sizes over all ranks. */
int csv_gathered_counts(csv_ctx* ctx, int64_t* n_cand, int64_t* n_names);
int csv_fetch_gathered(csv_ctx* ctx, csv_cand* cands, csv_geno* genos, int64_t cap_cand, int32_t* names, int64_t cap_names);
int csv_gathered_device_ptrs(csv_ctx* ctx, const csv_cand** cands, const csv_geno** genos, const int32_t** names);
/* Device counters of the last finished csv_cluster call, 32 words: [0] status, [1] candidates,
 * [2] names, [3] max support, [4..8] kept clusters per type, [9..13] CTA-class clusters,
 * [14..18] global-scratch-class clusters, [19] (read, window) pairs, [20..24] sorted-domain size per
 * type, [25..29] signatures inside kept clusters per type. */
int csv_debug_counters(csv_ctx* ctx, uint32_t out[32]);
/* Duration (ms) and element count of the last radix scatter pass launches (roofline probe). */
int csv_sort_probe(csv_ctx* ctx, float* ms_total, int64_t* bytes_total, int32_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* CUTESV_B200_H */
