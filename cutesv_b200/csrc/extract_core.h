// extract_core.h -- per-read signature extraction logic of cuteSV, host/device shared.
//
// Restates (not translates) parse_read / generate_combine_sigs / organize_split_signal /
// analysis_split_read / analysis_inv / analysis_bnd of the reference (cuteSV:50-681) on packed
// integer fields.  The CUDA kernel (extract.cuh) adds the warp-parallel CIGAR prefix scan; the
// test-only emulator walks the CIGAR serially.  Citations "cuteSV:N" = src/cuteSV/cuteSV line N.
//
// Every INS signature carries `seq_len` (what clustering needs, resolveINDEL.py:400) and a list of
// "pieces" = Python slices of the record's query sequence (or of its reverse complement) from which
// the host rebuilds the string; for packets with bases in GPU memory the routines at the end of this
// file build the same strings on the device.
#pragma once
#include "core.h"

namespace csv {

// BAM CIGAR op codes (pysam.CMATCH ..): M I D N S H P = X B
enum { OP_M = 0, OP_I = 1, OP_D = 2, OP_N = 3, OP_S = 4, OP_H = 5, OP_P = 6, OP_EQ = 7, OP_X = 8, OP_B = 9 };

CSV_HD bool op_ref_change(int op) { return op == OP_M || op == OP_D || op == OP_N || op == OP_EQ || op == OP_X; }  // cuteSV:592-603

// len(seq[a:b]) for a Python str of length L
CSV_HD int32_t py_slice_len(int64_t a, int64_t b, int64_t L) {
    if (a < 0) { a += L; if (a < 0) a = 0; } else if (a > L) a = L;
    if (b < 0) { b += L; if (b < 0) b = 0; } else if (b > L) b = L;
    return (int32_t)(b > a ? b - a : 0);
}

struct ExtractParams {
    int32_t min_size;          // SV_size
    int32_t max_size;          // MaxSize
    int32_t min_mapq, max_split_parts, min_read_len, min_siglength, merge_del_threshold, merge_ins_threshold;
};

// One INS sequence piece: Python slice [start:stop] of record `rec`'s query (rc != 0: of its
// reverse complement).  Pieces of one signature are consecutive in the piece buffer.
struct InsPiece { int32_t rec; int32_t start; int32_t stop; int32_t rc; };

// Output sink: append buffers in device (or host) memory.
struct ExtractOut {
    // signature columns per type: chrom, a, b, rid, c
    int32_t* col[CSV_NTYPES][5];
    uint32_t* n_sig;        // [CSV_NTYPES] counters
    uint32_t cap_sig[CSV_NTYPES];
    // INS piece descriptors: ins_piece_off[k], ins_piece_cnt[k] for INS signature k
    int32_t* ins_piece_off;
    int32_t* ins_piece_cnt;
    InsPiece* pieces;
    uint32_t* n_pieces;
    uint32_t cap_pieces;
    // reads rows
    int32_t* rr_chrom; int32_t* rr_start; int32_t* rr_end; int32_t* rr_id; uint8_t* rr_prim;
    uint32_t* n_rows;
    uint32_t cap_rows;
    uint32_t* status;       // ST_* bits (overflow)
    uint32_t* n_skipped;    // records whose split-read analysis was skipped (more than MAX_SEGS segments), may be null
    // record index (rec_base + packet index) of every signature / reads row, may be null.  One thread emits all rows of a
    // record, so inside one record and type the slot order is the emission order of parse_read (cuteSV:606-681)
    int32_t* rec_col[CSV_NTYPES];
    int32_t* rr_rec;
};

CSV_HD int64_t emit_sig(const ExtractOut& O, int t, int32_t chrom, int32_t a, int32_t b, int32_t rid, int32_t c, int32_t rec) {
    const uint32_t k = atomic_add_u32(&O.n_sig[t], 1u);
    if (k >= O.cap_sig[t]) { atomic_or_u32(O.status, ST_CAND_OVERFLOW); return -1; }
    O.col[t][0][k] = chrom; O.col[t][1][k] = a; O.col[t][2][k] = b; O.col[t][3][k] = rid;
    if (O.col[t][4]) O.col[t][4][k] = c;
    if (O.rec_col[t]) O.rec_col[t][k] = rec;
    return (int64_t)k;
}
// reserve n pieces; returns first index or -1
CSV_HD int64_t reserve_pieces(const ExtractOut& O, uint32_t n) {
    const uint32_t k = atomic_add_u32(O.n_pieces, n);
    if ((uint64_t)k + n > O.cap_pieces) { atomic_or_u32(O.status, ST_NAMES_OVERFLOW); return -1; }
    return (int64_t)k;
}
CSV_HD void emit_ins_single(const ExtractOut& O, int32_t chrom, int32_t pos2x, int32_t len, int32_t rid, int32_t rec, int64_t a,
                            int64_t b, int64_t L, int rc) {
    const int32_t sl = py_slice_len(a, b, L);
    const int64_t k = emit_sig(O, CSV_INS, chrom, pos2x, len, rid, sl, rec);
    if (k < 0) return;
    const int64_t p = reserve_pieces(O, 1);
    if (p < 0) { O.ins_piece_off[k] = 0; O.ins_piece_cnt[k] = 0; return; }
    InsPiece ip; ip.rec = rec; ip.start = (int32_t)a; ip.stop = (int32_t)b; ip.rc = rc;
    O.pieces[p] = ip;
    O.ins_piece_off[k] = (int32_t)p; O.ins_piece_cnt[k] = 1;
}

// ------------------------------------------------------------------------------------------
// generate_combine_sigs (cuteSV:515-575) as a streaming state machine: qualifying CIGAR ops
// arrive in read order; merged signatures are emitted as soon as they are complete.
// ------------------------------------------------------------------------------------------
struct MergeState {
    // INS
    int ins_open; int32_t ins_pos, ins_len, ins_seqlen, ins_last; int32_t ins_np;   // np: number of pieces so far
    // DEL
    int del_open; int32_t del_pos, del_len, del_cmp;
    CSV_HD void reset() { ins_open = 0; del_open = 0; ins_pos = ins_len = ins_seqlen = ins_last = ins_np = 0; del_pos = del_len = del_cmp = 0; }
};
static constexpr int MAX_OPEN_PIECES = 64;  // pieces buffered per open merged INS; longer chains are rebuilt on the host (flush_ins)

struct ReadCtx {
    int32_t rec, chrom, rid, qlen;
    int32_t base_rc;   // 1: the split-read engine works on the reverse complement of the stored query (flag 16, cuteSV:674-677)
};

CSV_HD void flush_ins(const ExtractOut& O, const ReadCtx& R, MergeState& S, const InsPiece* open_pieces) {
    if (!S.ins_open) return;
    const int64_t k = emit_sig(O, CSV_INS, R.chrom, 2 * S.ins_pos, S.ins_len, R.rid, S.ins_seqlen, R.rec);
    if (k >= 0) {
        // More merged insertions than the open-piece buffer holds (the reference has no limit, cuteSV:537-540): position, length
        // and len(seq) of the signature are complete; its piece list becomes ONE marker piece (rc == 2, start = reference
        // position of the merged group) from which the host rebuilds the string by walking that record's CIGAR again.
        const bool spill = S.ins_np > MAX_OPEN_PIECES;
        const int np = spill ? 1 : S.ins_np;
        const int64_t p = reserve_pieces(O, (uint32_t)np);
        if (p >= 0) {
            if (spill) { InsPiece mk; mk.rec = R.rec; mk.start = S.ins_pos; mk.stop = 0; mk.rc = 2; O.pieces[p] = mk; }
            else for (int i = 0; i < np; i++) O.pieces[p + i] = open_pieces[i];
            O.ins_piece_off[k] = (int32_t)p; O.ins_piece_cnt[k] = np;
        } else { O.ins_piece_off[k] = 0; O.ins_piece_cnt[k] = 0; }
    }
    S.ins_open = 0; S.ins_np = 0;
}
CSV_HD void flush_del(const ExtractOut& O, const ReadCtx& R, MergeState& S) {
    if (!S.del_open) return;
    emit_sig(O, CSV_DEL, R.chrom, S.del_pos, S.del_len, R.rid, 0, R.rec);
    S.del_open = 0;
}
// one qualifying insertion op: ref pos, length, query slice [qa, qb)
CSV_HD void push_ins(const ExtractOut& O, const ReadCtx& R, const ExtractParams& P, MergeState& S, InsPiece* open_pieces,
                     int32_t pos, int32_t len, int64_t qa, int64_t qb) {
    const int32_t sl = py_slice_len(qa, qb, R.qlen);
    InsPiece ip; ip.rec = R.rec; ip.start = (int32_t)qa; ip.stop = (int32_t)qb; ip.rc = 0;
    if (S.ins_open && pos - S.ins_last <= P.merge_ins_threshold) {  // cuteSV:537-540
        S.ins_len += len; S.ins_seqlen += sl; S.ins_last = pos;
        if (S.ins_np < MAX_OPEN_PIECES) open_pieces[S.ins_np] = ip;
        S.ins_np++;
        return;
    }
    flush_ins(O, R, S, open_pieces);
    S.ins_open = 1; S.ins_pos = pos; S.ins_len = len; S.ins_seqlen = sl; S.ins_last = pos; S.ins_np = 1;
    open_pieces[0] = ip;
}
CSV_HD void push_del(const ExtractOut& O, const ReadCtx& R, const ExtractParams& P, MergeState& S, int32_t pos, int32_t len) {
    if (S.del_open && pos - S.del_cmp <= P.merge_del_threshold) {  // cuteSV:560-562
        S.del_len += len; S.del_cmp = pos + len;
        return;
    }
    const int was_open = S.del_open;
    flush_del(O, R, S);
    S.del_open = 1; S.del_pos = pos; S.del_len = len;
    // the very first signature compares against its END (sum(sigs[0]), :557); after a flush the
    // comparator is reset to the new signature's START (temp_sig.append(i[0]), :569-570)
    S.del_cmp = was_open ? pos : pos + len;
}

// ------------------------------------------------------------------------------------------
// split-read engine: analysis_split_read (cuteSV:190-464)
// ------------------------------------------------------------------------------------------
struct Seg { int32_t rs, re, fs, fe, chr, strand; };  // read_start, read_end, ref_start, ref_end, chr id, 0 '+' / 1 '-'
static constexpr int MAX_SEGS = 64;

CSV_HD Seg seg_flip(const Seg& x, int32_t RL) { Seg y = x; y.rs = RL - x.re; y.re = RL - x.rs; return y; }  // cuteSV:220-221
CSV_HD double dmax(double a, double b) { return a > b ? a : b; }   // Python max(int, float): values compare numerically

struct SplitCtx {
    const ExtractOut* O; ReadCtx R; ExtractParams P;
};

CSV_HD void analysis_inv(const SplitCtx& C, const Seg& e1, const Seg& e2) {  // cuteSV:50-94
    const int32_t sv = C.P.min_size;
    if (e1.strand == 0) {
        if (e1.fe - e2.fe >= sv)
            if ((double)e2.rs + 0.5 * (double)(e1.fe - e2.fe) >= (double)e1.re) emit_sig(*C.O, CSV_INV, e1.chr, e2.fe, e1.fe, C.R.rid, 0, C.R.rec);
        if (e2.fe - e1.fe >= sv)
            if ((double)e2.rs + 0.5 * (double)(e2.fe - e1.fe) >= (double)e1.re) emit_sig(*C.O, CSV_INV, e1.chr, e1.fe, e2.fe, C.R.rid, 0, C.R.rec);
    } else {
        if (e2.fs - e1.fs >= sv)
            if ((double)e2.rs + 0.5 * (double)(e2.fs - e1.fs) >= (double)e1.re) emit_sig(*C.O, CSV_INV, e1.chr, e1.fs, e2.fs, C.R.rid, 1, C.R.rec);
        if (e1.fs - e2.fs >= sv)
            if ((double)e2.rs + 0.5 * (double)(e1.fs - e2.fs) >= (double)e1.re) emit_sig(*C.O, CSV_INV, e1.chr, e2.fs, e1.fs, C.R.rid, 1, C.R.rec);
    }
}

// TRA signature: (type, pos1, chr2, pos2) tagged with chr1; c = chr2*4 + type
CSV_HD void emit_tra(const SplitCtx& C, int type, int32_t pos1, int32_t chr2, int32_t pos2, int32_t chr1) {
    emit_sig(*C.O, CSV_TRA, chr1, pos1, pos2, C.R.rid, chr2 * 4 + type, C.R.rec);
}
CSV_HD void analysis_bnd(const SplitCtx& C, const Seg& e1, const Seg& e2) {  // cuteSV:97-188
    if (!(e2.rs - e1.re <= 100)) return;
    const bool lt = e1.chr < e2.chr;  // string compare of contig names == compare of rank ids
    if (e1.strand == 0) {
        if (e2.strand == 0) {
            if (lt) emit_tra(C, 0, e1.fe, e2.chr, e2.fs, e1.chr); else emit_tra(C, 3, e2.fs, e1.chr, e1.fe, e2.chr);
        } else {
            if (lt) emit_tra(C, 1, e1.fe, e2.chr, e2.fe, e1.chr); else emit_tra(C, 1, e2.fe, e1.chr, e1.fe, e2.chr);
        }
    } else {
        if (e2.strand == 0) {
            if (lt) emit_tra(C, 2, e1.fs, e2.chr, e2.fs, e1.chr); else emit_tra(C, 2, e2.fs, e1.chr, e1.fs, e2.chr);
        } else {
            if (lt) emit_tra(C, 3, e1.fs, e2.chr, e2.fe, e1.chr); else emit_tra(C, 0, e2.fe, e1.chr, e1.fs, e2.chr);
        }
    }
}

CSV_HD bool size_ok(const SplitCtx& C, int64_t d) { return d <= C.P.max_size || C.P.max_size == -1; }
CSV_HD int64_t trunc_half(int64_t x) { return (int64_t)((double)x / 2.0); }  // int(x/2): toward zero

// "INSpair": cuteSV:241-249 / 358-367 / 382-390 / 412-420
CSV_HD void ins_pair(const SplitCtx& C, const Seg& e1, const Seg& e2, int rc, bool gate) {
    const int64_t delta = (int64_t)e2.rs + e1.fe - e2.fs - e1.re;
    if ((double)(e1.fe - e2.fs) < dmax((double)C.P.min_size, (double)delta / 5.0) && delta >= C.P.min_size)
        if ((double)(e2.fs - e1.fe) <= dmax(100.0, (double)delta / 5.0) && size_ok(C, delta))
            if (gate) {
                const int64_t h = trunc_half((int64_t)e2.fs - e1.fe);
                emit_ins_single(*C.O, e2.chr, e2.fs + e1.fe, (int32_t)delta, C.R.rid, C.R.rec, (int64_t)e1.re + h, (int64_t)e2.rs - h,
                                C.R.qlen, rc ^ C.R.base_rc);
            }
}
// "DELpair": cuteSV:250-257 / 368-376 / 392-399 / 422-429
CSV_HD void del_pair(const SplitCtx& C, const Seg& e1, const Seg& e2, bool gate) {
    const int64_t delta = (int64_t)e2.fs - e2.rs + e1.re - e1.fe;
    if ((double)(e1.fe - e2.fs) < dmax((double)C.P.min_size, (double)delta / 5.0) && delta >= C.P.min_size)
        if ((double)(e2.rs - e1.re) <= dmax(100.0, (double)delta / 5.0) && size_ok(C, delta))
            if (gate) emit_sig(*C.O, CSV_DEL, e2.chr, e1.fe, (int32_t)delta, C.R.rid, 0, C.R.rec);
}

// segs[0..n): in insertion order (primary first, then SA entries); sorted here by read_start (stable)
CSV_HD void analysis_split_read(const SplitCtx& C, Seg* sp, int n) {
    const int32_t RL = C.R.qlen;
    const int32_t sv = C.P.min_size;
    for (int i = 1; i < n; i++) {  // stable insertion sort by read_start (cuteSV:195)
        Seg x = sp[i];
        int j = i - 1;
        while (j >= 0 && sp[j].rs > x.rs) { sp[j + 1] = sp[j]; j--; }
        sp[j + 1] = x;
    }
    int trigger = 0;
    if (n == 2) {  // cuteSV:205-259
        Seg e1 = sp[0], e2 = sp[1];
        if (e1.chr == e2.chr) {
            if (e1.strand != e2.strand) analysis_inv(C, e1, e2);
            else {
                int rc = 0;
                if (e1.strand == 1) { e1 = seg_flip(sp[1], RL); e2 = seg_flip(sp[0], RL); rc = 1; }
                if (e1.fe - e2.fs >= sv) {  // :225-239
                    if (e2.rs - e1.re >= e1.fe - e2.fs) {
                        const int64_t h = trunc_half((int64_t)e2.fs - e1.fe);
                        emit_ins_single(*C.O, e2.chr, e1.fe + e2.fs, e2.rs + e1.fe - e2.fs - e1.re, C.R.rid, C.R.rec, (int64_t)e1.re + h,
                                        (int64_t)e2.rs - h, RL, rc ^ C.R.base_rc);
                    } else emit_sig(*C.O, CSV_DUP, e2.chr, e2.fs, e1.fe, C.R.rid, 0, C.R.rec);
                }
                ins_pair(C, e1, e2, rc, true);
                del_pair(C, e1, e2, true);
            }
        } else analysis_bnd(C, e1, e2);
    } else if (n >= 3) {  // cuteSV:261-437
        for (int a = 0; a + 2 < n; a++) {
            Seg e1 = sp[a], e2 = sp[a + 1], e3 = sp[a + 2];
            const bool last = (n - 3 == a);
            bool e3_none = false;
            if (e1.chr == e2.chr) {
                if (e2.chr == e3.chr) {
                    if (e1.strand == e3.strand && e1.strand != e2.strand) {  // :270-314
                        if (e2.strand == 1) {  // +-+
                            const double half = 0.5 * (double)(e3.fs - e1.fe);
                            if ((double)e2.rs + half >= (double)e1.re && (double)e3.rs + half >= (double)e2.re)
                                if (e2.fs >= e1.fe && e3.fs >= e2.fe) {
                                    emit_sig(*C.O, CSV_INV, e1.chr, e1.fe, e2.fe, C.R.rid, 0, C.R.rec);
                                    emit_sig(*C.O, CSV_INV, e1.chr, e2.fs, e3.fs, C.R.rid, 1, C.R.rec);
                                }
                        } else {  // -+-
                            const double half = 0.5 * (double)(e1.fs - e3.fe);
                            if ((double)e1.re <= (double)e2.rs + half && (double)e3.rs + half >= (double)e2.re)
                                if (e2.fs - e3.fe >= -50 && e1.fs - e2.fe >= -50) {
                                    emit_sig(*C.O, CSV_INV, e1.chr, e3.fe, e2.fe, C.R.rid, 0, C.R.rec);
                                    emit_sig(*C.O, CSV_INV, e1.chr, e2.fs, e1.fs, C.R.rid, 1, C.R.rec);
                                }
                        }
                    }
                    if (last) {  // :316-331
                        if (e1.strand != e3.strand) {
                            if (e2.strand == e1.strand) analysis_inv(C, e2, e3); else analysis_inv(C, e1, e2);
                        }
                    }
                    int rc = 0;
                    if (e1.strand == e3.strand && e1.strand == e2.strand) {  // :333-399
                        if (e1.strand == 1) {
                            e1 = seg_flip(sp[a + 2], RL); e2 = seg_flip(sp[a + 1], RL); e3 = seg_flip(sp[a], RL); rc = 1;
                        }
                        if (e2.fe - e3.fs >= sv && e2.fs < e3.fe) emit_sig(*C.O, CSV_DUP, e2.chr, e3.fs, e2.fe, C.R.rid, 0, C.R.rec);
                        if (a == 0)
                            if (e1.fe - e2.fs >= sv) emit_sig(*C.O, CSV_DUP, e2.chr, e2.fs, e1.fe, C.R.rid, 0, C.R.rec);
                        const bool gate = e3.fs >= e2.fe;
                        ins_pair(C, e1, e2, rc, gate);
                        del_pair(C, e1, e2, gate);
                        if (last) {
                            e1 = e2; e2 = e3;
                            ins_pair(C, e1, e2, rc, true);
                            del_pair(C, e1, e2, true);
                        }
                    }
                    // :401-429 (evaluated on the possibly re-assigned e1, e2, e3)
                    if (last && e1.strand != e2.strand && e2.strand == e3.strand) { e1 = e2; e2 = e3; e3_none = true; }
                    if (e3_none || (e1.strand == e2.strand && e2.strand != e3.strand)) {
                        int rc2 = 0;
                        if (e1.strand == 1) {  // quirk: indices a+1, a even after the shift (:406-408)
                            e1 = seg_flip(sp[a + 1], RL); e2 = seg_flip(sp[a], RL); rc2 = 1;
                        }
                        ins_pair(C, e1, e2, rc2, true);
                        del_pair(C, e1, e2, true);
                    }
                }
            } else {  // :431-437
                trigger = 1;
                analysis_bnd(C, e1, e2);
                if (last && e2.chr != e3.chr) analysis_bnd(C, e2, e3);
            }
        }
    }
    if (n >= 3 && trigger == 1) {  // cuteSV:439-464
        const Seg& f = sp[0];
        const Seg& l = sp[n - 1];
        if (f.chr == l.chr && f.strand == l.strand) {
            Seg e1, e2;
            int rc = 0;
            if (f.strand == 0) { e1 = f; e2 = l; }
            else { e1 = seg_flip(l, RL); e2 = seg_flip(f, RL); rc = 1; }
            const int64_t dis_ref = (int64_t)e2.fs - e1.fe, dis_read = (int64_t)e2.rs - e1.re;
            const int64_t d = dis_read - dis_ref;
            const double adr = (double)(dis_ref < 0 ? -dis_ref : dis_ref);
            if (adr < dmax((double)sv, (double)d / 5.0) && d >= sv && size_ok(C, d)) {
                const int64_t h = trunc_half(dis_ref);
                const int32_t pos = e2.fs < e1.fe ? e2.fs : e1.fe;
                emit_ins_single(*C.O, e2.chr, 2 * pos, (int32_t)d, C.R.rid, C.R.rec, (int64_t)e1.re + h, (int64_t)e2.rs - h, RL,
                                rc ^ C.R.base_rc);
            }
            if (dis_ref <= -(int64_t)sv) emit_sig(*C.O, CSV_DUP, e2.chr, e2.fs, e1.fe, C.R.rid, 0, C.R.rec);
        }
    }
}

// organize_split_signal (cuteSV:483-513).  has_primary: primary_info non-empty (mapq passed).
struct SaView { const int32_t *chrom, *pos0, *strand, *mapq, *first_clip, *last_clip, *ref_span; };
CSV_HD void organize_split_signal(const SplitCtx& C, bool has_primary, const Seg& primary, const SaView& sa, int64_t sa_lo, int64_t sa_hi) {
    Seg segs[MAX_SEGS];
    int n = 0;
    int32_t min_mapq = C.P.min_mapq;
    if (has_primary) { segs[n++] = primary; min_mapq = 0; }
    int64_t total = n;
    for (int64_t i = sa_lo; i < sa_hi; i++) {
        if (sa.mapq[i] >= min_mapq) {
            total++;
            if (n < MAX_SEGS) {
                Seg s;
                if (sa.strand[i] == 0) { s.rs = sa.first_clip[i]; s.re = C.R.qlen - sa.last_clip[i]; }
                else { s.rs = sa.last_clip[i]; s.re = C.R.qlen - sa.first_clip[i]; }
                s.fs = sa.pos0[i]; s.fe = sa.pos0[i] + sa.ref_span[i]; s.chr = sa.chrom[i]; s.strand = sa.strand[i];
                segs[n++] = s;
            }
        }
    }
    if (total <= C.P.max_split_parts || C.P.max_split_parts == -1) {
        // only reachable with --max_split_parts -1: a record with more than MAX_SEGS qualifying segments is not analysed for
        // split signatures (its CIGAR signatures are taken); reported, not fatal (ST_SKIPPED, ExtractOut::n_skipped)
        if (total > MAX_SEGS) { atomic_or_u32(C.O->status, ST_SKIPPED); if (C.O->n_skipped) atomic_add_u32(C.O->n_skipped, 1u); return; }
        analysis_split_read(C, segs, n);
    }
}

// detect_flag (cuteSV:34-48): 1 forward primary (flag 0), 2 reverse primary (flag 16), else no SA analysis
CSV_HD int detect_flag(int32_t flag) { return flag == 0 ? 1 : flag == 16 ? 2 : 0; }

// ------------------------------------------------------------------------------------------
// INS sequences built from BAM's 4-bit packed query (csv_extract_device with a csv_seq_cols): the same strings the host
// builds from the piece list (cutesv_b200/packing.py ins_sequence / ins_block_from_packed), byte for byte.
// ------------------------------------------------------------------------------------------
// One record's packed bases: query_len bases from byte `seq4`, high nibble first.  have == false: BAM '*' (fewer than
// (query_len + 1) / 2 bytes stored), every slice of it is empty.
struct SeqRec { const uint8_t* seq4; int32_t qlen; bool have; };

CSV_HD uint8_t seq_base(const SeqRec& s, int64_t j) {   // ASCII of query base j (0 <= j < qlen)
    const uint8_t b = s.seq4[j >> 1];
    return (uint8_t)"=ACMGRSVTWYHKDBN"[(j & 1) ? (b & 15) : (b >> 4)];
}
CSV_HD uint8_t seq_comp(uint8_t c) {   // packing._COMP: only ACGTN / acgtn are complemented, every other code is kept
    switch (c) {
        case 'A': return 'T'; case 'C': return 'G'; case 'G': return 'C'; case 'T': return 'A'; case 'N': return 'N';
        case 'a': return 't'; case 'c': return 'g'; case 'g': return 'c'; case 't': return 'a'; case 'n': return 'n';
        default: return c;
    }
}
// Python slice [a:b] of a string of length L -> [lo, lo + len)
CSV_HD void py_slice(int64_t a, int64_t b, int64_t L, int64_t* lo, int64_t* len) {
    if (a < 0) { a += L; if (a < 0) a = 0; } else if (a > L) a = L;
    if (b < 0) { b += L; if (b < 0) b = 0; } else if (b > L) b = L;
    *lo = a;
    *len = b > a ? b - a : 0;
}
// Bytes of piece (a, b, rc in {0, 1}): q[a:b], or revcomp(q)[a:b].  out == nullptr: length only.  Writes lanes
// lane, lane + step, ... of the piece (step 1: all of it).
CSV_HD int64_t ins_piece_bytes(const SeqRec& s, int32_t a, int32_t b, int32_t rc, uint8_t* out, int lane, int step) {
    if (!s.have) return 0;
    int64_t lo, len;
    py_slice(a, b, s.qlen, &lo, &len);
    if (out)
        for (int64_t i = lane; i < len; i += step)
            out[i] = rc ? seq_comp(seq_base(s, (int64_t)s.qlen - 1 - (lo + i))) : seq_base(s, lo + i);
    return len;
}
// csv_fetch_ins_seqs: out_off[i] = start of the i-th requested row's string in the output (n + 1 entries), summed in 64 bits,
// since the rows may repeat and span the whole accumulation.  Returns the total.
CSV_HD int64_t ins_fetch_offsets(const int32_t* len, int64_t n, int64_t* out_off) {
    int64_t o = 0;
    for (int64_t i = 0; i < n; i++) { out_off[i] = o; o += len[i]; }
    out_off[n] = o;
    return o;
}
// Marker piece (rc == 2): the merged insertion that starts at reference position `pos`, rebuilt by the CIGAR walk of
// packing.merged_ins_from_cigar (parse_read's walk, cuteSV:616-645, and generate_combine_sigs' INS chain, cuteSV:530-545).
// Returns the string's length (out == nullptr: length only), -1 when no merged group starts at `pos`.
CSV_HD int64_t ins_marker_bytes(const SeqRec& s, const uint32_t* cigar, int64_t n_ops, int32_t ref_start, int32_t pos,
                                int32_t min_siglength, int32_t merge_ins_threshold, uint8_t* out) {
    int64_t ref = ref_start;
    int64_t q = (n_ops > 0 && (cigar[0] & 15) == OP_H) ? -(int64_t)(cigar[0] >> 4) : 0;   // shift_ins_read starts at -hardclip_left
    bool open = false, target = false;
    int64_t last = 0, written = 0;
    for (int64_t k = 0; k < n_ops; k++) {
        const int op = (int)(cigar[k] & 15);
        const int64_t ln = (int64_t)(cigar[k] >> 4);
        if (op != OP_D) q += ln;   // every op but D advances the query cursor (cuteSV:631-632)
        if (ln >= min_siglength && (op == OP_I || op == OP_D)) {
            if (op == OP_D) { ref += ln; continue; }
            if (open && ref - last <= merge_ins_threshold) last = ref;   // joins the open group
            else {
                if (target) break;   // the group starting at pos is complete
                open = true; last = ref; target = ref == pos;
            }
            if (target) written += ins_piece_bytes(s, (int32_t)(q - ln), (int32_t)q, 0, out ? out + written : nullptr, 0, 1);
        } else if (op_ref_change(op)) ref += ln;
    }
    return target ? written : -1;
}

}  // namespace csv
