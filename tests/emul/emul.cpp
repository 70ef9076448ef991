// emul.cpp -- TEST-ONLY single-threaded emulation of the GPU pipeline.
//
// Runs the exact per-cluster templates of cutesv_b200/csrc/core.h with a one-thread "team" and
// host stand-ins (std::stable_sort, loops) for the device-wide primitives, so that the logic of
// the kernels can be checked against the oracle without a GPU.  Never part of the product:
// libcutesv_b200.so has no host compute path.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <vector>

#include "../../cutesv_b200/csrc/core.h"
#include "../../cutesv_b200/csrc/host_tables.h"

using namespace csv;

namespace {

struct Ctx {
    const csv_params* P;
    int32_t n_contigs;
    std::vector<uint64_t> off;  // linear offsets, padded
    std::vector<csv_cand> cand_tmp;
    std::vector<int32_t> names;
    std::vector<uint32_t> cnt;
    std::vector<uint32_t> kept_type, kept_base;
    Counters ctr;
    std::vector<double> pow_half;
    std::vector<csv_geno> gl;
};

int64_t max_bias(const csv_params* P) {
    int64_t b = std::max<int64_t>({P->bias_del, P->bias_ins, P->bias_inv, P->bias_dup, P->bias_tra, P->gt_bias_ins});
    return b + 1;
}

Emit make_emit(Ctx& c) {
    Emit E;
    E.cand = c.cand_tmp.data(); E.names = c.names.data(); E.cnt = c.cnt.data(); E.ctr = &c.ctr;
    E.pow_half = c.pow_half.data();
    E.lim.cap_cand = (uint32_t)c.cand_tmp.size(); E.lim.cap_names = (uint32_t)c.names.size();
    E.lim.pow_n = (uint32_t)c.pow_half.size();
    E.cursor = nullptr;
    return E;
}

ClusterParams cluster_params(const csv_params* P, int t) {
    ClusterParams C;
    C.min_support = P->min_support; C.min_support_allele = P->min_support_allele;
    C.min_size = P->min_size; C.max_size = P->max_size;
    C.bias = t == CSV_DEL ? P->bias_del : t == CSV_INS ? P->bias_ins : t == CSV_INV ? P->bias_inv : t == CSV_DUP ? P->bias_dup : P->bias_tra;
    C.ratio = t == CSV_DEL ? P->ratio_del : t == CSV_INS ? P->ratio_ins : P->ratio_tra;
    C.keep = P->remain_reads_ratio > 1 ? 1 : P->remain_reads_ratio;
    C.genotype = P->genotype;
    return C;
}

void run_indel(Ctx& cx, const csv_sig_cols& S, int t, uint32_t& kslot) {
    const int64_t n = S.n;
    if (n == 0) return;
    const int is_ins = t == CSV_INS;
    std::vector<uint64_t> key(n);
    for (int64_t i = 0; i < n; i++) key[i] = cx.off[S.chrom[i]] + (uint64_t)(is_ins ? (S.a[i] >> 1) : S.a[i]);
    std::vector<uint32_t> sidx(n);
    std::iota(sidx.begin(), sidx.end(), 0u);
    std::stable_sort(sidx.begin(), sidx.end(), [&](uint32_t x, uint32_t y) { return key[x] < key[y]; });
    ClusterParams C = cluster_params(cx.P, t);
    IndelView V{S.chrom, S.a, S.b, S.read_id, S.c, sidx.data(), is_ins, nullptr, nullptr};
    Emit E = make_emit(cx);
    std::vector<char> arena;
    int64_t red[8];
    HostTeam tm;
    for (int64_t lo = 0; lo < n;) {
        int64_t hi = lo + 1;
        while (hi < n && !(key[sidx[hi]] - key[sidx[hi - 1]] > (uint64_t)C.bias)) hi++;
        if (hi - lo >= C.min_support) {
            int m = (int)(hi - lo), M = pow2ceil(m);
            arena.assign((size_t)INDEL_ARENA_PER * M + 64, 0);
            indel_cluster(tm, V, lo, m, M, arena.data(), red, C, t, kslot, E);
            kslot++;
        }
        lo = hi;
    }
}

void run_other(Ctx& cx, const csv_sig_cols& S, int t, uint32_t& kslot) {
    const int64_t n = S.n;
    if (n == 0) return;
    // full reference order (cuteSV:783-802) + exact-duplicate removal (cuteSV:958-969)
    std::vector<uint32_t> o(n);
    std::iota(o.begin(), o.end(), 0u);
    auto c_of = [&](uint32_t i) { return S.c ? S.c[i] : 0; };
    std::stable_sort(o.begin(), o.end(), [&](uint32_t x, uint32_t y) {
        if (S.chrom[x] != S.chrom[y]) return S.chrom[x] < S.chrom[y];
        if (t != CSV_DUP && c_of(x) != c_of(y)) return c_of(x) < c_of(y);
        if (S.a[x] != S.a[y]) return S.a[x] < S.a[y];
        if (S.b[x] != S.b[y]) return S.b[x] < S.b[y];
        return S.read_id[x] < S.read_id[y];
    });
    std::vector<int32_t> ch, a, b, rid, c;
    for (int64_t i = 0; i < n; i++) {
        uint32_t x = o[i];
        if (i > 0) {
            uint32_t y = o[i - 1];
            if (S.chrom[x] == S.chrom[y] && S.a[x] == S.a[y] && S.b[x] == S.b[y] && S.read_id[x] == S.read_id[y] && c_of(x) == c_of(y)) continue;
        }
        ch.push_back(S.chrom[x]); a.push_back(S.a[x]); b.push_back(S.b[x]); rid.push_back(S.read_id[x]); c.push_back(c_of(x));
    }
    const int64_t nu = (int64_t)ch.size();
    SortedView V{ch.data(), a.data(), b.data(), rid.data(), c.data()};
    ClusterParams C = cluster_params(cx.P, t);
    Emit E = make_emit(cx);
    std::vector<char> arena;
    int64_t red[8];
    HostTeam tm;
    for (int64_t lo = 0; lo < nu;) {
        int64_t hi = lo + 1;
        for (; hi < nu; hi++) {
            bool brk = ch[hi] != ch[hi - 1] || a[hi] - a[hi - 1] > C.bias;
            if (t == CSV_INV) brk = brk || b[hi] - b[hi - 1] > C.bias || c[hi] != c[hi - 1];
            if (t == CSV_TRA) brk = brk || c[hi] != c[hi - 1];
            if (brk) break;
        }
        if (hi - lo >= C.min_support) {
            int m = (int)(hi - lo), M = pow2ceil(m);
            arena.assign((size_t)OTHER_ARENA_PER * M + 64, 0);
            if (t == CSV_DUP) dup_cluster(tm, V, lo, m, M, arena.data(), red, C, kslot, E);
            else if (t == CSV_INV) inv_cluster(tm, V, lo, m, M, arena.data(), red, C, kslot, E);
            else tra_cluster(tm, V, lo, m, M, arena.data(), red, C, kslot, E);
            kslot++;
        }
        lo = hi;
    }
}

}  // namespace

extern "C" int emul_cluster(const csv_params* P, int32_t n_contigs, const int64_t* contig_len, const csv_sig_cols sigs[CSV_NTYPES],
                            const csv_reads_cols* reads, uint32_t type_mask, csv_cand* cands, csv_geno* genos, int64_t cap_cand,
                            int32_t* names, int64_t cap_names, int64_t* n_cand, int64_t* n_names, const csv_reads_cols* aln) {
    Ctx cx;
    cx.P = P; cx.n_contigs = n_contigs;
    cx.off.resize(n_contigs + 1);
    uint64_t run = 0;
    const int64_t pad = max_bias(P);
    for (int i = 0; i < n_contigs; i++) { cx.off[i] = run; run += (uint64_t)contig_len[i] + pad; }
    cx.off[n_contigs] = run;
    int64_t total = 0;
    for (int t = 0; t < CSV_NTYPES; t++) total += sigs[t].n;
    cx.cand_tmp.resize(total + 1); cx.names.resize(total + 1); cx.cnt.assign(total + 1, 0);
    memset(&cx.ctr, 0, sizeof(cx.ctr));
    cx.pow_half = build_pow_half(1u << 16);
    cx.gl = build_gl_table();
    uint32_t kslot = 0;
    for (int t = 0; t < CSV_NTYPES; t++) {
        if (!(type_mask >> t & 1)) continue;
        if (t == CSV_DEL || t == CSV_INS) run_indel(cx, sigs[t], t, kslot);
        else run_other(cx, sigs[t], t, kslot);
    }
    if (cx.ctr.status) { fprintf(stderr, "emul: status %u\n", cx.ctr.status); return CSV_E_INPUT; }
    // order: kslot-major, then emission rank (stored in reserved[0])
    const uint32_t nc = cx.ctr.n_cand;
    std::vector<uint32_t> base(kslot + 1, 0);
    for (uint32_t k = 0; k < kslot; k++) base[k + 1] = base[k] + cx.cnt[k];
    *n_cand = nc; *n_names = cx.ctr.n_names;
    if (base[kslot] != nc) { fprintf(stderr, "emul: count mismatch %u vs %u\n", base[kslot], nc); return CSV_E_STATE; }
    if ((int64_t)nc > cap_cand || (int64_t)cx.ctr.n_names > cap_names) return CSV_E_CAPACITY;
    for (uint32_t i = 0; i < nc; i++) {
        const csv_cand& c = cx.cand_tmp[i];
        cands[base[c.cluster] + c.reserved[0]] = c;
    }
    memcpy(names, cx.names.data(), sizeof(int32_t) * cx.ctr.n_names);
    // genotype: binned windows, one pass over the reads (mirrors the kernels)
    GtParams G{P->bias_del, P->gt_bias_ins, P->bias_dup, P->bias_inv};
    std::vector<uint32_t> dr(nc, 0);
    std::vector<uint8_t> has_rows(n_contigs, 0);
    for (uint32_t i = 0; i < nc; i++) {
        csv_geno g; g.dr = -1; g.dv = cands[i].names_cnt; g.gt = -1; g.pl[0] = g.pl[1] = g.pl[2] = 0; g.gq = 0; g.status = 1; g.qual = 0;
        genos[i] = g;
    }
    if (P->genotype) {
        const int shift = 12;
        const uint64_t nb = (cx.off[n_contigs] >> shift) + 2;
        std::vector<uint32_t> bstart(nb + 1, 0);
        struct W { uint32_t cand, which; };
        std::vector<std::pair<uint64_t, W>> wl;
        for (uint32_t i = 0; i < nc; i++) {
            int nw = n_windows_of(cands[i]);
            for (int w = 0; w < nw; w++) {
                int64_t s, e; window_of(cands[i], w, G, &s, &e);
                wl.push_back({(cx.off[cands[i].chrom] + (uint64_t)s) >> shift, W{i, (uint32_t)w}});
            }
        }
        for (auto& x : wl) bstart[x.first + 1]++;
        for (uint64_t b = 0; b < nb; b++) bstart[b + 1] += bstart[b];
        std::vector<W> wsorted(wl.size());
        std::vector<uint32_t> fill(nb, 0);
        for (auto& x : wl) wsorted[bstart[x.first] + fill[x.first]++] = x.second;
        for (int64_t r = 0; reads && r < reads->n; r++) {
            if (reads->start[r] < 0 || reads->end[r] < reads->start[r]) { fprintf(stderr, "emul: reads row %lld: end < start\n", (long long)r); return CSV_E_INPUT; }
            has_rows[reads->chrom[r]] = 1;
            if (!reads->is_primary[r]) continue;
            // the row's end clamped to the last linear coordinate of its contig (k_reads_pass)
            const uint64_t RS = cx.off[reads->chrom[r]] + (uint64_t)reads->start[r];
            const uint64_t RE = std::min(cx.off[reads->chrom[r]] + (uint64_t)reads->end[r], cx.off[reads->chrom[r] + 1] - 1);
            for (uint64_t b = RS >> shift; b <= (RE >> shift) && b < nb; b++)
                for (uint32_t w = bstart[b]; w < bstart[b + 1]; w++) {
                    const csv_cand& c = cands[wsorted[w].cand];
                    int64_t s, e; window_of(c, wsorted[w].which, G, &s, &e);
                    const uint64_t S = cx.off[c.chrom] + (uint64_t)s, Ee = cx.off[c.chrom] + (uint64_t)e;
                    if (!(RS <= S && RE >= Ee)) continue;
                    if (wsorted[w].which == 1) {  // union of the two covers: count once
                        int64_t s0, e0; window_of(c, 0, G, &s0, &e0);
                        if (RS <= cx.off[c.chrom] + (uint64_t)s0 && RE >= cx.off[c.chrom] + (uint64_t)e0) continue;
                    }
                    bool sup = false;
                    for (int k = 0; k < c.names_cnt; k++) if (names[c.names_off + k] == reads->read_id[r]) { sup = true; break; }
                    if (!sup) dr[wsorted[w].cand]++;
                }
        }
        for (uint32_t i = 0; i < nc; i++) {
            if (n_windows_of(cands[i]) == 0) continue;
            if (!has_rows[cands[i].chrom]) { cands[i].flags |= CSV_F_NO_READS; continue; }
            csv_geno g = cx.gl[gl_index((int32_t)dr[i], cands[i].names_cnt)];
            g.dr = (int32_t)dr[i]; g.dv = cands[i].names_cnt;
            genos[i] = g;
        }
    }
    if (P->genotype && aln && aln->n > 0) {  // TRA genotyper on the packed all-alignments table (mirrors k_aln_index + k_tra_genotype)
        std::vector<uint32_t> off(n_contigs + 2, 0xffffffffu);
        std::vector<int32_t> span(n_contigs + 2, 0);
        for (int64_t i = 0; i < aln->n; i++) {
            const int32_t c = aln->chrom[i];
            if (i == 0 || aln->chrom[i - 1] != c) off[c] = (uint32_t)i;
            span[c] = std::max(span[c], aln->end[i] - aln->start[i]);
        }
        off[n_contigs] = (uint32_t)aln->n;
        for (int c = n_contigs - 1; c >= 0; c--) if (off[c] == 0xffffffffu) off[c] = off[c + 1];
        AlnView A{aln->chrom, aln->start, aln->end, aln->read_id, aln->is_primary, off.data(), span.data(), contig_len};
        for (uint32_t i = 0; i < nc; i++) {
            if (cands[i].svtype != CSV_TRA) continue;
            tra_call_gt(A, cands[i], names + cands[i].names_off, P->bias_tra, P->gt_round, cx.gl.data(), &genos[i]);
            cands[i].flags &= ~CSV_F_GT_HOST;
        }
    }
    return CSV_OK;
}

// ------------------------------------------------------------------------------------------
// extraction emulator: serial CIGAR walk + the shared per-read logic of extract_core.h
// ------------------------------------------------------------------------------------------
#include "../../cutesv_b200/csrc/extract_core.h"

extern "C" int emul_extract(const csv_params* P0, const csv_read_cols* reads, const uint32_t* cigar, const csv_sa_cols* sa,
                            int32_t* out_cols /* [5 types][5 cols][cap] */, int64_t cap, int32_t* piece_off, int32_t* piece_cnt,
                            int32_t* pieces4, int64_t cap_pieces, int32_t* rr /* [4][cap_rows] */, uint8_t* rr_prim, int64_t cap_rows,
                            int64_t counts[8]) {
    using namespace csv;
    ExtractParams P;
    P.min_size = P0->min_size; P.max_size = P0->max_size; P.min_mapq = P0->min_mapq; P.max_split_parts = P0->max_split_parts;
    P.min_read_len = P0->min_read_len; P.min_siglength = P0->min_siglength; P.merge_del_threshold = P0->merge_del_threshold;
    P.merge_ins_threshold = P0->merge_ins_threshold;
    uint32_t ctr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    ExtractOut O;
    memset(&O, 0, sizeof(O));
    for (int t = 0; t < CSV_NTYPES; t++) {
        for (int k = 0; k < 5; k++) O.col[t][k] = out_cols + ((size_t)t * 5 + k) * cap;
        O.cap_sig[t] = (uint32_t)cap;
    }
    O.n_sig = ctr; O.n_pieces = ctr + 5; O.n_rows = ctr + 6; O.status = ctr + 7;
    O.ins_piece_off = piece_off; O.ins_piece_cnt = piece_cnt; O.pieces = (InsPiece*)pieces4; O.cap_pieces = (uint32_t)cap_pieces;
    O.rr_chrom = rr; O.rr_start = rr + cap_rows; O.rr_end = rr + 2 * cap_rows; O.rr_id = rr + 3 * cap_rows; O.rr_prim = rr_prim;
    O.cap_rows = (uint32_t)cap_rows;
    SaView S{sa->chrom, sa->pos0, sa->strand, sa->mapq, sa->first_clip, sa->last_clip, sa->ref_span};
    for (int64_t rec = 0; rec < reads->n; rec++) {
        const int32_t flag = reads->flag[rec];
        if (flag == 256 || flag == 272) continue;
        const int32_t mapq = reads->mapq[rec], qlen = reads->query_len[rec], chrom = reads->chrom[rec], rid = reads->read_id[rec];
        const bool mq_ok = mapq >= P.min_mapq;
        if (mq_ok) {
            uint32_t k = ctr[6]++;
            if ((int64_t)k < cap_rows) {
                O.rr_chrom[k] = chrom; O.rr_start[k] = reads->ref_start[rec]; O.rr_end[k] = reads->ref_end[rec]; O.rr_id[k] = rid;
                O.rr_prim[k] = (flag == 0 || flag == 16) ? 1 : 0;
            }
        }
        if (qlen < P.min_read_len) continue;
        ReadCtx RC; RC.rec = (int32_t)rec; RC.chrom = chrom; RC.rid = rid; RC.qlen = qlen; RC.base_rc = 0;
        const int64_t c_lo = reads->cigar_off[rec], c_hi = reads->cigar_off[rec + 1];
        int32_t clip_l = 0, clip_r = 0;
        if (mq_ok && c_hi > c_lo) {
            const uint32_t first = cigar[c_lo], last = cigar[c_hi - 1];
            const int fop = first & 15, lop = last & 15;
            const int32_t hard_l = fop == OP_H ? (int32_t)(first >> 4) : 0;
            if (fop == OP_S || fop == OP_H) clip_l = (int32_t)(first >> 4);
            if (lop == OP_S || lop == OP_H) clip_r = (int32_t)(last >> 4);
            MergeState St; St.reset();
            InsPiece open_pieces[MAX_OPEN_PIECES];
            int32_t ref = reads->ref_start[rec];
            int64_t q = -(int64_t)hard_l;
            for (int64_t i = c_lo; i < c_hi; i++) {
                const int op = cigar[i] & 15; const int32_t len = (int32_t)(cigar[i] >> 4);
                if (op != OP_D) q += len;
                if (len >= P.min_siglength && (op == OP_I || op == OP_D)) {
                    if (op == OP_D) { push_del(O, RC, P, St, ref, len); ref += len; }
                    else push_ins(O, RC, P, St, open_pieces, ref, len, q - len, q);
                } else if (op_ref_change(op)) ref += len;
            }
            flush_ins(O, RC, St, open_pieces); flush_del(O, RC, St);
        }
        const int sig = detect_flag(flag);
        const int64_t s_lo = reads->sa_off[rec], s_hi = reads->sa_off[rec + 1];
        if ((sig == 1 || sig == 2) && s_hi > s_lo) {
            SplitCtx C; C.O = &O; C.R = RC; C.P = P; C.R.base_rc = sig == 2 ? 1 : 0;
            Seg prim;
            if (sig == 1) { prim.rs = clip_l; prim.re = qlen - clip_r; } else { prim.rs = clip_r; prim.re = qlen - clip_l; }
            prim.fs = reads->ref_start[rec]; prim.fe = reads->ref_end[rec]; prim.chr = chrom; prim.strand = sig == 1 ? 0 : 1;
            organize_split_signal(C, mq_ok, prim, S, s_lo, s_hi);
        }
    }
    for (int k = 0; k < 8; k++) counts[k] = ctr[k];
    return CSV_OK;
}
