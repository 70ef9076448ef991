// emul_genotype.cpp -- TEST-ONLY serial emulation of csv_overlap_cover / csv_call_gt: the same per-contig bins, pair rules
// (core.h gc_*), segment sort + dedup (gc_sort_unique with a one-thread team) and DR (gc_union_minus) as the kernels.
// Never part of the product; tests/test_genotype_dropin_cpu.py compiles it with g++.
#include <algorithm>
#include <vector>

#include "../../cutesv_b200/csrc/core.h"
#include "../../cutesv_b200/csrc/host_tables.h"

using namespace csv;
namespace {

struct GcCsr { std::vector<int64_t> off; std::vector<int32_t> ids; };

int gc_emulate(const csv_window* win, int64_t n_win, const csv_reads_cols* R, std::vector<uint32_t>& iter, std::vector<uint32_t>& prim,
               GcCsr& cov, GcCsr& ovl) {
    int32_t n_wc = 0;
    for (int64_t i = 0; i < n_win; i++) {
        if (win[i].chrom < 0 || win[i].e2 <= win[i].s2) return CSV_E_INPUT;
        n_wc = std::max(n_wc, win[i].chrom + 1);
    }
    std::vector<int64_t> base(n_wc + 1, 0), last(n_wc, -1);
    for (int64_t i = 0; i < n_win; i++) last[win[i].chrom] = std::max(last[win[i].chrom], gc_bin(win[i].e2 - 1));
    for (int32_t k = 0; k < n_wc; k++) base[k + 1] = base[k] + last[k] + 1;
    std::vector<std::vector<uint32_t>> bins(base[n_wc]);
    for (int64_t i = 0; i < n_win; i++)
        for (int64_t b = gc_bin(win[i].s2); b <= gc_bin(win[i].e2 - 1); b++) bins[base[win[i].chrom] + b].push_back((uint32_t)i);
    iter.assign(n_win, 0); prim.assign(n_win, 0);
    std::vector<std::vector<int32_t>> cv(n_win), ov(n_win);
    for (int64_t r = 0; R && r < R->n; r++) {
        const int32_t ch = R->chrom[r];
        if (ch < 0 || R->end[r] < R->start[r]) return CSV_E_INPUT;
        if (ch >= n_wc) continue;
        const int64_t nb = base[ch + 1] - base[ch], rs2 = 2 * (int64_t)R->start[r], re2 = 2 * (int64_t)R->end[r];
        const bool pr = R->is_primary[r] != 0;
        for (int64_t b = gc_bin(rs2); b <= std::min(gc_bin(re2), nb - 1); b++)
            for (uint32_t w : bins[base[ch] + b]) {
                if (!gc_overlaps(rs2, re2, win[w].s2, win[w].e2) || !gc_pair_home(rs2, win[w].s2, b)) continue;
                iter[w]++;
                if (!pr) continue;
                prim[w]++;
                ov[w].push_back(R->read_id[r]);
                if (gc_covers(rs2, re2, win[w].s2, win[w].e2)) cv[w].push_back(R->read_id[r]);
            }
    }
    HostTeam tm;
    for (int k = 0; k < 2; k++) {
        auto& seg = k ? ov : cv;
        GcCsr& out = k ? ovl : cov;
        out.off.assign(n_win + 1, 0); out.ids.clear();
        for (int64_t w = 0; w < n_win; w++) {
            std::vector<uint8_t> first(seg[w].size() + 1);
            std::vector<int32_t> ded(seg[w].size() + 1);
            const int u = gc_sort_unique(tm, seg[w].data(), (int)seg[w].size(), first.data(), ded.data());
            out.ids.insert(out.ids.end(), ded.begin(), ded.begin() + u);
            out.off[w + 1] = (int64_t)out.ids.size();
        }
    }
    return CSV_OK;
}

}  // namespace

// cap: room in cover_ids / overlap_ids each; returns CSV_E_CAPACITY when too small
extern "C" int emul_overlap_cover(const csv_window* win, int64_t n_win, const csv_reads_cols* reads, int32_t* iteration, int32_t* primary_num,
                                  int64_t* cover_off, int32_t* cover_ids, int64_t* overlap_off, int32_t* overlap_ids, int64_t cap) {
    std::vector<uint32_t> it, pr;
    GcCsr cov, ovl;
    const int rc = gc_emulate(win, n_win, reads, it, pr, cov, ovl);
    if (rc) return rc;
    if ((int64_t)cov.ids.size() > cap || (int64_t)ovl.ids.size() > cap) return CSV_E_CAPACITY;
    for (int64_t w = 0; w < n_win; w++) { iteration[w] = (int32_t)it[w]; primary_num[w] = (int32_t)pr[w]; }
    std::copy(cov.off.begin(), cov.off.end(), cover_off); std::copy(ovl.off.begin(), ovl.off.end(), overlap_off);
    std::copy(cov.ids.begin(), cov.ids.end(), cover_ids); std::copy(ovl.ids.begin(), ovl.ids.end(), overlap_ids);
    return CSV_OK;
}

extern "C" int emul_call_gt(const csv_window* win, int64_t n_cand, int32_t per, const csv_reads_cols* reads, const int64_t* sup_off,
                            const int32_t* sup_ids, csv_geno* out) {
    std::vector<uint32_t> it, pr;
    GcCsr cov, ovl;
    const int rc = gc_emulate(win, n_cand * per, reads, it, pr, cov, ovl);
    if (rc) return rc;
    const std::vector<csv_geno> gl = build_gl_table();
    for (int64_t i = 0; i < n_cand; i++) {
        std::vector<int32_t> sup(sup_ids + sup_off[i], sup_ids + sup_off[i + 1]);
        std::sort(sup.begin(), sup.end());
        const int64_t w0 = i * per, w1 = w0 + per - 1;
        const int n1 = per == 2 ? (int)(cov.off[w1 + 1] - cov.off[w1]) : 0;
        const int32_t dr = gc_union_minus(cov.ids.data() + cov.off[w0], (int)(cov.off[w0 + 1] - cov.off[w0]), cov.ids.data() + cov.off[w1], n1,
                                          sup.data(), (int)sup.size());
        const int32_t dv = (int32_t)sup.size();
        out[i] = gl[gl_index(dr, dv)];
        out[i].dr = dr; out[i].dv = dv;
    }
    return CSV_OK;
}

extern "C" int emul_cal_gl(const int32_t* c0, const int32_t* c1, int64_t n, csv_geno* out) {
    const std::vector<csv_geno> gl = build_gl_table();
    for (int64_t i = 0; i < n; i++) { out[i] = gl[gl_index(c0[i], c1[i])]; out[i].dr = c0[i]; out[i].dv = c1[i]; }
    return CSV_OK;
}
