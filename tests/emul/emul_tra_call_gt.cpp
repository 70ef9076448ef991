// emul_tra_call_gt.cpp -- TEST-ONLY serial emulation of csv_tra_call_gt: the same input checks, contig index (k_aln_index +
// k_aln_off) and per-query rules (core.h tra_call_gt, the scalar count_coverage) as the library.
// Never part of the product; tests/test_tra_call_gt_cpu.py compiles it with g++.
#include <algorithm>
#include <vector>

#include "../../cutesv_b200/csrc/core.h"
#include "../../cutesv_b200/csrc/host_tables.h"

using namespace csv;

extern "C" int emul_tra_call_gt(const csv_tra_query* q, int64_t n, const csv_reads_cols* aln, int32_t n_contigs, const int64_t* contig_len,
                                int32_t bias, int32_t gt_round, const int64_t* sup_off, const int32_t* sup_ids, csv_geno* out) {
    if (n < 0 || bias < 0 || sup_off[0] != 0) return CSV_E_INVALID;
    for (int64_t i = 0; i < n; i++) {
        if (sup_off[i + 1] < sup_off[i]) return CSV_E_INVALID;
        const int32_t ch[2] = {q[i].chr1, q[i].chr2};
        const int64_t pos[2] = {q[i].pos1, q[i].pos2};
        for (int k = 0; k < 2; k++) {
            if (ch[k] < 0 || ch[k] >= n_contigs) return CSV_E_INPUT;
            if (std::max<int64_t>(pos[k] - bias, 0) > std::min<int64_t>(pos[k] + bias, contig_len[ch[k]])) return CSV_E_INPUT;
        }
    }
    std::vector<uint32_t> off(n_contigs + 2, 0);
    std::vector<int32_t> span(n_contigs + 2, 0);
    for (int64_t i = 0; i < aln->n; i++) {
        const int32_t c = aln->chrom[i];
        if (c < 0 || c >= n_contigs) return CSV_E_INPUT;
        if (i > 0 && (aln->chrom[i - 1] > c || (aln->chrom[i - 1] == c && aln->start[i - 1] > aln->start[i]))) return CSV_E_INPUT;
        span[c] = std::max(span[c], aln->end[i] - aln->start[i]);
    }
    for (int32_t c = 0; c <= n_contigs; c++)   // first row of contig c
        off[c] = (uint32_t)(std::lower_bound(aln->chrom, aln->chrom + aln->n, c) - aln->chrom);
    const AlnView A{aln->chrom, aln->start, aln->end, aln->read_id, aln->is_primary, off.data(), span.data(), contig_len};
    const std::vector<csv_geno> gl = build_gl_table();
    for (int64_t i = 0; i < n; i++) {
        std::vector<int32_t> sup(sup_ids + sup_off[i], sup_ids + sup_off[i + 1]);
        std::sort(sup.begin(), sup.end());
        out[i] = tra_call_gt(A, q[i].chr1, q[i].pos1, q[i].chr2, q[i].pos2, sup.data(), (int32_t)sup.size(), bias, gt_round, gl.data());
    }
    return CSV_OK;
}
