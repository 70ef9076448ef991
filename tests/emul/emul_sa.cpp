// emul_sa.cpp -- TEST-ONLY host build of the SA:Z reduction of cutesv_b200/csrc/sa_core.h: the strip walk of k_sa_count /
// k_sa_fill with the strips' bit masks built by a byte loop instead of ballots, and the per-entry parse.  Never part of the product.
#include <cstdint>

#include "../../cutesv_b200/csrc/sa_core.h"

using namespace csv;

// Reduces records [0, n) of (text, text_off) with the name table (names sorted bytewise, their ids).  Returns the SA_BAD_* bits
// (SA_BAD_OFF: nothing written); otherwise sa_off (n + 1) and the seven columns cols[k * cap + row] hold the table, and
// *n_rows its row count (rows past cap are counted, not written).
extern "C" uint32_t emul_sa_reduce(const uint8_t* name_bytes, const int64_t* name_off, const int32_t* name_id, int64_t n_names, const uint8_t* text,
                                   const int64_t* text_off, int64_t n_bytes, int64_t n, int64_t* sa_off, int32_t* cols, int64_t cap, int64_t* n_rows) {
    for (int64_t i = 0; i < n; i++)
        if (text_off[i] < 0 || text_off[i + 1] < text_off[i] || text_off[i + 1] > n_bytes) return SA_BAD_OFF;
    const SaNames N{name_bytes, name_off, name_id, n_names};
    uint32_t bad = 0;
    int64_t row = 0;
    for (int64_t i = 0; i < n; i++) {
        sa_off[i] = row;
        const int64_t lo = text_off[i], hi = text_off[i + 1];
        SaWalk W{lo, 0, false};
        for (int64_t b = lo; b < hi && !W.done; b += 32) {
            uint32_t semi = 0, comma = 0, nul = 0;
            for (int j = 0; j < 32 && b + j < hi; j++) {
                const uint8_t x = text[b + j];
                semi |= (uint32_t)(x == ';') << j;
                comma |= (uint32_t)(x == ',') << j;
                nul |= (uint32_t)(x == 0) << j;
            }
            const int64_t open = W.start;
            uint32_t s;
            for (uint32_t keep = sa_strip(semi, comma, nul, b, W, &s); keep; keep &= keep - 1u) {
                const int j = sa_ctz(keep);
                const int64_t start = sa_entry_start(s, j, b, open);
                SaRow R;
                bad |= sa_parse_entry(text + start, b + j - start, N, R);
                if (row < cap) {
                    const int32_t v[7] = {R.chrom, R.pos0, R.strand, R.mapq, R.first, R.last, R.span};
                    for (int k = 0; k < 7; k++) cols[k * cap + row] = v[k];
                }
                row++;
            }
        }
    }
    sa_off[n] = row;
    *n_rows = row;
    return bad;
}
