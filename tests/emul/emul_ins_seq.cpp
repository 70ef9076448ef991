// emul_ins_seq.cpp -- TEST-ONLY host build of the INS sequence routines of cutesv_b200/csrc/extract_core.h (SeqRec,
// ins_piece_bytes, ins_marker_bytes), driven like k_ins_len + k_ins_fill drive them on the device: a length pass over every
// INS row, an exclusive scan, a fill pass.  Also the output offsets of csv_fetch_ins_seqs (ins_fetch_offsets).  Never part of
// the product.
#include <cstdint>
#include <vector>

#include "../../cutesv_b200/csrc/extract_core.h"

using namespace csv;

namespace {
struct Packet {
    const int32_t* query_len; const int64_t* seq_off; const uint8_t* seq4;
    const int64_t* cigar_off; const uint32_t* cigar; const int32_t* ref_start;
    int32_t min_siglength, merge_ins_threshold;
};
SeqRec seq_rec(const Packet& P, int64_t rec) {
    SeqRec s;
    s.qlen = P.query_len[rec];
    s.have = P.seq_off[rec + 1] - P.seq_off[rec] >= ((int64_t)s.qlen + 1) / 2;
    s.seq4 = P.seq4 + P.seq_off[rec];
    return s;
}
// bytes of one INS row (out == nullptr: length only); -1 when a marker piece names no merged insertion
int64_t row_bytes(const Packet& P, const InsPiece* pieces, int32_t po, int32_t pc, int32_t rec_base, uint8_t* out) {
    int64_t w = 0;
    for (int32_t p = po; p < po + pc; p++) {
        const InsPiece ip = pieces[p];
        const int64_t rec = (int64_t)ip.rec - rec_base;
        const SeqRec s = seq_rec(P, rec);
        int64_t v;
        if (ip.rc == 2) {
            const int64_t c0 = P.cigar_off[rec];
            v = ins_marker_bytes(s, P.cigar + c0, P.cigar_off[rec + 1] - c0, P.ref_start[rec], ip.start, P.min_siglength, P.merge_ins_threshold,
                                 out ? out + w : nullptr);
            if (v < 0) return -1;
        } else v = ins_piece_bytes(s, ip.start, ip.stop, ip.rc, out ? out + w : nullptr, 0, 1);
        w += v;
    }
    return w;
}
}  // namespace

// Strings of INS rows 0..n_rows (pieces4: 4 int32 per piece; rows' pieces po[k] .. po[k] + pc[k]); row k is
// out[out_off[k] .. out_off[k + 1]).  Returns 0, -1 (marker without a merged insertion) or -3 (cap too small; out_off[n_rows]
// holds the size needed).
extern "C" int emul_ins_seqs(const int32_t* pieces4, const int32_t* po, const int32_t* pc, int64_t n_rows, int32_t rec_base,
                             const int32_t* query_len, const int64_t* seq_off, const uint8_t* seq4, const int64_t* cigar_off,
                             const uint32_t* cigar, const int32_t* ref_start, int32_t min_siglength, int32_t merge_ins_threshold,
                             uint8_t* out, int64_t cap, int64_t* out_off) {
    const Packet P{query_len, seq_off, seq4, cigar_off, cigar, ref_start, min_siglength, merge_ins_threshold};
    const InsPiece* pieces = reinterpret_cast<const InsPiece*>(pieces4);
    out_off[0] = 0;
    for (int64_t k = 0; k < n_rows; k++) {
        const int64_t v = row_bytes(P, pieces, po[k], pc[k], rec_base, nullptr);
        if (v < 0) return -1;
        out_off[k + 1] = out_off[k] + v;
    }
    if (out_off[n_rows] > cap) return -3;
    for (int64_t k = 0; k < n_rows; k++)
        if (row_bytes(P, pieces, po[k], pc[k], rec_base, out + out_off[k]) != out_off[k + 1] - out_off[k]) return -1;
    return 0;
}

// csv_fetch_ins_seqs' output offsets of rows with lengths len[0..n) (out_off: n + 1 entries); returns the total
extern "C" int64_t emul_fetch_offsets(const int32_t* len, int64_t n, int64_t* out_off) { return ins_fetch_offsets(len, n, out_off); }
