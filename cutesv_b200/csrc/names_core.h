// names_core.h -- read-name sort keys and the sequence order of INS tie groups, host/device shared.
//
// csv_rank_names sorts the read names of an accumulation byte-lexicographically (the order of Python `str` for UTF-8 text,
// which the reference's sort keys use through the read name, cuteSV:764-801) with LSD-chained radix rounds: one round on the
// name length, then one per 8-byte big-endian word from the last down to word 0.  Zero padding alone would tie "ab" with
// "ab\0"; the length round, the least significant key, puts the shorter name first.
// csv_order_ins_ties orders the INS rows that tie on (contig, int(pos), len, read) by their sequence strings (cuteSV:774).
// The test-only host build (tests/emul/emul_names.cpp) composes the same routines.
#pragma once
#include "core.h"

namespace csv {

static constexpr int NAME_MAX_BYTES = 254;   // BAM's l_read_name limit, NUL excluded

// big-endian word w (bytes [8w, 8w + 8)) of the name p[0 .. len), zero padded
CSV_HD uint64_t name_word(const uint8_t* p, int64_t len, int w) {
    uint64_t k = 0;
    const int64_t o = (int64_t)w * 8;
    for (int j = 0; j < 8; j++) {
        const int64_t i = o + j;
        k = (k << 8) | (uint64_t)(i < len ? p[i] : 0u);
    }
    return k;
}

// byte-lexicographic comparison (<0, 0, >0); a proper prefix sorts first, embedded NUL bytes included
CSV_HD int bytes_cmp(const uint8_t* a, int64_t la, const uint8_t* b, int64_t lb) {
    const int64_t m = la < lb ? la : lb;
    for (int64_t i = 0; i < m; i++)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return la < lb ? -1 : la > lb ? 1 : 0;
}

// Rank of member p of an INS tie group by (sequence bytes, row): the group's members are rows[0 .. m), ascending, so the row
// tie-break is the member index.  Row r's string is bytes[start[r] .. start[r] + len[r]).
CSV_HD int32_t tie_rank(const uint32_t* rows, int32_t m, int32_t p, const uint8_t* bytes, const int64_t* start, const int32_t* len) {
    const uint32_t rp = rows[p];
    const uint8_t* sp = bytes + start[rp];
    int32_t r = 0;
    for (int32_t q = 0; q < m; q++) {
        if (q == p) continue;
        const uint32_t rq = rows[q];
        const int c = bytes_cmp(bytes + start[rq], len[rq], sp, len[rp]);
        r += (c < 0 || (c == 0 && q < p)) ? 1 : 0;
    }
    return r;
}

// Moves the group's contents so that the content of rows[p] ends on rows[dst[p]] (dst: a permutation of [0, m)), one cycle at
// a time; dst entries are marked done with bit 31.  mv.load(row, T&) / mv.store(row, const T&) move one row's content.
template <class T, class Mover>
CSV_HD void tie_apply(const uint32_t* rows, uint32_t* dst, int32_t m, Mover& mv) {
    for (int32_t s = 0; s < m; s++) {
        if (dst[s] >> 31) continue;
        if ((int32_t)dst[s] == s) { dst[s] |= 1u << 31; continue; }
        T carry, next;
        mv.load(rows[s], carry);
        int32_t p = s;
        do {
            const int32_t q = (int32_t)(dst[p] & 0x7fffffffu);
            mv.load(rows[q], next);
            mv.store(rows[q], carry);
            dst[p] |= 1u << 31;
            carry = next;
            p = q;
        } while (p != s);
    }
}

}  // namespace csv
