// sa_core.h -- SA:Z tag text to the csv_sa_cols rows (csv_reduce_sa_device), host/device shared.
//
// The statement is the host reduction of bam_reader.cpp (parse_range, clip_pos), which the tests pin to the reference's
// split(';')[:-1] / split(',') / acquire_clip_pos (cuteSV:466-509, 678):
//   - a NUL byte ends the value; an entry ends at ';', and an entry without its ';' is dropped with everything after it;
//   - an entry is split at its first five commas and needs at least 5 fields (4 commas);
//   - rname -> contig id through the csv_set_contig_names table (-1 when unknown), pos0 = atoi(f1) - 1, strand '+' -> 0 else 1,
//     mapq = atoi(f4), the CIGAR f3 through clip_pos.
// A number whose value does not fit int32 sets an SA_BAD_* bit instead (the host's atoi is undefined there).
// The record walk is split into 32-byte strips: sa_strip takes a strip's ';', ',' and NUL bit masks (a warp's ballots on the
// device, a byte loop on the host) and returns the positions of the ';' that close a kept entry.
// The test-only host build (tests/emul/emul_sa.cpp) runs the same routines against bamio.BamReader's reduction.
#pragma once
#include "core.h"
#include "names_core.h"

namespace csv {

enum : uint32_t { SA_BAD_OFF = 1u, SA_BAD_POS = 2u, SA_BAD_MAPQ = 4u, SA_BAD_CIGAR = 8u };

// csv_set_contig_names' table: the names in byte order, name k at bytes[off[k], off[k + 1]) with contig id id[k]
struct SaNames {
    const uint8_t* bytes;
    const int64_t* off;
    const int32_t* id;
    int64_t n;
};

struct SaRow {
    int32_t chrom, pos0, strand, mapq, first, last, span;
};

// The walk of one record's value across strips
struct SaWalk {
    int64_t start;    // first byte of the open entry
    int32_t commas;   // commas of the open entry so far (saturates at 4)
    bool done;        // a NUL was seen: nothing after it counts
};

CSV_HD uint32_t sa_popc(uint32_t x) {
#ifdef __CUDA_ARCH__
    return (uint32_t)__popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}
CSV_HD int sa_ctz(uint32_t x) {
#ifdef __CUDA_ARCH__
    return __ffs((int)x) - 1;
#else
    return __builtin_ctz(x);
#endif
}
CSV_HD int sa_msb(uint32_t x) {
#ifdef __CUDA_ARCH__
    return 31 - __clz((int)x);
#else
    return 31 - __builtin_clz(x);
#endif
}

// One strip: bytes [base, base + 32) of the value, bit j of semi / comma / nul set for the byte at base + j (bits past the
// value's end clear).  Returns the bits of the ';' that close an entry of >= 5 fields.  *semi_out: the ';' bits before the
// first NUL (sa_entry_start's input).  Updates W.
CSV_HD uint32_t sa_strip(uint32_t semi, uint32_t comma, uint32_t nul, int64_t base, SaWalk& W, uint32_t* semi_out) {
    if (nul) {
        const uint32_t below = (nul & (0u - nul)) - 1u;
        semi &= below;
        comma &= below;
        W.done = true;
    }
    *semi_out = semi;
    uint32_t keep = 0, rest = semi;
    int lo = 0;   // first bit of the open entry inside the strip
    int32_t carry = W.commas;
    while (rest) {
        const int j = sa_ctz(rest);
        rest &= rest - 1u;
        const uint32_t seg = (j == 0 ? 0u : (0xffffffffu >> (32 - j))) & (0xffffffffu << lo);
        if (carry + (int32_t)sa_popc(comma & seg) >= 4) keep |= 1u << j;
        carry = 0;
        lo = j + 1;
    }
    if (semi) W.start = base + sa_msb(semi) + 1;
    const int32_t c = carry + (lo < 32 ? (int32_t)sa_popc(comma >> lo) : 0);
    W.commas = c < 4 ? c : 4;
    return keep;
}

// First byte of the entry closed by the ';' at bit j of a strip at `base`; open_start: W.start before sa_strip ran
CSV_HD int64_t sa_entry_start(uint32_t semi, int j, int64_t base, int64_t open_start) {
    const uint32_t lower = j == 0 ? 0u : semi & (0xffffffffu >> (32 - j));
    return lower ? base + sa_msb(lower) + 1 : open_start;
}

// atoi of the field p[0, len) (atoi stops at the field's end, a ',' or ';', anyway): C whitespace, one sign, digits.
// *ovf when the value is outside [lo, 2^31 - 1].
CSV_HD int32_t sa_atoi(const uint8_t* p, int64_t len, int64_t lo, bool* ovf) {
    int64_t i = 0;
    while (i < len && (p[i] == ' ' || (p[i] >= '\t' && p[i] <= '\r'))) i++;
    bool neg = false;
    if (i < len && (p[i] == '+' || p[i] == '-')) neg = p[i++] == '-';
    int64_t v = 0;
    for (; i < len && p[i] >= '0' && p[i] <= '9'; i++) {
        v = v * 10 + (p[i] - '0');
        if (v > (1ll << 31)) { *ovf = true; return 0; }
    }
    if (neg) v = -v;
    if (v < lo || v > 2147483647ll) { *ovf = true; return 0; }
    return (int32_t)v;
}

// Contig id of the name p[0, len) (-1 when the table has no such name)
CSV_HD int32_t sa_contig(const SaNames& N, const uint8_t* p, int64_t len) {
    int64_t lo = 0, hi = N.n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        const int64_t o = N.off[mid];
        const int c = bytes_cmp(N.bytes + o, N.off[mid + 1] - o, p, len);
        if (c == 0) return N.id[mid];
        if (c < 0) lo = mid + 1; else hi = mid;
    }
    return -1;
}

// The row of one kept entry p[0, len) (its ';' excluded; at least 4 commas).  Returns SA_BAD_* bits (0: R is the row).
CSV_HD uint32_t sa_parse_entry(const uint8_t* p, int64_t len, const SaNames& N, SaRow& R) {
    // starts of fields 1 .. 5 (scalars, not an array: a dynamically indexed array would live in local memory on the device);
    // field k ends one byte before field k + 1 starts, field 4 at len when there is no field 5
    int64_t f1 = 0, f2 = 0, f3 = 0, f4 = 0, end4 = len;
    int nf = 1;
    for (int64_t q = 0; q < len && nf < 6; q++) {
        if (p[q] != ',') continue;
        if (nf == 1) f1 = q + 1;
        else if (nf == 2) f2 = q + 1;
        else if (nf == 3) f3 = q + 1;
        else if (nf == 4) f4 = q + 1;
        else end4 = q;
        nf++;
    }
    uint32_t bad = 0;
    bool ovf = false;
    R.chrom = sa_contig(N, p, f1 - 1);
    R.pos0 = sa_atoi(p + f1, f2 - 1 - f1, -2147483647ll, &ovf) - 1;
    if (ovf) bad |= SA_BAD_POS;
    ovf = false;
    R.strand = p[f2] == '+' ? 0 : 1;
    R.mapq = sa_atoi(p + f4, end4 - f4, -2147483647ll - 1, &ovf);
    if (ovf) bad |= SA_BAD_MAPQ;
    // clip_pos: the first op's S, M D = X toward the span, the last op's S
    int64_t num = 0, span = 0;
    int32_t first = 0, last_len = 0;
    bool first_op = true;
    uint8_t last_op = 0;
    for (int64_t i = f3; i < f4 - 1; i++) {
        const uint8_t c = p[i];
        if (c >= '0' && c <= '9') {
            num = num * 10 + (c - '0');
            if (num > 2147483647ll) { bad |= SA_BAD_CIGAR; num = 0; }
            continue;
        }
        if (first_op) { if (c == 'S') first = (int32_t)num; first_op = false; }
        if (c == 'M' || c == 'D' || c == '=' || c == 'X') span += num;
        last_len = (int32_t)num;
        last_op = c;
        num = 0;
    }
    if (span > 2147483647ll) bad |= SA_BAD_CIGAR;
    R.first = first;
    R.last = last_op == 'S' ? last_len : 0;
    R.span = (int32_t)span;
    return bad;
}

}  // namespace csv
