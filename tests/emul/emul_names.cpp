// emul_names.cpp -- TEST-ONLY host build of the routines of cutesv_b200/csrc/names_core.h, composed as csv_rank_names and
// csv_order_ins_ties compose them on the device: stable LSD rounds (length, then 8-byte words from the last down to word 0),
// adjacent comparison and dense ranks; per tie group the (sequence, row) ranks and the cycle moves.  Never part of the product.
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <vector>

#include "../../cutesv_b200/csrc/names_core.h"

using namespace csv;

// rank[i] = dense rank of name i (names[off[i] .. off[i + 1])) in byte order; returns the number of distinct names
extern "C" int64_t emul_name_ranks(const uint8_t* names, const int64_t* off, int64_t n, int32_t* rank) {
    std::vector<uint32_t> perm((size_t)n);
    std::iota(perm.begin(), perm.end(), 0u);
    auto len = [&](uint32_t x) { return off[x + 1] - off[x]; };
    int64_t max_len = 0;
    for (int64_t i = 0; i < n; i++) max_len = std::max(max_len, len((uint32_t)i));
    std::stable_sort(perm.begin(), perm.end(), [&](uint32_t x, uint32_t y) { return len(x) < len(y); });
    for (int w = (int)((max_len + 7) / 8) - 1; w >= 0; w--) {
        std::vector<uint64_t> key((size_t)n);
        for (int64_t i = 0; i < n; i++) key[(size_t)i] = name_word(names + off[i], len((uint32_t)i), w);
        std::stable_sort(perm.begin(), perm.end(), [&](uint32_t x, uint32_t y) { return key[x] < key[y]; });
    }
    int64_t r = -1;
    for (int64_t i = 0; i < n; i++) {
        const uint32_t x = perm[(size_t)i];
        if (i == 0 || bytes_cmp(names + off[perm[(size_t)i - 1]], len(perm[(size_t)i - 1]), names + off[x], len(x)) != 0) r++;
        rank[x] = (int32_t)r;
    }
    return r + 1;
}

namespace {
struct ContentMover {
    int32_t* content;
    void load(uint32_t r, int32_t& v) const { v = content[r]; }
    void store(uint32_t r, const int32_t& v) const { content[r] = v; }
};
}  // namespace

// INS rows sorted by (contig, int(pos), len, read, row) in perm, tie[i] = sorted row i ties with sorted row i - 1; the strings
// of row r are bytes[start[r] .. start[r] + len[r]).  content[r] (in: any labels) is moved as the device moves a row's
// columns.  Returns the number of rows whose content changed.
extern "C" int64_t emul_tie_order(const uint32_t* perm, const uint8_t* tie, int64_t n, const uint8_t* bytes, const int64_t* start,
                                  const int32_t* len, int32_t* content) {
    int64_t moved = 0;
    std::vector<uint32_t> dst;
    ContentMover mv{content};
    for (int64_t h = 0; h + 1 < n; h++) {
        if (tie[h] || !tie[h + 1]) continue;
        int64_t e = h + 2;
        while (e < n && tie[e]) e++;
        const int32_t m = (int32_t)(e - h);
        dst.assign((size_t)m, 0u);
        for (int32_t p = 0; p < m; p++) dst[(size_t)p] = (uint32_t)tie_rank(perm + h, m, p, bytes, start, len);
        for (int32_t p = 0; p < m; p++) moved += dst[(size_t)p] != (uint32_t)p;
        tie_apply<int32_t>(perm + h, dst.data(), m, mv);
    }
    return moved;
}
