// emul_part_filter.cpp -- TEST-ONLY serial emulation of k_part_filter's density flags and bucket offsets for one
// partition: the same strip templates (core.h pf_strip_flags / pf_strip_offsets) over the same transposed histogram,
// with the CTA's exclusive scan over the 256 strips done serially.  tests/test_part_filter_strip_cpu.py compiles it with g++.
#include <vector>

#include "../../cutesv_b200/csrc/core.h"

using namespace csv;

// hist: bp = 256 * per bucket counts in bucket order (per = 1, 2, 4, ..., 64); hl / hr: 64 halo counts each (only j < rb
// may be read).  keep[b] = 1 for a kept bucket; off[b] = its exclusive offset among the kept buckets' signatures; returns
// the total.
extern "C" uint32_t emul_part_filter(const uint32_t* hist, int per, int rb, uint32_t need, const uint32_t* hl, const uint32_t* hr,
                                     uint8_t* keep, uint32_t* off) {
    const int bp = 256 * per;
    int lper = 0;
    while ((1 << lper) < per) lper++;
    auto phys = [&](int b) { return ((b & (per - 1)) << 8) | (b >> lper); };
    std::vector<uint32_t> h(bp);
    for (int b = 0; b < bp; b++) h[phys(b)] = hist[b];
    auto count = [&](int b) -> uint32_t { return h[phys(b)]; };
    std::vector<uint64_t> flags(256);
    std::vector<uint32_t> first(256);
    uint32_t total = 0;
    for (int t = 0; t < 256; t++) {
        uint32_t kept;
        flags[t] = pf_strip_flags(count, t * per, per, bp, rb, need, hl, hr, &kept);
        first[t] = total;
        total += kept;
    }
    for (int t = 0; t < 256; t++)
        pf_strip_offsets(count, t * per, per, flags[t], first[t], [&](int j, uint32_t o, bool f, uint32_t) {
            keep[t * per + j] = f ? 1 : 0;
            off[t * per + j] = o;
        });
    return total;
}
