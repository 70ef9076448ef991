// emul_part_strip_nt.cpp -- TEST-ONLY serial emulation of k_part_filter's strip pass over nt strips (the CTA's threads)
// for any partition width: the histogram stored transposed as the kernel stores it (bucket b at (b % per) * nt + b / per,
// per = max(1, bp / nt)), every strip read through both of core.h's accessors the kernel passes (interior strips: word
// j * nt + strip + s, no bounds test), the strips at or past bp empty when bp < nt, and the CTA's exclusive scan over the
// nt strips done serially.  tests/test_part_filter_512_cpu.py compiles it with g++.
#include <vector>

#include "../../cutesv_b200/csrc/core.h"

using namespace csv;

// hist: bp = 2^k bucket counts in bucket order; nt = 2^m strips of per = max(1, bp / nt) buckets (per <= 64); hl / hr: 64
// halo counts each (only j < rb may be read).  keep[b] = 1 for a kept bucket; off[b] = its exclusive offset among the
// kept buckets' signatures; *n_interior = strips that took the interior path.  Returns the total.
extern "C" uint32_t emul_part_strip_nt(const uint32_t* hist, int bp, int nt, int rb, uint32_t need, const uint32_t* hl,
                                       const uint32_t* hr, uint8_t* keep, uint32_t* off, int* n_interior) {
    const int per = bp > nt ? bp / nt : 1, owners = bp < nt ? bp : nt;
    auto phys = [&](int b) { return (b % per) * nt + b / per; };
    std::vector<uint32_t> h(bp);
    for (int b = 0; b < bp; b++) h[phys(b)] = hist[b];
    auto count = [&](int b) -> uint32_t { return h[phys(b)]; };
    std::vector<uint64_t> flags(nt, 0);
    std::vector<uint32_t> first(nt);
    uint32_t total = 0;
    *n_interior = 0;
    for (int t = 0; t < nt; t++) {
        uint32_t kept = 0;
        if (t < owners) {
            auto strip = [&](int s, int j) -> uint32_t { return h[j * nt + t + s]; };
            flags[t] = pf_strip_flags(count, strip, t * per, per, bp, rb, need, hl, hr, &kept);
            *n_interior += pf_strip_interior(t * per, per, bp, rb) ? 1 : 0;
        }
        first[t] = total;
        total += kept;
    }
    for (int t = 0; t < owners; t++)
        pf_strip_offsets([&](int b) -> uint32_t { return h[(b - t * per) * nt + t]; }, t * per, per, flags[t], first[t],
                         [&](int j, uint32_t o, bool f, uint32_t) {
                             keep[t * per + j] = f ? 1 : 0;
                             off[t * per + j] = o;
                         });
    return total;
}
