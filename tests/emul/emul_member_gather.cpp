// emul_member_gather.cpp -- TEST-ONLY serial emulation of k_select_heads' record-mode bit tests for one tile: the same
// core.h routines (chain_head, chain_member, chain_size_class) over the same link mask, with back words of halo before
// the tile.  tests/test_member_gather_cpu.py compiles it with g++.
#include "../../cutesv_b200/csrc/core.h"

using namespace csv;

// link: the mask words (back before the tile, then the tile, then the forward halo); tile positions p < n_valid exist.
// member[p] / head[p] = 1 for a member / head of a cluster of >= need members; cls[p] = the head's size class, else 0.
extern "C" void emul_member_gather(const uint32_t* link, int back, int tile, int n_valid, int need, int split, uint8_t* member,
                                   uint8_t* head, uint8_t* cls) {
    const int q0 = back * 32;
    for (int p = 0; p < tile; p++) {
        const bool ok = p < n_valid;
        member[p] = ok && chain_member(link, q0 + p, need) ? 1 : 0;
        head[p] = ok && chain_head(link, q0 + p, need) ? 1 : 0;
        cls[p] = head[p] ? (uint8_t)chain_size_class(link, q0 + p, split) : 0;
    }
}
