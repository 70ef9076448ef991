// scan_core.h -- the -include_bed rule of a scanned packet (csv_scan_append_named_device), host/device shared.
//
// The reference fetches every task window of a contig and, with -include_bed, keeps a record iff it overlaps one of the
// padded regions assigned to that window (cuteSV:697-733, cuteSV_genotype.py:704-726).  One sequential pass over a sorted BAM
// sees each record once; the window that owns it is the last window of its contig starting at or before its reference start
// (cuteSV:725).  Window bounds can be fractional (cuteSV:1026-1034), so the starts are float64 and compared as such.
// The test-only host build (tests/emul/emul_scan.cpp) runs the same routine against cutesv_b200/cli.py's numpy rule.
#pragma once
#include "core.h"

namespace csv {

struct ScanRegions {
    const int64_t* win_off;    // n_contigs + 1: the windows of contig k are [win_off[k], win_off[k + 1]), starts ascending
    const double* win_start;   // per window
    const int64_t* reg_off;    // n_windows + 1: the regions of window w are [reg_off[w], reg_off[w + 1])
    const int64_t* reg;        // (lo, hi) per region; lo may be negative (the 1000 bp padding)
    int32_t n_contigs;         // 0: no table, every record passes
};

// true iff the record [start, end) on contig `chrom` passes the region table
CSV_HD bool scan_in_regions(const ScanRegions& T, int32_t chrom, int32_t start, int32_t end) {
    if (T.n_contigs == 0) return true;
    if (chrom < 0 || chrom >= T.n_contigs) return false;
    const int64_t w0 = T.win_off[chrom];
    int64_t lo = w0, hi = T.win_off[chrom + 1];
    const double s = (double)start;
    while (lo < hi) {   // first window whose start is > s
        const int64_t mid = (lo + hi) >> 1;
        if (T.win_start[mid] <= s) lo = mid + 1; else hi = mid;
    }
    if (lo == w0) return false;   // no window of the contig owns the record: the reference never fetches it
    const int64_t w = lo - 1;
    for (int64_t k = T.reg_off[w]; k < T.reg_off[w + 1]; k++)
        if (!((int64_t)end <= T.reg[2 * k] || (int64_t)start >= T.reg[2 * k + 1])) return true;
    return false;
}

}  // namespace csv
