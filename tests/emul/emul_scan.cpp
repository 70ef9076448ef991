// emul_scan.cpp -- TEST-ONLY host build of the region rule of cutesv_b200/csrc/scan_core.h (scan_in_regions), the test
// k_scan_flags applies to every scanned record.  Never part of the product.
#include <cstdint>

#include "../../cutesv_b200/csrc/scan_core.h"

using namespace csv;

// keep[i] = record i ([start[i], end[i]) on contig chrom[i]) passes the region table
extern "C" void emul_scan_keep(int32_t n_contigs, const int64_t* win_off, const double* win_start, const int64_t* reg_off, const int64_t* reg,
                               const int32_t* chrom, const int32_t* start, const int32_t* end, int64_t n, uint8_t* keep) {
    const ScanRegions T{win_off, win_start, reg_off, reg, n_contigs};
    for (int64_t i = 0; i < n; i++) keep[i] = scan_in_regions(T, chrom[i], start[i], end[i]) ? 1 : 0;
}
