// host_tables.h -- lookup tables the kernels consume, built on the HOST with the same libm the
// reference's CPython uses (glibc pow / log10), because cal_GL and cal_CIPOS go through libm and
// must match bit for bit (SURVEY.md section 7, hard part 1).
//   * cal_GL(c0, c1) is a pure function of two small ints: after rescale_read_counts
//     c0 + c1 <= 100, so a 101 x 101 table (+2 special cases) covers the whole domain.
//   * cal_CIPOS needs n ** 0.5 as libm pow evaluates it (differs from sqrt for some n).
#pragma once
#include <math.h>
#include <stdint.h>
#include <vector>
#include "../../include/cutesv_b200.h"

namespace csv {

// cal_GL after rescale (cuteSV_genotype.py:39-56); special cases handled by the caller
inline void host_cal_gl_core(int c0, int c1, csv_geno* g) {
    const double err = 0.1;
    const double prior = (double)(1.0 / 3.0);
    volatile double a00 = pow((1 - err), (double)c0), b00 = pow(err, (double)c1);
    volatile double a11 = pow(err, (double)c0), b11 = pow((1 - err), (double)c1);
    double gl00 = a00 * b00 * (1 - prior) / 2;
    double gl11 = a11 * b11 * (1 - prior) / 2;
    double gl01 = pow(0.5, (double)(c0 + c1)) * prior;
    double lp[3] = {log10(gl00), log10(gl01), log10(gl11)};
    double m = lp[0];
    if (lp[1] > m) m = lp[1];
    if (lp[2] > m) m = lp[2];
    double s = 0.0;
    for (int i = 0; i < 3; i++) s = s + pow(10.0, lp[i] - m);
    double lse = m + log10(s);
    double prob[3], P[3];
    for (int i = 0; i < 3; i++) {
        prob[i] = lp[i] - lse;
        if (prob[i] > 0.0) prob[i] = 0.0;
        P[i] = pow(10.0, prob[i]);
    }
    for (int i = 0; i < 3; i++) g->pl[i] = (int)nearbyint(-10 * log10(P[i]));
    int gq0 = (int)(-10 * log10(P[1] + P[2]));
    int gq1 = (int)(-10 * log10(P[0] + P[2]));
    int gq2 = (int)(-10 * log10(P[0] + P[1]));
    int gq = gq0;
    if (gq1 > gq) gq = gq1;
    if (gq2 > gq) gq = gq2;
    g->gq = gq;
    g->qual = fabs(nearbyint((-10 * log10(P[0])) * 10.0) / 10.0);
    int best = 0;
    if (prob[1] > prob[best]) best = 1;
    if (prob[2] > prob[best]) best = 2;
    g->gt = best;
    g->status = 0;
}

// table[c0*101+c1]; entries with c0+c1 > 100 are never addressed (gl_index rescales first)
inline std::vector<csv_geno> build_gl_table() {
    std::vector<csv_geno> t(10203);
    for (int c0 = 0; c0 <= 100; c0++)
        for (int c1 = 0; c1 <= 100; c1++) {
            csv_geno g;
            g.dr = c0; g.dv = c1; g.gt = -1; g.pl[0] = g.pl[1] = g.pl[2] = 0; g.gq = 0; g.status = 1; g.qual = 0.0;
            if (c0 + c1 <= 100) host_cal_gl_core(c0, c1, &g);   // (0, 0): call_gt of resolveTRA with no supporting reads
            t[c0 * 101 + c1] = g;
        }
    csv_geno s;
    s.dr = 3; s.dv = 1; s.gt = 1; s.pl[0] = 3; s.pl[1] = 3; s.pl[2] = 24; s.gq = 3; s.status = 0; s.qual = 3.0;
    t[10201] = s;  // cal_GL(3,1) cuteSV_genotype.py:34-35
    s.dr = 6; s.dv = 2; s.pl[2] = 45;
    t[10202] = s;  // cal_GL(6,2) :36-37
    return t;
}

inline std::vector<double> build_pow_half(uint32_t n) {
    std::vector<double> t(n);
    for (uint32_t i = 0; i < n; i++) {
        volatile double x = (double)i;
        t[i] = pow(x, 0.5);
    }
    return t;
}

}  // namespace csv
