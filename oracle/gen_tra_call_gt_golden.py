"""Stores what the UNMODIFIED reference's call_gt of cuteSV_resolveTRA (resolveTRA.py:260-309, with count_coverage of
cuteSV_genotype.py:72-93) returns for breakpoint pairs over a fake BAM (tests/golden/tra_call_gt.json.gz): the BAM's contigs
and records (flags 0, 16, 256, 272, 2048 and 2064) and, per case, the arguments, the returned tuple and its value types.

Cases: count_coverage returning -1; 1 through the gt_round ratio test; 1 through up_bound in each threshold_ref_count tier;
0 and a second window on another contig, one of which would return -1 and one on a contig without records; chr1 == chr2
with overlapping and with disjoint windows; windows clamped at 0 and at the contig end; records starting or ending exactly
on a window bound; records overlapping a window from more than the window's length before it; gt_round reached at scan
positions 0, 31 and 32 (lanes 0 and 31 of one warp step, lane 0 of the next); a pile-up of more than 2 000 records;
support lists with duplicates and names absent from the BAM; cal_GL's special case (3, 1); seeded random pairs.
The generator checks that every designed case takes its intended path.

Needs the reference (ref_harness.py):  CUTESV_REF_SRC=<cuteSV checkout>/src python -m oracle.gen_tra_call_gt_golden
"""
import gzip
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import tra_call_gt_golden as tg  # noqa: E402
from oracle import ref_harness  # noqa: E402

OUT = tg.GOLDEN
CONTIGS = [["chr1", 200_000], ["chr2", 100_000], ["chr3", 50_000], ["chr4", 30_000], ["chr5", 50_000]]
SECONDARY = (256, 272, 2048, 2064)


class Bam(object):
    def __init__(self):
        self.records, self.n_names, self.n_sec = [], 0, 0

    def prim(self, chrom, start, end):
        """A primary record (flag 0 / 16) of a fresh read; returns its name."""
        name = "r%05d" % self.n_names
        self.records.append([chrom, int(start), int(end), 16 * (self.n_names & 1), name])
        self.n_names += 1
        return name

    def sec(self, chrom, start, end, name=None):
        """A secondary or supplementary record (256, 272, 2048, 2064), by default of a read named after it."""
        flag = SECONDARY[self.n_sec % 4]
        self.n_sec += 1
        self.records.append([chrom, int(start), int(end), flag, name or "s%05d" % self.n_sec])


def build(rng):
    b = Bam()
    cases = []

    def case(name, pos_1, pos_2, chr_1, chr_2, sup, bias=50, gt_round=500, path=None):
        cases.append(dict(name=name, pos_1=pos_1, pos_2=pos_2, chr_1=chr_1, chr_2=chr_2, read_id_list=list(sup), bias=bias,
                          gt_round=gt_round, path=path))

    # -1: 30 primary records inside the window, none spanning, gt_round 20
    P = 10_000
    names = [b.prim("chr1", P - 40 + i, P + 200) for i in range(30)]
    case("noisy", P, 40_000, "chr1", "chr2", names[:2], gt_round=20, path=(-1,))
    # 1 by the ratio: 2 spanning primaries, then mostly secondary records; gt_round 20
    P = 20_000
    sp = [b.prim("chr1", P - 100, P + 100) for _ in range(2)]
    for i in range(40):
        if i % 9 == 4:
            b.prim("chr1", P - 30 + i, P + 300)
        else:
            b.sec("chr1", P - 30 + i, P + 300, name=sp[i % 2] if i % 7 == 0 else None)
    case("ratio", P, 40_000, "chr1", "chr2", sp[:1], gt_round=20, path=(1,))
    # 1 by up_bound in every threshold_ref_count tier: n_sup 2 (40), 4 (36), 10 (70), 20 (100)
    for k, n_sup in enumerate((2, 4, 10, 20)):
        P = 30_000 + 2_000 * k
        up = 20 * n_sup if n_sup <= 2 else 9 * n_sup if n_sup <= 5 else 7 * n_sup if n_sup <= 15 else 5 * n_sup
        spans = []
        for i in range(up + 10):
            if i % 6 == 5:
                b.sec("chr1", P - 400 + i, P + 400)
            spans.append(b.prim("chr1", P - 400 + i, P + 300 + i))
        case("up_bound_%d" % n_sup, P, 40_000, "chr1", "chr2", spans[3:3 + n_sup], path=(1,))
    # 0, then the second window: 3 spanning primaries and 5 others on chr1 (8 records: under any gt_round used below)
    P = 40_000
    w1 = [b.prim("chr1", P - 80 + i, P + 90) for i in range(3)]
    for i in range(5):
        (b.prim if i % 2 else b.sec)("chr1", P - 40 + 10 * i, P + 500)
    P2 = 10_000   # chr2: 5 spanning primaries
    w2 = [b.prim("chr2", P2 - 70 + i, P2 + 70) for i in range(5)]
    b.sec("chr2", P2 - 10, P2 + 20)
    case("second_window", 40_000, P2, "chr1", "chr2", [w1[0], w2[1], w2[2]], path=(0, 0))
    case("second_window_sup_dup_absent", 40_000, P2, "chr1", "chr2", [w2[1], w2[1], w1[0], "absent1", "absent2", w2[4]], path=(0, 0))
    case("second_window_no_records", 40_000, 20_000, "chr1", "chr3", ["absent1"], path=(0, 0))   # DR 3, DV 1: cal_GL's (3, 1)
    P2 = 20_000   # chr2: 3 spanning primaries, then 30 primaries inside the window: -1 at gt_round 20 (ignored)
    for i in range(3):
        b.prim("chr2", P2 - 90 + i, P2 + 90)
    for i in range(30):
        b.prim("chr2", P2 - 30 + i, P2 + 400)
    case("second_window_noisy", 40_000, P2, "chr1", "chr2", [w1[1]], gt_round=20, path=(0, -1))
    case("first_contig_without_records", 30_000, P2, "chr3", "chr2", [w1[1]], gt_round=20, path=(0, -1))
    # chr1 == chr2: overlapping windows [49950, 50050] / [50010, 50110], disjoint ones [51950, 52050] / [52950, 53050]
    P = 50_000
    both = b.prim("chr1", P - 100, P + 200)
    only1 = b.prim("chr1", P - 60, P + 55)
    only2 = b.prim("chr1", P + 5, P + 120)
    b.sec("chr1", P + 6, P + 130)
    case("same_contig_overlapping", P, P + 60, "chr1", "chr1", [only2], path=(0, 0))
    P = 52_000
    b.prim("chr1", P - 100, P + 1_100)
    b.prim("chr1", P - 60, P + 60)
    b.prim("chr1", P + 940, P + 1_070)
    b.prim("chr1", P + 945, P + 1_060)
    case("same_contig_disjoint", P, P + 1_000, "chr1", "chr1", [both, only1], path=(0, 0))
    case("same_contig_reversed_pair", P + 1_000, P, "chr1", "chr1", [both], path=(0, 0))
    # windows clamped at 0 (chr2, pos 20) and at the contig end (chr2, pos 99 980: e = 100 000)
    b.prim("chr2", 0, 200)
    b.prim("chr2", 0, 60)
    b.sec("chr2", 5, 100)
    L = 100_000
    b.prim("chr2", L - 200, L)
    b.prim("chr2", L - 120, L + 5)   # spans [99930, 100000] only because the window is clamped at the contig end
    b.prim("chr2", L - 60, L)
    case("clamp_zero_and_end", 20, L - 20, "chr2", "chr2", ["absent1"], path=(0, 0))
    case("no_support", 20, L - 20, "chr2", "chr2", [], path=(0, 1))   # up_bound 0: the first spanning record returns
    case("no_support_no_spanning", 20, 20_000, "chr2", "chr3", [], path=(0, 0))   # cal_GL(0, 0)
    case("clamp_end_first", L - 20, 20, "chr2", "chr2", ["r00000"], bias=200, path=(0, 0))
    # records on the bounds of [59950, 60050]
    P = 60_000
    s, e = P - 50, P + 50
    b.prim("chr1", s - 150, s)        # end == s: not fetched
    b.prim("chr1", s - 1, e + 1)      # spans
    b.prim("chr1", s, e + 50)         # start == s: fetched, not spanning
    b.prim("chr1", s - 50, e)         # end == e: fetched, not spanning
    b.prim("chr1", s - 2, e + 1)      # spans
    b.prim("chr1", e, e + 100)        # start == e: ends the scan
    b.prim("chr1", e + 5, e + 100)
    case("bounds", P, P + 300, "chr1", "chr1", ["absent1"], path=(0, 0))
    # records overlapping the window from far before it (start 5 000 before), with short records in between that end
    # before the window: scanned, not fetched
    P = 70_000
    far = [b.prim("chr1", P - 5_000 + 10 * i, P + 5_000) for i in range(4)]
    for i in range(50):
        b.prim("chr1", P - 4_000 + 50 * i, P - 3_900 + 50 * i)
    b.sec("chr1", P - 4_500, P + 200)
    case("far_starts", P, P + 3_000, "chr1", "chr1", far[1:2], path=(0, 0))
    # gt_round reached at scan positions 0, 31 and 32 on chr5: records k = 0..99 start at P - 60 + k, all 300 long, so the
    # scan starts at record 0; primaries at k in {0, 3, 31, 32} and at even k >= 40
    P = 10_000
    lane_names = {}
    for k in range(100):
        if k in (0, 3, 31, 32) or (k >= 40 and k % 2 == 0):
            lane_names[k] = b.prim("chr5", P - 60 + k, P + 240 + k)
        else:
            b.sec("chr5", P - 60 + k, P + 240 + k)
    case("round_at_0", P, 40_000, "chr5", "chr2", ["absent1"], gt_round=1, path=(-1,))
    case("round_at_3", P, 40_000, "chr5", "chr2", ["absent1"], gt_round=2, path=(-1,))
    case("round_at_31", P, 40_000, "chr5", "chr2", [lane_names[0]], gt_round=32, path=(1,))
    case("round_at_32", P, 40_000, "chr5", "chr2", [lane_names[3]], gt_round=33, path=(1,))
    case("round_at_64", P, 40_000, "chr5", "chr2", ["absent1"], gt_round=64, path=(-1,))
    # a pile-up of 2 100 records on chr4 around 15 000: 70% primary spanning
    P = 15_000
    starts = np.sort(rng.integers(P - 2_000, P + 40, 2_100))
    pile = []
    for st in starts.tolist():
        if rng.random() < 0.7 and st < P - 50:
            pile.append(b.prim("chr4", st, int(rng.integers(P + 51, P + 2_000))))
        elif rng.random() < 0.5:
            b.prim("chr4", st, int(rng.integers(st + 1, P + 2_000)))
        else:
            b.sec("chr4", st, int(rng.integers(st + 1, P + 2_000)))
    sup = [pile[int(i)] for i in rng.integers(0, len(pile), 400)] + ["absent%d" % i for i in range(600)]
    case("pileup_whole_scan", P, 10_000, "chr4", "chr2", sup, gt_round=3_000, path=(0, 0))   # up_bound 5 000: the scan runs through
    case("pileup_up_bound", P, 10_000, "chr4", "chr2", sup[:200], gt_round=3_000, path=(1,))   # up_bound 1 000
    case("pileup_round", P, 10_000, "chr4", "chr2", sup[:100], gt_round=500, path=(-1,))      # up_bound 500
    # background on chr1 [100 000, 200 000) and chr2 [40 000, 90 000), and seeded random pairs over it
    for chrom, lo, hi, n in (("chr1", 100_000, 200_000, 1_200), ("chr2", 40_000, 90_000, 600)):
        for st in np.sort(rng.integers(lo, hi, n)).tolist():
            ln = int(rng.integers(100, 3_000))
            if rng.random() < 0.8:
                b.prim(chrom, st, st + ln)
            else:
                b.sec(chrom, st, st + ln)
    bg = [r[4] for r in b.records if r[0] in ("chr1", "chr2") and r[1] >= 40_000 and r[3] in (0, 16)]
    for k in range(40):
        c1, c2 = ("chr1", "chr2") if k % 3 else ("chr1", "chr1")
        p1 = int(rng.integers(100_000, 200_000))
        p2 = int(rng.integers(40_000, 90_000)) if c2 == "chr2" else int(rng.integers(100_000, 200_000))
        sup = [bg[int(i)] for i in rng.integers(0, len(bg), int(rng.integers(1, 20)))]
        case("random_%02d" % k, p1, p2, c1, c2, sup, bias=int(rng.choice([50, 200, 1000])), gt_round=int(rng.choice([20, 100, 500])))
    return b.records, cases


def main():
    mods = ref_harness.modules()
    tra = mods["tra"]
    records, cases = build(np.random.default_rng(20261018))
    with tempfile.TemporaryDirectory() as d:
        bam = os.path.join(d, "tra.bam")
        tg.write_bam(bam, CONTIGS, records)
        for c in cases:
            res = tra.call_gt(bam, c["pos_1"], c["pos_2"], c["chr_1"], c["chr_2"], c["read_id_list"], c["bias"], c["gt_round"])
            c["result"], c["types"] = list(res), [type(v).__name__ for v in res]
        # the path of every designed case: the statuses count_coverage returned, observed through a wrapper
        real, seen = tra.count_coverage, []
        tra.count_coverage = lambda *a: seen.append(real(*a)) or seen[-1]
        try:
            for c in cases:
                del seen[:]
                tra.call_gt(bam, c["pos_1"], c["pos_2"], c["chr_1"], c["chr_2"], c["read_id_list"], c["bias"], c["gt_round"])
                want = c.pop("path")
                assert want is None or tuple(seen) == want, (c["name"], seen, want)
        finally:
            tra.count_coverage = real
    assert any(c["types"][-1] == "float" for c in cases) and any(c["types"][-1] == "float64" for c in cases)
    blob = json.dumps(dict(contigs=CONTIGS, records=records, cases=cases), separators=(",", ":")) + "\n"
    with open(OUT, "wb") as f, gzip.GzipFile(fileobj=f, mode="wb", mtime=0, filename="") as z:   # mtime 0: reproducible bytes
        z.write(blob.encode())
    print("wrote %s: %d records, %d cases" % (OUT, len(records), len(cases)))


if __name__ == "__main__":
    main()
