"""Stores what the UNMODIFIED reference's genotype helpers compute on adversarial inputs (tests/golden/genotype_dropin.json.gz):

  overlap_cover   cuteSV_genotype.overlap_cover(svs_list, reads_list): the four dicts (key order kept, sets sorted)
  assign_gt       cuteSV_genotype.assign_gt on the reference's own overlap_cover output of a named overlap_cover case and
                  seeded support lists
  call_gt         resolveINDEL / resolveDUP / resolveINV call_gt over a work dir written by cutesv_b200.workdir

Cases cover non-primary rows, names repeated within a window and across the two DUP / INV windows, rows starting or
ending exactly on a window bound, zero-length rows, x.5 windows, windows clamped at 0, a pile-up of more than 2048 rows
on one window, windows with e <= s (the reference raises KeyError; the index is recorded) and a contig missing from
reads.pickle.

Needs the reference (ref_harness.py):  CUTESV_REF_SRC=<cuteSV checkout>/src python -m oracle.gen_genotype_golden
"""
import gzip
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cutesv_b200 import workdir  # noqa: E402
from oracle import ref_harness  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "genotype_dropin.json.gz")
GRID = 50   # coordinates on a coarse grid, so that rows often start or end exactly on a window bound


def rand_reads(rng, n, span, n_names, long_frac=0.2, zero_frac=0.05, prim_frac=0.8):
    rows = []
    for _ in range(n):
        s = int(rng.integers(0, span // GRID)) * GRID + (int(rng.integers(0, 3)) if rng.random() < 0.3 else 0)
        if rng.random() < zero_frac:
            ln = 0
        elif rng.random() < long_frac:
            ln = int(rng.integers(20, 120)) * GRID
        else:
            ln = int(rng.integers(1, 30)) * GRID
        rows.append([s, s + ln, 1 if rng.random() < prim_frac else int(rng.choice([0, 2])), "read%03d" % int(rng.integers(0, n_names))])
    return rows


def rand_windows(rng, n, span, biases):
    out = []
    for _ in range(n):
        c = int(rng.integers(0, span // GRID)) * GRID
        b = biases[int(rng.integers(0, len(biases)))]
        out.append([max(c - b, 0), c + b])
    return out


def dict_rows(d4):
    it, pn, cov, ovl = d4
    assert list(it) == list(pn) == list(cov) == list(ovl)
    return [[k, it[k], pn[k], sorted(cov[k]), sorted(ovl[k])] for k in cov]


def overlap_cases(G, rng):
    cases = []
    svs = rand_windows(rng, 40, 20000, [100, 150, 37.5, 250.5]) + [[0, 120], [0, 0.5], [100.3, 900.7], [4000, 4000.5]]
    cases.append(dict(name="mixed", svs=svs, reads=rand_reads(rng, 250, 20000, 40)))
    pile = [[int(rng.integers(0, 4)) * GRID, 1400 + int(rng.integers(0, 4)) * GRID, 1 if rng.random() < 0.9 else 0, "p%d" % int(rng.integers(0, 400))]
            for _ in range(2100)]
    pile += rand_reads(rng, 50, 5000, 30)
    cases.append(dict(name="pileup", svs=[[200, 1200], [1000, 1000.5], [0, 3000], [1400, 1500]], reads=pile))
    cases.append(dict(name="no_reads", svs=[[10, 20], [0, 5.5]], reads=[]))
    cases.append(dict(name="no_windows", svs=[], reads=rand_reads(rng, 20, 3000, 5)))
    bad = rand_windows(rng, 10, 5000, [100])
    bad[3] = [700, 700]
    bad[7] = [650, 600]
    cases.append(dict(name="empty_window", svs=bad, reads=rand_reads(rng, 80, 5000, 10)))
    bad = rand_windows(rng, 10, 5000, [100])
    bad[2] = [300, 250.5]
    bad[8] = [300, 250.5]
    cases.append(dict(name="reversed_windows_tie", svs=bad, reads=rand_reads(rng, 80, 5000, 10)))
    reads = rand_reads(rng, 50, 5000, 10)
    reads[11] = [900, 850, 1, "bad"]
    cases.append(dict(name="reversed_read", svs=rand_windows(rng, 10, 5000, [100]) + [[850, 850]], reads=reads))
    for c in cases:
        try:
            c["result"] = dict_rows(G.overlap_cover([tuple(w) for w in c["svs"]], c["reads"]))
        except KeyError as e:
            c["key_error"] = e.args[0]
    return cases


def assign_cases(G, rng, oc):
    out = []
    for c in oc:
        if "result" not in c or not c["result"]:
            continue
        it, pn, cov, _ = G.overlap_cover([tuple(w) for w in c["svs"]], c["reads"])
        names = sorted({r[3] for r in c["reads"]}) + ["absent1", "absent2"]
        rid = {}
        for k in sorted(cov):
            picks = [names[int(i)] for i in rng.integers(0, len(names), int(rng.integers(0, 12)))]
            rid[k] = picks + picks[:int(rng.integers(0, 2))]   # duplicates in a support list count in DV
        res = G.assign_gt(it, pn, cov, rid)
        out.append(dict(case=c["name"], read_id=[[k, v] for k, v in rid.items()],
                        result=[[a, b, gt, gl, gq, str(q)] for a, b, gt, gl, gq, q in res]))
    return out


def names_for(rng, pool, k):
    return list(dict.fromkeys(pool[int(i)] for i in rng.integers(0, len(pool), k)))


def call_gt_cases(mods, rng):
    reads = {"chr1": rand_reads(rng, 400, 30000, 60), "chr2": rand_reads(rng, 200, 12000, 25, long_frac=0.5)}
    # a pile-up on chr3: more than 2048 rows cover the windows around 2000
    reads["chr3"] = [[int(rng.integers(0, 10)) * GRID, 4000 + int(rng.integers(0, 10)) * GRID, 1 if rng.random() < 0.9 else 0,
                      "p%d" % int(rng.integers(0, 400))] for _ in range(2100)]
    pool = {c: sorted({r[3] for r in rows}) + ["nowhere"] for c, rows in reads.items()}
    cases = []
    for chrom, n_c in (("chr1", 15), ("chr2", 8), ("chr3", 3), ("chrX", 4)):
        p = pool.get(chrom, ["x1", "x2"])
        span = 30000 if chrom != "chr3" else 4000
        for svtype, bias in (("DEL", 200), ("INS", 1000)):
            cand = []
            for _ in range(n_c):
                pos = int(rng.integers(0, span // GRID)) * GRID
                search = pos if rng.random() < 0.7 else int(rng.integers(0, 300))
                item = [chrom, svtype, pos, int(rng.integers(30, 500)) * (-1 if svtype == "DEL" else 1), int(rng.integers(2, 12)), "-3,3", "-1,1",
                        search, names_for(rng, p, int(rng.integers(1, 12)))]
                if svtype == "INS":
                    item.append("ACGT" * int(rng.integers(1, 5)))
                cand.append(item)
            cases.append(dict(name="%s_%s" % (svtype, chrom), module="INDEL", chr=chrom, bias=bias, svtype=svtype, candidates=cand))
        cand = []
        for _ in range(n_c):
            bp1 = int(rng.integers(0, span // GRID)) * GRID
            cand.append([chrom, "DUP", bp1, bp1 + int(rng.integers(1, 40)) * 25 + int(rng.integers(0, 2)), names_for(rng, p, int(rng.integers(1, 12)))])
        cases.append(dict(name="DUP_%s" % chrom, module="DUP", chr=chrom, bias=501, candidates=cand))
        cand = []
        for _ in range(n_c):
            bp1 = int(rng.integers(0, span // GRID)) * GRID
            ln = int(rng.integers(1, 60)) * 25
            sup = names_for(rng, p, int(rng.integers(1, 12)))
            cand.append([chrom, "INV", bp1, ln, len(sup), "++" if rng.random() < 0.5 else "--", sup, bp1 + ln])
        cases.append(dict(name="INV_%s" % chrom, module="INV", chr=chrom, bias=int(rng.choice([500, 501, 77])), candidates=cand))
    # bp2 == bp1: the window half-width is 0, so both windows have e == s
    cases.append(dict(name="DUP_zero_width", module="DUP", chr="chr1", bias=500,
                      candidates=[["chr1", "DUP", 1000, 1500, ["read001"]], ["chr1", "DUP", 2000, 2000, ["read002"]]]))
    with tempfile.TemporaryDirectory() as d:
        path = d + "/"
        idx = workdir.write_workdir(path, {"reads": [tuple(r) + (c,) for c, rows in sorted(reads.items()) for r in rows]})
        for c in cases:
            m = mods["indel"] if c["module"] == "INDEL" else mods["dup"] if c["module"] == "DUP" else mods["inv"]
            cand = [list(x) for x in c["candidates"]]
            try:
                if c["module"] == "INDEL":
                    c["result"] = m.call_gt(path, c["chr"], cand, c["bias"], c["svtype"], idx)
                else:
                    c["result"] = m.call_gt(path, c["chr"], cand, c["bias"], idx)
            except KeyError as e:
                c["key_error"] = e.args[0]
    return reads, cases


def main():
    mods = ref_harness.modules()
    G = mods["genotype"]
    rng = np.random.default_rng(20261015)
    oc = overlap_cases(G, rng)
    ac = assign_cases(G, rng, oc)
    reads, gc = call_gt_cases(mods, rng)
    blob = json.dumps(dict(overlap_cover=oc, assign_gt=ac, call_gt_reads=reads, call_gt=gc), separators=(",", ":")) + "\n"
    with open(OUT, "wb") as f, gzip.GzipFile(fileobj=f, mode="wb", mtime=0, filename="") as z:   # mtime 0: reproducible bytes
        z.write(blob.encode())
    print("wrote %s: %d overlap_cover, %d assign_gt, %d call_gt cases" % (OUT, len(oc), len(ac), len(gc)))


if __name__ == "__main__":
    main()
