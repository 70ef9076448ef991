"""Read sets of the signature-phase goldens (tests/golden/sigs_dropin.json.gz, oracle/gen_sigs_dropin_golden.py): seeded
synthetic alignment records in the layout tests/fake_pysam reads, the task windows, -include_bed regions and the
single_pipe arguments of every case.  The generator and the tests rebuild the same records from the case description."""
import gzip
import json
import os
import pickle

import numpy as np

from cutesv_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sigs_dropin.json.gz")
TYPES = ("DEL", "INS", "DUP", "INV", "TRA", "reads")
PIDS = (4101, 4102, 4103)
CASES = (
    # -mi -1: two insertions at one position stay two signatures that tie up to their sequence
    dict(name="mixed_s3", kind="mixed", seed=3, window=40000, bed=False,
         params=dict(min_length=30, min_mapq=20, max_split_parts=7, min_read_len=100, min_siglength=10, merge_del_threshold=0,
                     merge_ins_threshold=-1, MaxSize=100000)),
    dict(name="bed_split_all_s5", kind="mixed", seed=5, window=50000, bed=True,
         params=dict(min_length=30, min_mapq=0, max_split_parts=-1, min_read_len=100, min_siglength=10, merge_del_threshold=500,
                     merge_ins_threshold=100, MaxSize=-1)),
    # a draft assembly: 33 000 scaffolds in the header, reads on a few of them (string-order ranks above 32 767 included)
    dict(name="draft_33k", kind="draft", seed=11, window=30000, bed=False,
         params=dict(min_length=30, min_mapq=20, max_split_parts=7, min_read_len=500, min_siglength=10, merge_del_threshold=0,
                     merge_ins_threshold=100, MaxSize=100000)),
)


def _dup_pair(name, chrom, s1, dist):
    """A primary and a supplementary record of one read that start in different windows and both align across the same
    deletion: the same DEL signature in both windows (exact duplicates across worker pids)."""
    out = []
    for flag, start, ops in ((0, s1, [(0, dist), (2, 400), (0, 2000)]), (2048, s1 + dist - 3000, [(4, dist - 3000), (0, 3000), (2, 400), (0, 2000)])):
        r = synth.SynthRead()
        r.query_name, r.flag, r.mapq, r.reference_name, r.reference_start = name, flag, 60, chrom, start
        r.cigartuples = r.cigar = ops
        r.query_length = sum(l for o, l in ops if o in (0, 1, 4, 7, 8))
        r.reference_end = start + sum(l for o, l in ops if o in (0, 2, 3, 7, 8))
        r.query_sequence = ("ACGTTGCAAGCT" * (r.query_length // 12 + 1))[:r.query_length]
        r.tags = [("NM", 1)]
        out.append(r)
    return out


def _split_ins(name, chrom, s, gap):
    """A primary record whose SA segment continues the read `gap` bp further on: a split-read INS at (2s + 4000 + gap) / 2,
    an x.5 position for odd gaps (cuteSV:242-249)."""
    r = synth.SynthRead()
    r.query_name, r.flag, r.mapq, r.reference_name, r.reference_start = name, 0, 60, chrom, s
    r.cigartuples = r.cigar = [(0, 2000), (4, 1500)]
    r.query_length, r.reference_end = 3500, s + 2000
    r.query_sequence = ("GATTACACAT" * 350)[:3500]
    r.tags = [("NM", 1), ("SA", "%s,%d,+,2500S1000M,60,0;" % (chrom, s + 2000 + gap + 1))]
    return r


def dataset(case):
    """(fake-BAM dict(contigs, reads), tasks, bed regions per task or None)."""
    if case["kind"] == "draft":
        ds, _ = synth.synth_draft_bam_dataset(seed=case["seed"], n_header=33000, n_active=6, contig_len=40000, coverage=5)
        contigs, reads = ds["contigs"], ds["reads"]
    else:
        seed = case["seed"]
        ds, _ = synth.synth_bam_dataset(seed=seed, n_contigs=3, contig_len=60000, coverage=4, double_ins=0.5)
        reads = list(ds["reads"])
        extra, names, lens = synth.synth_alignments(seed, 120, 3)
        for r in extra:
            r.reference_start = r.reference_start % 150000
            r.reference_end = r.reference_start + sum(l for o, l in r.cigartuples if o in (0, 2, 3, 7, 8))
        reads += extra
        for k in range(3):
            reads += _dup_pair("dupread%d" % k, "chrA", 30000 + 300 * k, 15000)
            reads.append(_split_ins("splitins%d" % k, "chrB", 20000 + 40 * k, 1 + k))
        contigs = list(ds["contigs"]) + [(n, int(min(l, 200000))) for n, l in zip(names, lens)]
    active = sorted({r.reference_name for r in reads})
    lens = dict(contigs)
    tasks = []
    for c in active:
        for s in range(0, lens[c], case["window"]):
            tasks.append([c, s, min(s + case["window"], lens[c])])
    bed = None
    if case["bed"]:
        rng = np.random.default_rng(case["seed"])
        bed = []
        for t in tasks:
            lo = t[1] + int(rng.integers(0, (t[2] - t[1]) // 3))
            bed.append([] if rng.random() < 0.15 else [(lo, lo + int(rng.integers(3000, 20000))), (lo + 25000, lo + 30000)])
    return dict(contigs=contigs, reads=reads), tasks, bed


def write_fake_bam(path, ds):
    with open(path, "wb") as f:
        pickle.dump(ds, f)


def task_args(case, tmp, task, bed_regions):
    """The 12 single_pipe arguments (cuteSV:1058-1070) of one task."""
    p = case["params"]
    return ("unused.bam", p["min_length"], p["min_mapq"], p["max_split_parts"], p["min_read_len"], tmp, task, p["min_siglength"],
            p["merge_del_threshold"], p["merge_ins_threshold"], p["MaxSize"], bed_regions)


def as_tuples(lst):
    return [tuple(x) for x in lst]


def load():
    with gzip.open(GOLDEN, "rt") as f:
        return json.load(f)


def read_pid_dumps(path):
    out = []
    with open(path, "rb") as f:
        while True:
            try:
                out.append(pickle.load(f))
            except EOFError:
                return out


def write_pid_pickles(tmp, case_golden):
    """The reference-written pid pickles of a golden case, dump by dump in task order."""
    os.makedirs(os.path.join(tmp, "signatures"), exist_ok=True)
    for w, pid in zip(case_golden["windows"], case_golden["task_pid"]):
        for t in TYPES:
            with open("%ssignatures/%s%s.pickle" % (tmp, pid, t), "ab") as f:
                pickle.dump(as_tuples(w[t]), f)


def resolve_calls(tmp, sigs_index, min_support=2):
    """(type, contig, run_* argument tuple) of the reference's clustering phase (cuteSV:1116-1189) over a rebuilt work dir, with
    low support so that the small read sets yield calls; genotyping off (TRA's call_gt would re-open the BAM)."""
    out = []
    for chrom in sigs_index["DEL"]:
        out.append(("DEL", chrom, (tmp, chrom, "DEL", min_support, 0.5, 200, min(min_support, 5), "", False, 500, 1.0, sigs_index)))
    for chrom in sigs_index["INS"]:
        out.append(("INS", chrom, (tmp, chrom, "INS", min_support, 0.3, 100, min(min_support, 5), "", False, 500, 1.0, sigs_index)))
    for chrom in sigs_index["INV"]:
        out.append(("INV", chrom, (tmp, chrom, "INV", min_support, 500, 30, "", False, 100000, 500, sigs_index)))
    for chrom in sigs_index["DUP"]:
        out.append(("DUP", chrom, (tmp, chrom, min_support, 500, 30, "", False, 100000, 500, sigs_index)))
    for chrom in sigs_index["TRA"]:
        out.append(("TRA", chrom, (tmp, chrom, min_support, 0.6, 50, "", False, 500, sigs_index)))
    return out


def np_sort_sigs(svtype, cols, n_contigs):
    """csv_sort_sigs in numpy: stable lexsort on the documented key, adjacent duplicates dropped (INS: tie flags instead)."""
    n = len(cols["chrom"])
    if svtype == "reads":
        keys = [cols["chrom"]]
    elif svtype == "INS":
        keys = [cols["chrom"], cols["a"] >> 1, cols["b"], cols["read_id"]]
    elif svtype in ("INV", "TRA"):
        keys = [cols["chrom"], cols["c"], cols["a"], cols["b"], cols["read_id"]]
    else:
        keys = [cols["chrom"], cols["a"], cols["b"], cols["read_id"]]
    order = np.lexsort([np.arange(n)] + [np.asarray(k, np.int64) for k in reversed(keys)]) if n else np.zeros(0, np.int64)
    k = np.stack([np.asarray(x, np.int64)[order] for x in keys]) if n else np.zeros((len(keys), 0), np.int64)
    same = np.concatenate([[False], np.all(k[:, 1:] == k[:, :-1], axis=0)]) if n else np.zeros(0, bool)
    tie = same.astype(np.uint8) if svtype == "INS" else np.zeros(n, np.uint8)
    keep = np.ones(n, bool) if svtype in ("INS", "reads") else ~same
    order = order[keep]
    ch = np.asarray(cols["chrom"], np.int64)[order]
    off = np.searchsorted(ch, np.arange(n_contigs + 1), side="left").astype(np.int64)
    return dict(order=order.astype(np.int64), contig_off=off, ins_tie=tie[keep])
