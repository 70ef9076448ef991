"""Runs the REAL reference CLI core (main_ctrl) through the test-only fake pysam on a draft-assembly BAM: about 40 000
scaffolds in the header, reads on a few dozen of them (some with string-order ids above 32767), split reads that make TRA
between them, --genotype and -include_bed.  Commits the VCF body as tests/golden/cli_draft_40k.json.
Authoring container only:  CUTESV_REF_SRC=<cuteSV checkout>/src python -m oracle.gen_cli_golden_draft"""
import json
import os
import pickle
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "fake_pysam"))

SEED = 11
N_HEADER = 40000
FLAGS = ["--genotype", "-s", "3", "--threads", "4", "--max_cluster_bias_INS", "100", "--diff_ratio_merging_INS", "0.3",
         "--max_cluster_bias_DEL", "100", "--diff_ratio_merging_DEL", "0.3"]


def materialise(d):
    from cutesv_b200 import synth
    ds, fasta = synth.synth_draft_bam_dataset(SEED, N_HEADER)
    bam = os.path.join(d, "draft.bam")
    with open(bam, "wb") as f:
        pickle.dump(ds, f)
    fa = os.path.join(d, "draft.fa")
    with open(fa, "w") as f:
        f.write("".join(">%s\n%s\n" % (k, v) for k, v in fasta.items()))
    wd = os.path.join(d, "wd")
    os.mkdir(wd)
    return bam, fa, os.path.join(d, "draft.vcf"), wd, ds


def write_bed(d, ds):
    """-include_bed regions on the scaffolds that carry reads: most of each, with gaps that drop some loci."""
    names = sorted({r.reference_name for r in ds["reads"]})
    bed = os.path.join(d, "draft.bed")
    with open(bed, "w") as f:
        for k, n in enumerate(names):
            f.write("%s\t%d\t%d\n" % (n, 1000 + 3000 * (k % 3), 30000))
            f.write("%s\t%d\t%d\n" % (n, 36000, 58000 - 4000 * (k % 2)))
    return bed


def main():
    import pysam  # noqa: F401  (the fake one, first on sys.path)
    from oracle import ref_harness
    m = ref_harness.modules()
    from cuteSV.cuteSV_Description import parseArgs
    d = tempfile.mkdtemp()
    bam, fa, out, wd, ds = materialise(d)
    argv = [bam, fa, out, wd] + FLAGS + ["-include_bed", write_bed(d, ds)]
    m["main"].main_ctrl(parseArgs(argv), argv)
    lines = [l for l in open(out) if not l.startswith("##")]
    with open(os.path.join(ROOT, "tests", "golden", "cli_draft_40k.json"), "w") as f:
        json.dump(dict(flags=FLAGS, seed=SEED, n_header=N_HEADER, lines=lines), f)
    print(len(lines) - 1, "records")


if __name__ == "__main__":
    main()
