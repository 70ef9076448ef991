"""Cost of the contig count: the same seeded draft-assembly workload (synth.draft_assembly: reads and signatures of all five
types on 40 scaffolds of 50 Mb, 25 when there are only 25 contigs) with 25, 10^5 and 10^6 contigs in the table, the ones
without signatures about 1 kb long.  Reports per contig count:
  - csv_cluster step time (all types, --genotype, all-alignments table; CUDA-graph replays, mean over --steps),
  - csv_upload_alignments wall time (H2D copies + contig index, ends in a stream synchronise; median of --reps),
  - the linear coordinate's span (contig lengths + max(bias)+1 padding per contig) and whether it fits 32 bits,
  - whether INS and DEL took the 32-bit partitioned front end (k_part_filter).
One JSON line per contig count, then the card, its power limit and SM clocks.
python scripts/time_many_contigs.py [--steps 20] [--reps 20] [--sizes 25,100000,1000000]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from cutesv_b200 import _abi, synth  # noqa: E402
from cutesv_b200.engine import Engine  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [x.strip() for x in out.splitlines()[0].split(",")])) if out else {}


def one(n, steps, reps):
    # signatures on 50 Mb scaffolds (a density at which the INS/DEL filter engages), the rest small (median 1 kb), so that
    # the contig count itself, through the per-contig padding, decides whether the linear coordinate fits 32 bits
    case = synth.draft_assembly(n, seed=20261015, n_active=min(n, 40), active_len=50000000, n_reads=80000, scale=10.0,
                                median_len=1000.0)
    p = _abi.default_params(**case["params"])
    r = case["reads"]
    order = np.lexsort((np.arange(len(r["chrom"])), r["start"], r["chrom"]))
    aln = {k: np.ascontiguousarray(v[order]) for k, v in r.items()}
    e = Engine(0, params=p, contig_lens=case["lens"])
    pad = max(p.bias_del, p.bias_ins, p.bias_inv, p.bias_dup, p.bias_tra, p.gt_bias_ins) + 1   # csv_set_params
    span = int(case["lens"].sum()) + n * pad
    res = dict(n_contigs=n, n_sigs=case["n_sigs"], n_aln=len(aln["chrom"]), linear_span=span, linear_span_fits_32_bits=span < (1 << 32))
    ts = []
    for _ in range(reps + 2):
        t0 = time.perf_counter()
        e.upload_alignments(aln)
        ts.append(time.perf_counter() - t0)
    res["upload_alignments_ms"] = round(1e3 * float(np.median(ts[2:])), 3)
    try:
        e.upload(case["sigs"], case["reads"])
        for _ in range(3):
            e.cluster_device(0x1F)
        e.counts()
        t0 = time.perf_counter()
        for _ in range(steps):
            e.cluster_device(0x1F)
        e.counts()   # ends in a stream synchronise
        res["cluster_step_ms"] = round(1e3 * (time.perf_counter() - t0) / steps, 3)
        res["n_cand"] = e.counts()[0]
        e.set_profiling(True)
        e.cluster_device(0x1F)
        e.fetch()
        kt = e.kernel_times()
        res["indel_partitioned_front_end"] = "k_part_filter" in kt
    except Exception as err:   # a build without large-contig TRA support
        res["cluster_error"] = str(err)
    e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sizes", default="25,100000,1000000")
    a = ap.parse_args()
    for n in [int(x) for x in a.sizes.split(",")]:
        print(json.dumps(one(n, a.steps, a.reps)), flush=True)
    print(json.dumps(dict(card=card())), flush=True)


if __name__ == "__main__":
    main()
