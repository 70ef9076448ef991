"""Times csv_tra_call_gt, the call_gt of resolveTRA.py:260-309, on a config-3-shaped all-alignments table: the reads table
of synth.make_config(3, scale) in BAM order, with N breakpoint pairs drawn from a seed (both breakpoints on random
contigs, 3-20 supporting read ids each, bias 50 and gt_round 500 as cuteSV's defaults).

  python scripts/time_tra_call_gt.py [--scale 0.25] [--queries 10000] [--reps 20]

Prints the GPU name and power limit read in the same process, then for a host table and for the installed table
(aln=None): the k_tra_call_gt kernel time (CUDA events of one profiled call) and the whole call (median and p10-p90 of a
host clock around the call, which returns with the genotypes on the host).  The baseline is a Python loop over the same
queries and table: count_coverage per window as the reference scans its fetch() results, one candidate at a time, without
the BAM decoding the reference also does per candidate."""
import argparse
import bisect
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cutesv_b200 import _abi, synth  # noqa: E402
from cutesv_b200.engine import Engine  # noqa: E402


def make_case(scale, n_q, seed=3):
    cfg = synth.make_config(3, scale)
    reads, lens = cfg["reads"], np.asarray(cfg["lens"], np.int64)
    order = np.lexsort((np.arange(len(reads["chrom"])), reads["start"], reads["chrom"]))
    aln = {k: np.ascontiguousarray(v[order]) for k, v in reads.items()}
    rng = np.random.default_rng(seed)
    q = np.zeros(n_q, _abi.TRA_QUERY_DTYPE)
    q["chr1"], q["chr2"] = rng.integers(0, len(lens), n_q), rng.integers(0, len(lens), n_q)
    q["pos1"] = (rng.random(n_q) * lens[q["chr1"]]).astype(np.int64)
    q["pos2"] = (rng.random(n_q) * lens[q["chr2"]]).astype(np.int64)
    n_sup = rng.integers(3, 21, n_q)
    off = np.zeros(n_q + 1, np.int64)
    np.cumsum(n_sup, out=off[1:])
    ids = aln["read_id"][rng.integers(0, len(aln["read_id"]), int(off[-1]))].astype(np.int32)
    return lens, aln, q, off, ids


def host_loop(lens, aln, q, off, ids, bias, gt_round):
    """DR per query (-1: the first window returned -1), one query at a time."""
    by = {}
    for c in range(len(lens)):
        lo, hi = np.searchsorted(aln["chrom"], [c, c + 1])
        st, en = aln["start"][lo:hi], aln["end"][lo:hi]
        by[c] = (st.tolist(), en.tolist(), aln["read_id"][lo:hi].tolist(), aln["is_primary"][lo:hi].tolist(), int((en - st).max()) if hi > lo else 0)

    def count_coverage(c, s, e, sup, up, acc, xs, xe):
        st, en, rid, prim, span = by[c]
        it = pr = 0
        for i in range(bisect.bisect_left(st, s - span), len(st)):
            if st[i] >= e:
                break
            if en[i] <= s:
                continue
            it += 1
            if not prim[i]:
                continue
            pr += 1
            if st[i] < s and en[i] > e:
                if not (xs <= xe and st[i] < xs and en[i] > xe):
                    acc[0] += 1
                    acc[1] += rid[i] not in sup
                if acc[0] >= up:
                    return 1
            if it >= gt_round:
                return 1 if pr / it <= 0.2 else -1
        return 0

    dr = np.zeros(len(q), np.int32)
    for i, (chr1, chr2, pos1, pos2) in enumerate(q.tolist()):
        sup = set(ids[off[i]:off[i + 1]].tolist())
        n = int(off[i + 1] - off[i])
        up = 20 * n if n <= 2 else 9 * n if n <= 5 else 7 * n if n <= 15 else 5 * n
        acc = [0, 0]
        s, e = max(pos1 - bias, 0), min(pos1 + bias, int(lens[chr1]))
        r = count_coverage(chr1, s, e, sup, up, acc, 1, 0)
        if r == 0:
            s2, e2 = max(pos2 - bias, 0), min(pos2 + bias, int(lens[chr2]))
            count_coverage(chr2, s2, e2, sup, up, acc, *((s, e) if chr2 == chr1 else (1, 0)))
        dr[i] = -1 if r == -1 else acc[1]
    return dr


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return dict(median_ms=round(float(np.median(ts)), 3), p10_ms=round(float(np.percentile(ts, 10)), 3),
                p90_ms=round(float(np.percentile(ts, 90)), 3), calls=reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=0.25)
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    bias, gt_round = 50, 500
    lens, aln, q, off, ids = make_case(a.scale, a.queries)
    print(json.dumps(dict(gpu=subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                             capture_output=True, text=True).stdout.strip(),
                          alignments=len(aln["chrom"]), contigs=len(lens), queries=len(q), support_ids=len(ids))))
    eng = Engine(0, contig_lens=lens)
    eng.upload_alignments(aln)
    results = {}
    for name, tbl in (("host_table", aln), ("installed_table", None)):
        call = lambda: eng.tra_call_gt(q, off, ids, bias, gt_round, aln=tbl)   # noqa: E731
        results[name] = call()   # warm-up: allocations, module load
        eng.set_profiling(True)
        call()
        kt = {k: round(v[1], 4) for k, v in eng.kernel_times().items()}
        eng.set_profiling(False)
        print(json.dumps(dict(table=name, kernel_ms=kt, call=timed(call, a.reps))))
    assert all(np.array_equal(results["host_table"][k], results["installed_table"][k]) for k in ("dr", "dv", "gt", "status"))
    t0 = time.perf_counter()
    dr = host_loop(lens, aln, q, off, ids, bias, gt_round)
    loop_ms = (time.perf_counter() - t0) * 1e3
    got = results["host_table"]
    assert np.array_equal(dr, got["dr"]), "host loop and device disagree"
    print(json.dumps(dict(host_loop_ms=round(loop_ms, 1), noisy_queries=int((got["status"] == 2).sum()))))
    eng.close()


if __name__ == "__main__":
    main()
