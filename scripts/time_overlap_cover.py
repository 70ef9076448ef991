"""Times overlap_cover (cuteSV_genotype.py:95-159) on one contig-sized case: one 50 Mb contig at 30x coverage of 15 kb
reads (100 000 rows, 10 % non-primary) and 10 000 DEL-style windows (position +- 200), generated from a seed.

  CUTESV_REF_SRC=<cuteSV checkout>/src python scripts/time_overlap_cover.py --impl ref   (the reference's Python, 1 CPU core)
  python scripts/time_overlap_cover.py --impl gpu                                         (the drop-in and Engine.overlap_cover)

--impl gpu prints the GPU name, power limit and SM clocks read in the same process, median and p10-p90 of every timed
call, and the per-kernel CUDA-event times of one profiled call."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def make_case(seed=1, contig=50_000_000, n_reads=100_000, n_win=10_000, bias=200):
    rng = np.random.default_rng(seed)
    start = np.sort(rng.integers(0, contig - 15_000, n_reads))
    ln = np.clip(rng.normal(15_000, 4_000, n_reads), 500, 60_000).astype(np.int64)
    prim = (rng.random(n_reads) < 0.9).astype(int)
    reads_list = [[int(s), int(s + l), int(p), "m64011/%d/ccs" % i] for i, (s, l, p) in enumerate(zip(start, ln, prim))]
    svs_list = [(max(int(p) - bias, 0), int(p) + bias) for p in np.sort(rng.integers(0, contig, n_win))]
    return svs_list, reads_list


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()   # the GPU calls end with a stream synchronise
        ts.append((time.perf_counter() - t0) * 1e3)
    return "median %.3f ms, p10-p90 %.3f-%.3f ms, %d calls" % (np.median(ts), np.percentile(ts, 10), np.percentile(ts, 90), reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", choices=("ref", "gpu"), required=True)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    svs_list, reads_list = make_case()
    if a.impl == "ref":
        from oracle import ref_harness
        G = ref_harness.modules()["genotype"]
        print("reference overlap_cover:", timed(lambda: G.overlap_cover(svs_list, reads_list), max(a.reps // 4, 3)))
        return
    from cutesv_b200 import cuteSV_genotype, runtime
    eng = runtime.get_engine()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    cols, _, _ = cuteSV_genotype.reads_columns(reads_list)
    win = cuteSV_genotype.windows_of(*cuteSV_genotype._bounds(svs_list))
    cuteSV_genotype.overlap_cover(svs_list, reads_list)   # warm-up: allocations, module load
    print("drop-in overlap_cover:", timed(lambda: cuteSV_genotype.overlap_cover(svs_list, reads_list), a.reps))
    print("Engine.overlap_cover on columns:", timed(lambda: eng.overlap_cover(win, cols), a.reps))
    eng.set_profiling(True)
    eng.overlap_cover(win, cols)
    eng.set_profiling(False)
    print("kernel ms:", json.dumps({k: round(v[1], 4) for k, v in eng.kernel_times().items()}))


if __name__ == "__main__":
    main()
