"""Times the signature rebuild of process_process_sigs_type (cuteSV:750-857) on N seeded signatures per type (and N reads
rows): tuples spread over three worker-pid pickles in a temporary work dir, positions on 24 contigs with duplicates and
INS ties.

  CUTESV_REF_SRC=<cuteSV checkout>/src python scripts/time_sigs_rebuild.py --impl ref   (the reference's Python, 1 CPU core)
  python scripts/time_sigs_rebuild.py --impl gpu                                         (the drop-in and Engine.sort_sigs)

--impl gpu prints the GPU name, power limit and SM clocks read in the same process, then per type:
  kernels        the summed CUDA-event times of the kernels of one profiled csv_sort_sigs call
  csv_sort_sigs  wall time of ONE csv_sort_sigs call on already uploaded columns (Engine.sort_sigs: kernels, the two
                 synchronisations, the D2H of order / offsets / tie flags)
  drop-in        the whole process_process_sigs_type (pickle load, conversion, upload, sort, pickle write)"""
import argparse
import os
import pickle
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TYPES = ("DEL", "INS", "DUP", "INV", "TRA", "reads")
PIDS = (101, 102, 103)


def make_tuples(t, n, seed=1):
    rng = np.random.default_rng(seed)
    chrom = ["chr%d" % k for k in rng.integers(1, 25, n)]
    pos = rng.integers(0, 50_000_000, n).tolist()
    ln = rng.integers(30, 5000, n).tolist()
    name = ["m64011/%d/ccs" % k for k in rng.integers(0, n // 4 + 1, n)]
    if t in ("DEL", "DUP"):
        out = list(zip(pos, ln, name, [t] * n, chrom))
    elif t == "INS":
        half = rng.random(n) < 0.05
        p = [x + 0.5 if h else x for x, h in zip(pos, half)]
        out = list(zip(p, ln, name, ["ACGT"[k % 4] * 8 for k in range(n)], ["INS"] * n, chrom))
    elif t == "INV":
        out = list(zip(["++" if k else "--" for k in rng.integers(0, 2, n)], pos, [p + l for p, l in zip(pos, ln)], name, ["INV"] * n, chrom))
    elif t == "TRA":
        out = list(zip(["ABCD"[k] for k in rng.integers(0, 4, n)], pos, ["chr%d" % k for k in rng.integers(1, 25, n)], ln, name, ["TRA"] * n, chrom))
    else:
        out = list(zip(pos, [p + l for p, l in zip(pos, ln)], rng.integers(0, 2, n).tolist(), name, chrom))
    out += out[: n // 50]   # exact duplicates
    return out


def write_pids(d, t, tuples):
    os.makedirs(d + "signatures", exist_ok=True)
    for j, pid in enumerate(PIDS):
        with open("%ssignatures/%s%s.pickle" % (d, pid, t), "wb") as f:
            pickle.dump(tuples[j::len(PIDS)], f)


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()   # every GPU call ends with a stream synchronise
        ts.append((time.perf_counter() - t0) * 1e3)
    return "median %.3f ms, p10-p90 %.3f-%.3f ms, %d calls" % (np.median(ts), np.percentile(ts, 10), np.percentile(ts, 90), reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", choices=("ref", "gpu"), required=True)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        d += "/"
        for t in TYPES:
            write_pids(d, t, make_tuples(t, a.n))
        if a.impl == "ref":
            from oracle import ref_harness
            main_mod = ref_harness.modules()["main"]
            for t in TYPES:
                print("reference process_process_sigs_type %s:" % t, timed(lambda: main_mod.process_process_sigs_type((t, d, list(PIDS), False)), a.reps))
            return
        from cutesv_b200 import cuteSV_signatures as S, runtime
        eng = runtime.get_engine()
        print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip())
        for t in TYPES:
            S.process_process_sigs_type((t, d, list(PIDS), False))   # warm-up: allocations, module load
            whole = timed(lambda: S.process_process_sigs_type((t, d, list(PIDS), False)), a.reps)
            tuples = S._load_pid_lists(d, list(PIDS), t)
            S.rebuild_type(t, tuples)   # leaves this type's columns on the device
            dev = timed(lambda: eng.sort_sigs(t), a.reps)
            eng.set_profiling(True)
            eng.sort_sigs(t)
            eng.set_profiling(False)
            kt = eng.kernel_times()
            print("%s: %d tuples; kernels %.3f ms (%d launches); csv_sort_sigs %s; drop-in process_process_sigs_type %s"
                  % (t, len(tuples), sum(v[1] for v in kt.values()), sum(v[0] for v in kt.values()), dev, whole))


if __name__ == "__main__":
    main()
