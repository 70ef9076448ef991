"""Times the device read-name ranking (csv_rank_names) and INS tie ordering (csv_order_ins_ties) against the host passes a
device pipeline makes without them.  Prints the card, its power limit, medians with min / max over the repetitions (the two
paths alternate), and per-kernel times from the library's profiling events.

    python scripts/time_device_names.py [--reps 3] [--sizes 1000000,9300000] [--ins-records 2100000]
    (--sizes "" or --ins-records 0 skips that part)

Name ranking: named device packets of records that yield no signatures (empty CIGAR), with ONT UUID, PacBio movie/zmw/ccs and
64-byte shared-prefix names; host side: np.unique over an `S` array and Python sorted().  Tie ordering: records with four
35 bp insertions each (8.4 M INS rows at the default size), the last 1 % of records repeating the first 1 % with other bases,
so that their INS rows tie; host side: fetch four INS columns, cli.ins_tie_rows, fetch the tie rows' strings,
cli.ins_tie_swaps, csv_swap_ins_rows."""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from cutesv_b200 import _abi, cli  # noqa: E402
from cutesv_b200.engine import Engine  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except Exception as e:   # reported, not guessed
        pl = "unknown (%s)" % e
    return name, pl


def stats(xs):
    xs = sorted(xs)
    return "median %.2f ms (min %.2f, max %.2f, n=%d)" % (1e3 * xs[len(xs) // 2], 1e3 * xs[0], 1e3 * xs[-1], len(xs))


def names_of(shape, n, rng):
    if shape == "ont_uuid":
        hexd = np.frombuffer(b"0123456789abcdef", np.uint8)
        digits = hexd[rng.integers(0, 16, (n, 32))]
        out = np.full((n, 36), ord("-"), np.uint8)
        for a, b, o in ((0, 8, 0), (8, 12, 9), (12, 16, 14), (16, 20, 19), (20, 32, 24)):
            out[:, o:o + b - a] = digits[:, a:b]
        return out.reshape(-1), np.arange(n + 1, dtype=np.int64) * 36
    if shape == "pacbio_ccs":
        raw = [("m64011_190830_220126/%d/ccs" % z).encode() for z in rng.integers(0, 180_000_000, n).tolist()]
    else:   # 64 shared bytes, then a number
        raw = [("x" * 64 + "%d" % z).encode() for z in rng.integers(0, 10 * n, n).tolist()]
    off = np.zeros(n + 1, np.int64)
    np.cumsum([len(r) for r in raw], out=off[1:])
    return np.frombuffer(b"".join(raw), np.uint8).copy(), off


def empty_packet(n, dev):
    import torch
    z = torch.zeros(n, dtype=torch.int32, device=dev)
    pk = {f: z for f in _abi.READ_FIELDS if f != "read_id"}
    pk["flag"] = torch.full((n,), 4, dtype=torch.int32, device=dev)
    pk["cigar_off"] = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    pk["sa_off"] = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    pk["cigar"] = torch.zeros(0, dtype=torch.int32, device=dev)
    pk["sa"] = {f: torch.zeros(0, dtype=torch.int32, device=dev) for f in _abi.SA_FIELDS}
    return pk


def time_ranking(eng, sizes, reps, dev):
    import torch
    rng = np.random.default_rng(1)
    for n in sizes:
        pk = empty_packet(n, dev)
        for shape in ("ont_uuid", "pacbio_ccs", "prefix64"):
            b, off = names_of(shape, n, rng)
            pk["names"] = torch.from_numpy(b).to(dev)
            pk["name_off"] = torch.from_numpy(off).to(dev)
            py = [b[off[i]:off[i + 1]].tobytes().decode() for i in range(n)]
            sarr = np.array([s.encode() for s in py], dtype="S%d" % max(int(np.diff(off).max()), 1))
            t_dev, t_np, t_py = [], [], []
            eng.extract(pk)   # warm-up
            eng.rank_names()
            for r in range(reps):
                eng.extract(pk)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                nd = eng.rank_names()   # blocks until the ranks are on the device
                t_dev.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                u, inv = np.unique(sarr, return_inverse=True)
                t_np.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                srt = {s: i for i, s in enumerate(sorted(set(py)))}
                rk = [srt[s] for s in py]
                t_py.append(time.perf_counter() - t0)
            assert nd == len(u) == len(srt)
            print("rank %-10s n=%8d  device rank_names %s | host np.unique %s | host sorted %s" % (shape, n, stats(t_dev), stats(t_np), stats(t_py)))
            del rk, inv
            eng.set_profiling(True)
            eng.extract(pk)
            eng.rank_names()
            kt = {k: v for k, v in eng.kernel_times().items() if "name" in k or "rs_" in k or "scan" in k or "remap" in k}
            eng.set_profiling(False)
            print("    kernels: " + ", ".join("%s %d x %.3f ms" % (k, v[0], v[1]) for k, v in sorted(kt.items(), key=lambda kv: -kv[1][1])))


def ins_packet(n, rng):
    """n records on one contig, each with CIGAR 150M 35I 150M 35I 150M 35I 150M 35I 150M; the last 1 % repeat the first 1 %."""
    cig_one = np.array([150 << 4 | 0, 35 << 4 | 1] * 4 + [150 << 4 | 0], dtype=np.uint32)
    qlen = 5 * 150 + 4 * 35
    k = n // 100
    start = (np.arange(n, dtype=np.int64) % (n - k)) * 500   # int32 coordinates: 2.1 M records stay below 2^31
    pk = dict(chrom=np.zeros(n, np.int32), ref_start=start.astype(np.int32), ref_end=(start + 750).astype(np.int32),
              flag=np.zeros(n, np.int32), mapq=np.full(n, 60, np.int32), query_len=np.full(n, qlen, np.int32))
    pk["cigar"] = np.tile(cig_one, n).view(np.int32)
    pk["cigar_off"] = np.arange(n + 1, dtype=np.int64) * len(cig_one)
    pk["sa_off"] = np.zeros(n + 1, np.int64)
    pk["sa"] = {f: np.zeros(0, np.int32) for f in _abi.SA_FIELDS}
    nb = (qlen + 1) // 2
    pk["seq4"] = rng.integers(0, 256, n * nb).astype(np.uint8)
    pk["seq_off"] = np.arange(n + 1, dtype=np.int64) * nb
    names = ["read_%d" % (i % (n - k)) for i in range(n)]
    return pk, names, int(start.max()) + 10_000


def time_ties(eng, n, reps, dev):
    import torch
    rng = np.random.default_rng(2)
    pk, names, clen = ins_packet(n, rng)
    eng.set_params(_abi.default_params(min_mapq=0, min_read_len=100))
    eng.set_contigs(np.array([clen], np.int64))
    b = np.frombuffer("".join(names).encode(), np.uint8).copy()
    off = np.zeros(n + 1, np.int64)
    np.cumsum([len(s) for s in names], out=off[1:])
    d = {k: (torch.from_numpy(v).to(dev) if not isinstance(v, dict) else {kk: torch.from_numpy(vv).to(dev) for kk, vv in v.items()})
         for k, v in pk.items()}
    d["names"], d["name_off"] = torch.from_numpy(b).to(dev), torch.from_numpy(off).to(dev)

    def fresh():
        eng.extract(d)
        eng.rank_names()
        torch.cuda.synchronize()

    def host():
        c = eng.fetch_sig_cols("INS", cols=("chrom", "a", "b", "read_id"))
        tie = cli.ins_tie_rows(c["chrom"], c["a"], c["b"], c["read_id"])
        pairs = cli.ins_tie_swaps(c["chrom"], c["a"], c["b"], c["read_id"], dict(zip(tie.tolist(), eng.fetch_ins_seqs(tie))))
        eng.swap_ins_rows(pairs)
        return len(pairs)
    fresh()
    eng.order_ins_ties()   # warm-up
    t_dev, t_host = [], []
    for r in range(reps):
        fresh()
        t0 = time.perf_counter()
        moved = eng.order_ins_ties()
        t_dev.append(time.perf_counter() - t0)
        fresh()
        t0 = time.perf_counter()
        n_pairs = host()
        t_host.append(time.perf_counter() - t0)
    print("ties  INS rows=%d (moved %d rows, host %d swaps)  device order_ins_ties %s | host route %s"
          % (eng._ex_counts[_abi.CSV_INS], moved, n_pairs, stats(t_dev), stats(t_host)))
    fresh()
    eng.set_profiling(True)
    eng.order_ins_ties()
    kt = eng.kernel_times()
    eng.set_profiling(False)
    print("    kernels: " + ", ".join("%s %d x %.3f ms" % (k, v[0], v[1]) for k, v in sorted(kt.items(), key=lambda kv: -kv[1][1])[:8]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="1000000,9300000")
    ap.add_argument("--ins-records", type=int, default=2_100_000)
    a = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    name, pl = card()
    print("card: %s, power limit %s" % (name, pl))
    eng = Engine(0, contig_lens=[1_000_000])
    if a.sizes:
        time_ranking(eng, [int(x) for x in a.sizes.split(",")], a.reps, dev)
    if a.ins_records:
        time_ties(eng, a.ins_records, a.reps, dev)
    eng.close()


if __name__ == "__main__":
    main()
