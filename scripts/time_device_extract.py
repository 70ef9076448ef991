"""Extraction of one ONT-ultra-long-shaped packet (synth.synth_cigar_packet as in scripts/bench_extract.py, plus seeded bases) two ways:

  host    pinned host packet -> csv_extract -> INS strings rebuilt on the host (packing.ins_block_from_packed + slow path)
  device  torch CUDA packet  -> csv_extract_device with the sequence arena (strings built on the GPU)

Reports per path the median / min / max wall time of the call plus the string build, and the device split from CUDA events
(profiling on, a run of its own): H2D or D2D copy stage, k_check_packet, k_extract, sequence kernels.  Checks that both paths
give equal signatures and strings.  One JSON line; the card name and power limit are read in the same run.
python scripts/time_device_extract.py [n_reads] [reps]"""
import collections
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

from cutesv_b200 import _abi, bamio, packing, synth
from cutesv_b200.engine import Engine

n_reads = int(sys.argv[1]) if len(sys.argv) > 1 else 50000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=60).stdout.strip()
    except Exception as e:   # reported, not fatal
        return "unknown (%s)" % e


def main():
    import torch
    pk, names, lens = synth.synth_cigar_packet(n_reads)
    rng = np.random.default_rng(7)
    nb = (pk["query_len"].astype(np.int64) + 1) // 2
    pk["seq_off"] = np.concatenate([[0], np.cumsum(nb)]).astype(np.int64)
    codes = np.array([1, 2, 4, 8], np.uint8)                  # A C G T
    pk["seq4"] = (codes[rng.integers(0, 4, int(nb.sum()))] << 4) | codes[rng.integers(0, 4, int(nb.sum()))]
    p = _abi.default_params()
    eng = Engine(0, params=p, contig_lens=lens)
    torch.cuda.set_device(0)
    pinned = eng.pin_packet(pk)
    dev = {k: (torch.from_numpy(np.ascontiguousarray(v).view(np.int32) if v.dtype == np.uint32 else np.ascontiguousarray(v)).cuda()) for k, v in pk.items()
           if k != "sa"}
    dev["sa"] = {k: torch.from_numpy(v).cuda() for k, v in pk["sa"].items()}
    host_only = {k: v for k, v in pinned.items() if k not in ("seq_off", "seq4")}

    def run_host():
        r = eng.extract(host_only)
        t1 = time.perf_counter()
        n = r["counts"]["INS"]
        po, pc, pieces = eng.fetch_ins_pieces(0, n, 0, r["n_pieces"])
        bases, off, rest = packing.ins_block_from_packed(pieces, po, pc, pk["seq4"], pk["seq_off"][:-1], pk["seq_off"][1:], pk["query_len"])
        store = packing.InsStore()
        store.add_block(bases, off)
        for i in rest.tolist():
            store[i] = packing.ins_sequence(pieces, int(po[i]), int(pc[i]), lambda rec: bamio.decode_seq(pk, rec),
                                            lambda rec: (pk["cigar"][pk["cigar_off"][rec]:pk["cigar_off"][rec + 1]], int(pk["ref_start"][rec])),
                                            (p.min_siglength, p.merge_ins_threshold))
        return store, time.perf_counter() - t1

    def run_device():
        eng.extract(dev)
        torch.cuda.synchronize()

    def timed(fn):
        t0 = time.perf_counter()
        out = fn()
        return time.perf_counter() - t0, out

    for _ in range(2):   # warm-up: module load, allocations of every buffer at this size
        run_host()
        run_device()
    wall = {"host": [], "device": []}
    host_rebuild = []
    for _ in range(reps):   # alternating, so that both see the same neighbours on a shared machine
        t, (store, tr) = timed(run_host)
        wall["host"].append(t * 1e3)
        host_rebuild.append(tr * 1e3)
        t, _ = timed(run_device)
        wall["device"].append(t * 1e3)

    # parity: signatures and (row, string) multisets of both paths
    run_host_out, _ = run_host()
    h = eng.fetch_extracted()
    host_seqs = list(run_host_out)
    run_device()
    d = eng.fetch_extracted()
    dev_seqs = eng.fetch_ins_seqs(np.arange(len(d["sigs"]["INS"]["chrom"])))

    def canon(ex, seqs):
        out = {t: collections.Counter(zip(*[c[k].tolist() for k in ("chrom", "a", "b", "read_id", "c")])) for t, c in ex["sigs"].items()}
        s = ex["sigs"]["INS"]
        out["INS+seq"] = collections.Counter(zip(s["a"].tolist(), s["b"].tolist(), s["read_id"].tolist(), seqs))
        return out
    equal = canon(h, host_seqs) == canon(d, dev_seqs)

    # device split from CUDA events (a run of its own: the events sit between the launches)
    eng.set_profiling(True)
    split = {}
    for name, fn in (("host", lambda: eng.extract(host_only)), ("device", run_device)):
        acc = collections.defaultdict(float)
        for _ in range(reps):
            fn()
            st = eng.stage_ms()
            acc["copy_stage_ms"] += st["h2d"] / reps
            for k, (n, ms) in eng.kernel_times().items():
                acc[k] += ms / reps
        split[name] = dict(acc)
    eng.set_profiling(False)

    def stats(v):
        return dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v)))
    print(json.dumps(dict(card=card(), n_reads=n_reads, n_cigar_ops=int(len(pk["cigar"])), query_bases=int(pk["query_len"].sum()),
                          ins_rows=int(len(d["sigs"]["INS"]["chrom"])), ins_bytes=int(sum(map(len, dev_seqs))), reps=reps,
                          host_wall_ms=stats(wall["host"]), host_rebuild_ms=stats(host_rebuild), device_wall_ms=stats(wall["device"]),
                          device_split_ms=split, equal=equal)))
    eng.close()
    if not equal:
        sys.exit(1)


if __name__ == "__main__":
    main()
