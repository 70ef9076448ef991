"""Where the serial tail of a csv_cluster step goes: everything after the lane join (order scans, k_permute, the bin scan,
k_windows, the reads pass, the pair test, k_finalize), on one config.
python scripts/time_tail.py [config] [scale] [steps]

Prints:
  * the interval from the lane join to the end of the call's chain, with the lanes, programmatic launches and side streams
    running as they do unprofiled (Engine.set_profiling("lanes"): one event pair on the ctx stream, no graph replay), and
    the whole csv_cluster step on the same calls (host clock around calls that end in a synchronise);
  * every tail kernel's time (lanes serialised, CUDA events around each launch) and, for the reads pass, the bytes it must
    read (17 B per reads row) over its time against HBM bandwidth (MEASURED_PEAKS.json if present, else the data sheet);
  * the counts that size the work, computed on the host from the candidates the step returns: candidates, genotype windows,
    occupied bins, (read, window) pairs P (the library's counter), pairs whose read covers the window (the supporting-id
    test runs on these) and the supporting-id slice lengths of the windowed candidates;
  * the card's name, power limit and max SM clock, read in the same run."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

from cutesv_b200 import _abi, synth
from cutesv_b200.engine import Engine
from genotype_edges import layout, n_windows, windows_of_candidates

TAIL = ("k_scan_excl<8>", "k_permute", "k_scan_excl<4>", "k_windows<1>", "k_reads_pass<true>", "k_reads_pass<false>",
        "k_pairs_test<true>", "k_pairs_test<false>", "k_finalize", "k_fold_status", "k_tra_genotype")


def hbm_gbs():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
        except (ValueError, KeyError):
            pass
    return 3350.0, "data sheet, not measured"


def pair_counts(cands, names, reads, p, lens):
    """(windows, occupied bins, covering pairs, covering pairs whose read supports the candidate): the reads pass's rule,
    restated with numpy on linear coordinates (row ends clamped to their contig, primary rows only)."""
    L = layout(p, lens)
    off, shift = L["off"], L["shift"]
    nw = n_windows(cands)
    win = windows_of_candidates(cands, p)
    ci, wi = np.nonzero(np.arange(2)[None, :] < nw[:, None])
    ch = cands["chrom"][ci].astype(np.int64)
    S = off[ch] + win["s2"][ci, wi] // 2
    E = off[ch] + (win["e2"][ci, wi] + 1) // 2
    bins = np.minimum(S >> shift, L["n_bins"] - 1)
    prim = np.asarray(reads["is_primary"]) != 0
    rc = np.asarray(reads["chrom"], np.int64)[prim]
    RS = off[rc] + np.asarray(reads["start"], np.int64)[prim]
    RE = np.minimum(off[rc] + np.asarray(reads["end"], np.int64)[prim], off[rc + 1] - 1)
    rid = np.asarray(reads["read_id"])[prim]
    o = np.argsort(RS, kind="stable")
    RS, RE, rid = RS[o], RE[o], rid[o]
    max_len = int((RE - RS).max(initial=0))
    cover = support = 0
    for k in range(len(S)):
        lo, hi = np.searchsorted(RS, S[k] - max_len), np.searchsorted(RS, S[k], side="right")
        m = RE[lo:hi] >= E[k]
        n = int(m.sum())
        if not n:
            continue
        cover += n
        i = ci[k]
        sup = names[cands["names_off"][i]:cands["names_off"][i] + cands["names_cnt"][i]]
        support += int(np.isin(rid[lo:hi][m], sup).sum())
    return len(S), len(np.unique(bins)), cover, support


cid = int(sys.argv[1]) if len(sys.argv) > 1 else 2
scale = float(sys.argv[2]) if len(sys.argv) > 2 else 1.0
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 20
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
except OSError:
    card = "unknown"
cfg = synth.make_config(cid, scale)
p = _abi.default_params(**cfg["params"])
e = Engine(0, params=p, contig_lens=cfg["lens"])
mask = sum(1 << _abi.TYPE_IDS[k] for k in cfg["sigs"])
if "TRA" in cfg["sigs"]:
    r = cfg["reads"]
    order = np.lexsort((np.arange(len(r["chrom"])), r["start"], r["chrom"]))
    e.upload_alignments({k: v[order] for k, v in r.items()})
e.upload(cfg["sigs"], cfg["reads"])
for _ in range(3):
    e.cluster_device(mask)
res = e.fetch()
ctr = e.counters()

# the tail as it runs: lanes, programmatic launches and side streams on; one event pair on the ctx stream
e.set_profiling("lanes")
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(steps):
    e.cluster_device(mask)
e.fetch()
step_ms = 1e3 * (time.perf_counter() - t0) / steps
kt = e.kernel_times()
e.set_profiling(False)
n_tail, ms_tail = kt.get("tail", (0, 0.0))
tail_us = 1e3 * ms_tail / n_tail if n_tail else None

# per-kernel times, lanes serialised
e.set_lanes(False)
e.set_profiling(True)
for _ in range(steps):
    e.cluster_device(mask)
e.fetch()
kt = e.kernel_times()
e.set_profiling(False)
e.close()

cands, _, names = res
n_win, n_occ, n_cover, n_support = pair_counts(cands, names, cfg["reads"], p, cfg["lens"])
nw = n_windows(cands)
ncnt = cands["names_cnt"][nw > 0]
n_reads = len(cfg["reads"]["chrom"])
peak, peak_src = hbm_gbs()
print("config %d scale %g, %s: %d signatures, %d reads rows, %d steps" % (cid, scale, card, cfg["n_sigs"], n_reads, steps))
print("  tail (lane join -> end of chain), lanes overlapped: %s us per step; host step (profiling marks on) %.3f ms"
      % ("%.1f" % tail_us if tail_us is not None else "n/a", step_ms))
out = {"card": card, "config": cid, "scale": scale, "tail_us": tail_us, "step_ms_marked": step_ms, "kernels": {}}
tot = 0.0
for nm in TAIL:
    if nm not in kt:
        continue
    n, ms = kt[nm]
    us = 1e3 * ms / steps
    tot += us
    row = {"launches_per_step": n / steps, "us_per_step": us}
    line = "  %-22s %4.1f launches/step  %8.2f us/step" % (nm, n / steps, us)
    if nm.startswith("k_reads_pass"):
        gbs = 17.0 * n_reads / (us * 1e-6) / 1e9
        floor_us = 17.0 * n_reads / (peak * 1e9) * 1e6
        row.update(gbs=gbs, floor_us=floor_us, over_floor=us / floor_us)
        line += "  %.0f GB/s, floor %.1f us at %.0f GB/s (%s), %.2fx the floor" % (gbs, floor_us, peak, peak_src, us / floor_us)
    out["kernels"][nm] = row
    print(line)
print("  sum of tail kernels, lanes serialised: %.1f us/step" % tot)
counts = dict(candidates=int(len(cands)), windows=n_win, occupied_bins=n_occ, bins=int(layout(p, cfg["lens"])["n_bins"]),
              pairs=int(ctr["pairs"]), pairs_covering=n_cover, pairs_covering_supporting=n_support,
              names_cnt_mean=float(ncnt.mean()) if len(ncnt) else 0.0, names_cnt_max=int(ncnt.max(initial=0)))
out["counts"] = counts
print("  counts: " + ", ".join("%s %s" % kv for kv in counts.items()))
print(json.dumps(out))
