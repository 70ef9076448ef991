"""Where the INS / DEL back end's time goes, on one config (CUDA events on the lane streams, lanes on).
python scripts/time_backend.py [config] [scale] [steps]

Prints, per type:
  * the interval from the end of k_part_filter to the end of the lane (k_select_heads, the cluster kernels and the side
    stream's join), with every lane running as it does unprofiled: programmatic launches, side streams, INS and DEL
    lanes side by side.  Only the graph replay is off, and one event pair per lane sits in the stream;
  * the kept-cluster sizes by route: <= 32 (register kernel), 33-128 (k_cluster_warp), 129-2048 (k_cluster_block in
    shared memory), larger (global scratch), from Engine.counters() of a call of that type alone;
  * the k_select_heads tiles (2048 survivors each) against the CTA slots of one wave: 256 threads and 32 registers per
    thread (-Xptxas -v) make eight CTAs per SM, and the host launches min(tiles of the signature count, one wave);
  * the back-end kernels one by one (lanes serialised, CUDA events around every launch): time per launch;
  * the counts that size the work, per type: density-filter survivors, kept clusters by size class, members and
    candidates emitted."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from cutesv_b200 import _abi, synth
from cutesv_b200.engine import Engine

SEL_TILE = 2048
SEL_CTAS_PER_SM = 8

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
types = [t for t in ("DEL", "INS") if t in cfg["sigs"]]
mask = sum(1 << _abi.TYPE_IDS[k] for k in cfg["sigs"])
e.upload(cfg["sigs"], cfg["reads"])
for _ in range(3):
    e.cluster_device(mask)
e.fetch()
e.set_profiling("lanes")
for _ in range(steps):
    e.cluster_device(mask)
e.fetch()
kt = e.kernel_times()
e.set_profiling(False)
e.set_lanes(False)
e.set_profiling(True)
for _ in range(steps):
    e.cluster_device(mask)
e.fetch()
kser = e.kernel_times()
e.set_profiling(False)
e.set_lanes(True)
n_sm = torch.cuda.get_device_properties(0).multi_processor_count
print("config %d scale %g, %s: %d signatures, %d steps" % (cid, scale, card, cfg["n_sigs"], steps))
out = {"card": card, "config": cid, "scale": scale}
for t in types:
    nm = "back end<%s>" % t
    n, ms = kt.get(nm, (0, 0.0))
    e.cluster_device(1 << _abi.TYPE_IDS[t])
    e.fetch()
    c = e.counters()
    kept, big, giant, small = c["kept"][t], c["big"][t], c["giant"][t], c["small_path"]
    surv = c["domain"][t]
    n_sig = len(cfg["sigs"][t]["a"])
    tiles = (surv + SEL_TILE - 1) // SEL_TILE
    ctas = min(max((n_sig + SEL_TILE - 1) // SEL_TILE, 1), SEL_CTAS_PER_SM * n_sm)
    row = dict(backend_us=1e3 * ms / n if n else None, candidates=c["n_cand"], kept=kept, le32=small, c33_128=kept - small - big, c129_2048=big - giant,
               gt2048=giant, members=c["members"][t], survivors=surv, select_tiles=tiles, select_ctas=ctas, sms=n_sm)
    out[t] = row
    print("  %s: filter end -> lane end %s us; kept %d: <=32 %d, 33-128 %d, 129-2048 %d, >2048 %d (members %d, candidates %d); "
          "k_select_heads %d tiles of %d survivors, %d CTAs launched (%d SMs)"
          % (t, "%.1f" % row["backend_us"] if n else "n/a (no density filter)", kept, small, row["c33_128"], row["c129_2048"],
             giant, row["members"], row["candidates"], tiles, surv, ctas, n_sm))
BACK_END = ("k_part_filter", "k_select_heads", "k_cluster_small", "k_cluster_warp<DEL", "k_cluster_warp<INS", "k_cluster_block<INDEL")
print("  back-end kernels, lanes serialised (per launch):")
out["kernels_us"] = {}
for nm, (n, ms) in sorted(kser.items()):
    if nm.startswith(BACK_END):
        out["kernels_us"][nm] = 1e3 * ms / n
        print("    %-40s launches/step %4.1f  %8.2f us" % (nm, n / steps, 1e3 * ms / n))
print(json.dumps(out))
