"""Small end-to-end run for compute-sanitizer (memcheck / racecheck / initcheck): adversarial cases,
a pile-up (CTA-class clusters), extraction, the TRA genotyper and the standalone signature sort."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from cutesv_b200 import _abi, synth, packing
from cutesv_b200.engine import Engine

e = Engine(0)
n = 0
for seed in (1, 34, 144):
    cfg = synth.adversarial(seed)
    p = _abi.default_params(**cfg["params"])
    e.set_params(p); e.set_contigs(cfg["lens"])
    order = np.lexsort((np.arange(len(cfg["reads"]["chrom"])), cfg["reads"]["start"], cfg["reads"]["chrom"]))
    e.upload_alignments({k: v[order] for k, v in cfg["reads"].items()})
    n += len(e.cluster(cfg["sigs"], cfg["reads"])[0])
    e.upload_alignments(None)
cfg = synth.make_config(2, 0.01)
e.set_params(_abi.default_params(**cfg["params"])); e.set_contigs(cfg["lens"])
n += len(e.cluster(cfg["sigs"], cfg["reads"])[0])
# all five SV types on their stream lanes + the grouped-by-contig upload path
cfg = synth.make_config(3, 0.02)
e.set_params(_abi.default_params(**cfg["params"])); e.set_contigs(cfg["lens"])
nc = len(cfg["lens"])
n += len(e.cluster({k: _abi.group_by_contig(v, nc) for k, v in cfg["sigs"].items()}, _abi.group_by_contig(cfg["reads"], nc), grouped=True)[0])
rng = np.random.default_rng(7)
names, lens = synth.contigs(0.01)
m = 700
sig = dict(chrom=np.zeros(m, np.int32), a=(20000 + rng.integers(0, 300, m)).astype(np.int32), b=(300 + rng.integers(0, 40, m)).astype(np.int32),
           read_id=rng.integers(0, 500, m).astype(np.int32), c=None)
reads = dict(chrom=np.zeros(500, np.int32), start=np.full(500, 1000, np.int32), end=np.full(500, 60000, np.int32), read_id=np.arange(500, dtype=np.int32),
             is_primary=np.ones(500, np.uint8))
e.set_params(_abi.default_params(min_support=10, genotype=1)); e.set_contigs(lens)
n += len(e.cluster({"DEL": sig}, reads)[0])
rd, cn, cl = synth.synth_alignments(3, 150)
rn = sorted(set(r.query_name for r in rd))
pk = packing.pack_alignments(rd, {x: i for i, x in enumerate(cn)}, {x: i for i, x in enumerate(rn)})
e.set_params(_abi.default_params(min_support=2, min_mapq=0, min_read_len=100, genotype=1)); e.set_contigs(cl)
e.extract(pk); e.cluster_device(0x1F); n += len(e.fetch()[0])
# append-mode extraction (two packets into the device-resident columns), read-id remap, repeated calls (CUDA graph capture + replay)
e.extract_reset()
e.extract(pk, append=True); e.extract(pk, append=True)
e.remap_read_ids(np.arange(len(rn), dtype=np.int32))
for _ in range(3):
    e.cluster_device(0x1F)
n += len(e.fetch()[0])
# standalone signature sort + de-duplication (csv_sort_sigs) over the extracted columns and the reads table, with their
# record column (csv_extract_records / csv_fetch_records)
e.set_extract_records(True); e.extract(pk); e.set_extract_records(False)
for t in list(_abi.TYPE_NAMES) + ["reads"]:
    e.fetch_records(t)
    n += len(e.sort_sigs(t)["order"])
print("sanitize run ok, candidates:", n)
