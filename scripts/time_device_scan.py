"""Times the device scan (Engine.scan + rank_names: record filter, -include_bed and the TRA genotyper's alignment table on the
GPU) against the host route a device pipeline takes without it: the numpy record filter and cli.bed_filter, bamio.subset_packet
+ flat_seq, the named device extraction of the subset, and the alignment table built in Python (provisional ids through a
name -> record dict, argsort by contig, one gather through name_rank_tensor, upload_alignments).  Both routes end with the
ranks and the alignment table on the device.  The packets are decoded from a synthetic coordinate-sorted BAM (scripts/bench_cli.py's
writer) before the timing: the device route starts from torch CUDA packets, the host route from the decoder's host packets (it
uploads the subsets it keeps), as the test of the host route does.
Prints the card, its power limit, and per route the median with min / max over the repetitions (the routes alternate).

    python scripts/time_device_scan.py [n_reads] [--reps 3]"""
import argparse
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from cutesv_b200 import bamio, cli  # noqa: E402
from cutesv_b200.engine import Engine  # noqa: E402

import bench_cli  # noqa: E402
import device_packet_util as dpu  # noqa: E402
import name_util  # noqa: E402
from time_device_names import card, stats  # noqa: E402


def write_bed(path, tasks, rng):
    """Two 20 kb regions per window on average, some straddling window borders."""
    with open(path, "w") as f:
        for t in tasks:
            lo = int(t[1])
            for _ in range(2):
                s = lo + int(rng.integers(-5_000, max(int(t[2]) - lo, 1)))
                f.write("%s\t%d\t%d\n" % (t[0], max(s, 0), max(s, 0) + 20_000))


def device_route(eng, dev_packets, layout):
    tasks, bed, chrom_id = layout
    eng.extract_reset()
    eng.set_scan_regions(tasks, bed, chrom_id)
    for d in dev_packets:
        eng.scan(d, alignments=True)
    eng.rank_names()


def host_route(eng, host_packets, layout):
    import torch
    tasks, bed, chrom_id = layout
    starts, first_task = cli.window_starts(tasks, chrom_id)
    eng.extract_reset()
    eng.set_scan_regions([], None, {})
    aln, aln_names, rec_of_name, n_rec = [], [], {}, 0
    for pk, names in host_packets:
        has_cigar = pk["cigar_off"][1:] > pk["cigar_off"][:-1]
        v = np.flatnonzero(has_cigar & (pk["chrom"] >= 0))
        aln.append(dict(chrom=pk["chrom"][v], start=pk["ref_start"][v], end=pk["ref_end"][v],
                        is_primary=((pk["flag"][v] == 0) | (pk["flag"][v] == 16)).astype(np.uint8)))
        aln_names += [names[i] for i in v.tolist()]
        keep = has_cigar & (pk["flag"] != 256) & (pk["flag"] != 272) & (pk["chrom"] >= 0)
        if bed is not None:
            cli.bed_filter(pk, keep, bed, starts, first_task)
        k = np.flatnonzero(keep)
        sub = dpu.flat_seq(bamio.subset_packet(pk, k))
        rec_names = [names[i] for i in k.tolist()]
        for j, nm in enumerate(rec_names):
            rec_of_name.setdefault(nm, n_rec + j)
        n_rec += len(rec_names)
        eng.extract(name_util.named(dpu.to_device(sub), rec_names), append=True)
    eng.rank_names()
    a = {k: np.concatenate([x[k] for x in aln]) for k in aln[0]}
    # a read seen only in filtered records has no extracted record, so this route cannot give it its rank: record 0 stands in
    # (same cost; the device route gets it right)
    prov = np.array([rec_of_name.get(nm, 0) for nm in aln_names], dtype=np.int64)
    order = np.argsort(a["chrom"], kind="stable")
    dev = torch.device("cuda", eng.device)
    cols = {k: torch.from_numpy(np.ascontiguousarray(v[order])).to(dev) for k, v in a.items()}
    cols["read_id"] = eng.name_rank_tensor()[torch.from_numpy(prov[order]).to(dev)].contiguous()
    eng.upload_alignments(cols)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("n_reads", nargs="?", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="scan_")
    bam = os.path.join(tmp, "synth.bam")
    n, fa = bench_cli.write_bam_parallel(bam, a.n_reads, os.cpu_count() or 4)
    rd = bamio.BamReader(bam, threads=8)
    stats_ = rd.index_statistics()
    tasks, contig_info = cli.task_windows(stats_, rd.get_reference_length, 16, 10_000_000)
    chrom_names = sorted(c[0] for c in contig_info)
    chrom_id = {nm: i for i, nm in enumerate(chrom_names)}
    rd.set_chrom_ids(chrom_id)
    host_packets = []
    while True:
        pk = rd.next_packet(cli.PACKET_READS)
        if pk is None:
            break
        names = rd.names()
        host_packets.append((pk, [names[i] for i in pk["read_id"].tolist()]))
    rd.close()
    dev_packets = [name_util.named(dpu.to_device(pk), names) for pk, names in host_packets]
    bed_path = os.path.join(tmp, "regions.bed")
    write_bed(bed_path, tasks, np.random.default_rng(1))
    eng = Engine(0)
    eng.set_contigs(np.array([dict(contig_info)[nm] for nm in chrom_names], dtype=np.int64))
    name, pl = card()
    print("card: %s, power limit %s; %d records in %d packets, %d windows" % (name, pl, n, len(host_packets), len(tasks)))
    for label, bed in (("no BED", None), ("-include_bed", cli.load_bed(bed_path, tasks))):
        layout = (tasks, bed, chrom_id)
        times = {"device": [], "host": []}
        for rep in range(a.reps + 1):   # the first round warms up both routes
            for route, fn, arg in (("device", device_route, dev_packets), ("host", host_route, host_packets)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(eng, arg, layout)
                torch.cuda.synchronize()
                if rep:
                    times[route].append(time.perf_counter() - t0)
        print("%s: device scan %s; host route %s" % (label, stats(times["device"]), stats(times["host"])))
    eng.close()


if __name__ == "__main__":
    main()
