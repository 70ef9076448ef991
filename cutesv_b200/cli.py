"""`cuteSV <bam> <ref> <vcf> <work_dir> [flags]` -- the reference's CLI shell around the H100 path.

Same positionals, flags, defaults and pre-flight errors as the reference (cuteSV_Description.py:53-263,
cuteSV:992-1011).  BAM decoding: the native BGZF/BAM decoder (bamio.py) for .bam input, pysam for CRAM/SAM; everything between decoded records and
candidate rows runs through the C-ABI: csv_extract (replaces Pool#1), csv_cluster (Pool#2 + Pool#3,
including the TRA genotyper, which reads a packed all-alignments table instead of re-opening the BAM).
VCF formatting is host code (cutesv_b200/vcf.py).
"""
import argparse
import logging
import os
import sys
import time

import numpy as np

from . import _abi, packing, rows, vcf, workdir

VERSION = vcf.VERSION
PACKET_READS = 50000


def build_parser():
    p = argparse.ArgumentParser(prog="cuteSV", description="Long-read SV detection (cuteSV hot path on H100).",
                                formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--version", "-v", action="version", version="%(prog)s {version}".format(version=VERSION))
    p.add_argument("input", metavar="[BAM]", type=str, help="Sorted .bam file from NGMLR or Minimap2.")
    p.add_argument("reference", type=str, help="The reference genome in fasta format.")
    p.add_argument("output", type=str, help="Output VCF format file.")
    p.add_argument("work_dir", type=str, help="Work-directory for distributed jobs")
    p.add_argument("-t", "--threads", default=16, type=int)
    p.add_argument("-b", "--batches", default=10000000, type=int)
    p.add_argument("-S", "--sample", default="NULL", type=str)
    p.add_argument("--retain_work_dir", action="store_true")
    p.add_argument("--write_old_sigs", action="store_true")
    p.add_argument("--report_readid", action="store_true")
    p.add_argument("--ignore_sequence", action="store_true")
    g = p.add_argument_group("Collection of SV signatures")
    g.add_argument("-p", "--max_split_parts", default=7, type=int)
    g.add_argument("-q", "--min_mapq", default=20, type=int)
    g.add_argument("-r", "--min_read_len", default=500, type=int)
    g.add_argument("-md", "--merge_del_threshold", default=0, type=int)
    g.add_argument("-mi", "--merge_ins_threshold", default=100, type=int)
    g.add_argument("-include_bed", default=None, type=str)
    g = p.add_argument_group("Generation of SV clusters")
    g.add_argument("-s", "--min_support", default=10, type=int)
    g.add_argument("-l", "--min_size", default=30, type=int)
    g.add_argument("-L", "--max_size", default=100000, type=int)
    g.add_argument("-sl", "--min_siglength", default=10, type=int)
    g = p.add_argument_group("Computing genotypes")
    g.add_argument("--genotype", action="store_true")
    g.add_argument("--gt_round", default=500, type=int)
    g.add_argument("--read_range", default=1000, type=int)
    g = p.add_argument_group("Force calling")
    g.add_argument("-Ivcf", default=None, type=str)
    g = p.add_argument_group("Advanced")
    g.add_argument("--max_cluster_bias_INS", default=100, type=int)
    g.add_argument("--diff_ratio_merging_INS", default=0.3, type=float)
    g.add_argument("--max_cluster_bias_DEL", default=200, type=int)
    g.add_argument("--diff_ratio_merging_DEL", default=0.5, type=float)
    g.add_argument("--max_cluster_bias_INV", default=500, type=int)
    g.add_argument("--max_cluster_bias_DUP", default=500, type=int)
    g.add_argument("--max_cluster_bias_TRA", default=50, type=int)
    g.add_argument("--diff_ratio_filtering_TRA", default=0.6, type=float)
    g.add_argument("--remain_reads_ratio", default=1.0, type=float)
    return p


def params_from_args(a):
    return _abi.default_params(
        min_support=a.min_support, min_size=a.min_size, max_size=a.max_size, bias_del=a.max_cluster_bias_DEL,
        bias_ins=a.max_cluster_bias_INS, bias_inv=a.max_cluster_bias_INV, bias_dup=a.max_cluster_bias_DUP,
        bias_tra=a.max_cluster_bias_TRA, genotype=1 if a.genotype else 0, gt_round=a.gt_round, ratio_del=a.diff_ratio_merging_DEL,
        ratio_ins=a.diff_ratio_merging_INS, ratio_tra=a.diff_ratio_filtering_TRA, remain_reads_ratio=a.remain_reads_ratio,
        min_mapq=a.min_mapq, max_split_parts=a.max_split_parts, min_read_len=a.min_read_len, min_siglength=a.min_siglength,
        merge_del_threshold=a.merge_del_threshold, merge_ins_threshold=a.merge_ins_threshold)


def task_windows(ref_stats, get_len, threads, batches):
    """Genome windows exactly like cuteSV:1018-1044 (coverage-balanced, float bounds included)."""
    total_mapped = sum(i[1] for i in ref_stats)
    mapped_unit = total_mapped / threads / 10
    tasks, contig_info = [], []
    for i in ref_stats:
        n = get_len(i[0])
        contig_info.append([i[0], n])
        batch = batches if (total_mapped == 0 or i[1] <= mapped_unit) else n / (int(i[1] / mapped_unit) + 1)
        if n < batch:
            tasks.append([i[0], 0, n])
        else:
            pos = 0
            for _ in range(int(n / batch)):
                tasks.append([i[0], pos, pos + batch])
                pos += batch
            if pos < n:
                tasks.append([i[0], pos, n])
    return tasks, contig_info


def load_bed(bed_file, tasks):
    """-include_bed: regions padded by 1000 bp, assigned to windows (cuteSV_genotype.py:704-726)."""
    if bed_file is None:
        return None
    regions = {}
    with open(bed_file) as f:
        for line in f:
            s = line.strip().split("\t")
            regions.setdefault(s[0], []).append((int(s[1]) - 1000, int(s[2]) + 1000))
    out = [[] for _ in tasks]
    # the reference scans every task for every region; only the tasks of the region's own contig can match, so visiting
    # just those (in task order) gives the same lists in the same order without O(regions x tasks) on many-contig genomes
    by_contig = {}
    for i, t in enumerate(tasks):
        by_contig.setdefault(t[0], []).append(i)
    for chrom in regions:
        regions[chrom].sort()
        own = [(i, tasks[i]) for i in by_contig.get(chrom, ())]
        for item in regions[chrom]:
            for i, t in own:
                if (t[1] <= item[0] and t[2] > item[0]) or item[0] <= t[1] < item[1]:
                    out[i].append(item)
    return out


class _Accumulator(object):
    """Host side of the scan: the extracted signatures and reads rows stay ON THE DEVICE (csv_extract_append); the host keeps
    only what the device cannot hold -- INS sequence strings (rebuilt per packet from the piece descriptors), provisional
    read ids, and the all-alignments table of the TRA genotyper."""

    def __init__(self, eng, min_siglength, merge_ins_threshold):
        self.eng = eng
        self.ins_seq = packing.InsStore()   # INS sequence of every INS signature, by input index
        self.rec_base = 0
        self.name_id = {}
        self.names = []
        self.aln = {k: [] for k in ("chrom", "start", "end", "read_id", "is_primary")}  # every record, BAM order
        self.aln_chunks = []
        self.merge = (min_siglength, merge_ins_threshold)
        self.t_extract = 0.0    # seconds inside csv_extract_append (H2D of the packet + kernel (a) + counts)
        self.t_ins_seq = 0.0    # seconds rebuilding INS sequence strings on the host
        eng.extract_reset()

    def rid(self, name):
        i = self.name_id.get(name)
        if i is None:
            i = len(self.names)
            self.name_id[name] = i
            self.names.append(name)
        return i

    def extract(self, packet, n_records, query_of, want_seq, cigar_of=None):
        """One packet through csv_extract_append.  query_of(rec) -> query sequence of packet record `rec`;
        cigar_of(rec) -> (uint32 CIGAR array, reference_start) for the rare signatures the host rebuilds.
        A packet of the native decoder carries BAM's packed bases: the INS sequences are then cut out of them for the
        whole packet at once (packing.ins_block_from_packed), per-signature Python only for the exceptions."""
        t0 = time.perf_counter()
        r = self.eng.extract(packet, append=True)
        t1 = time.perf_counter()
        self.t_extract += t1 - t0
        n_new = r["counts"]["INS"] - r["first"]["INS"]
        if want_seq and n_new:
            po, pc, pieces = self.eng.fetch_ins_pieces(r["first"]["INS"], n_new, r["first_pieces"], r["n_pieces"] - r["first_pieces"])
            base = self.rec_base

            def slow(i):
                return packing.ins_sequence(pieces, int(po[i]), int(pc[i]), lambda rec: query_of(rec - base),
                                            (lambda rec: cigar_of(rec - base)) if cigar_of else None, self.merge)
            if "seq4" in packet:
                local = np.array(pieces, dtype=np.int32, copy=True)
                local[:, 0] -= base
                lo, hi = (packet["seq_lo"], packet["seq_hi"]) if "seq_lo" in packet else (packet["seq_off"][:-1], packet["seq_off"][1:])
                bases, off, rest = packing.ins_block_from_packed(local, po, pc, packet["seq4"], lo, hi, packet["query_len"])
                first = len(self.ins_seq)
                self.ins_seq.add_block(bases, off)
                for i in rest.tolist():
                    self.ins_seq[first + i] = slow(i)
            else:
                self.ins_seq.add_strings([slow(i) for i in range(n_new)])
        else:
            self.ins_seq.add_empty(n_new)
        self.rec_base += n_records
        self.t_ins_seq += time.perf_counter() - t1

    def add_alignment(self, chrom_id, read):
        a = self.aln
        a["chrom"].append(chrom_id); a["start"].append(read.reference_start); a["end"].append(read.reference_end)
        a["read_id"].append(self.rid(read.query_name)); a["is_primary"].append(1 if read.flag in (0, 16) else 0)

    def add_alignment_chunk(self, chrom, start, end, read_id, is_primary):
        """Columns of many records at once (native decoder path); ids are provisional like rid()."""
        self.aln_chunks.append(dict(chrom=chrom, start=start, end=end, read_id=read_id, is_primary=is_primary))

    def alignments(self, rank):
        """All-alignments table sorted by contig id (stable: BAM order inside a contig), ids as ranks."""
        a = {k: np.asarray(v, dtype=np.uint8 if k == "is_primary" else np.int32) for k, v in self.aln.items()}
        if self.aln_chunks:
            a = {k: np.concatenate([a[k]] + [np.asarray(c[k], dtype=a[k].dtype) for c in self.aln_chunks]) for k in a}
        if len(a["chrom"]) == 0:
            return None
        a["read_id"] = rank[a["read_id"]]
        order = np.argsort(a["chrom"], kind="stable")
        return {k: v[order] for k, v in a.items()}

    def finish(self, names=None, rank=None, want_seq=True):
        """Turn the provisional read ids on the device into ranks in Python string order (csv_remap_read_ids) and put INS rows
        that tie on (contig, int(pos), len, read) into the order of their sequences (cuteSV:774).  The native decoder keeps
        the name table itself and passes (names, rank).  Returns the read names in rank order."""
        if names is None:
            names = self.names
            order = sorted(range(len(names)), key=lambda i: names[i])
            rank = np.zeros(max(len(order), 1), dtype=np.int32)
            rank[np.array(order, dtype=np.int64)] = np.arange(len(order), dtype=np.int32)
        else:
            order = np.argsort(rank[:len(names)], kind="stable")
        sorted_names = [names[i] for i in order]
        self.rank = rank
        self.eng.remap_read_ids(rank[:max(len(names), 1)])
        if want_seq and len(self.ins_seq) > 1:
            c = self.eng.fetch_sig_cols("INS", cols=("chrom", "a", "b", "read_id"))
            pairs = ins_tie_swaps(c["chrom"], c["a"], c["b"], c["read_id"], self.ins_seq)
            if len(pairs):
                self.eng.swap_ins_rows(pairs)
                for i, j in pairs:
                    self.ins_seq[i], self.ins_seq[j] = self.ins_seq[j], self.ins_seq[i]
        return sorted_names


def _tie_runs(chrom, a, b, read_id):
    """INS rows sorted by (contig, int(pos), len, read, row) and the mask `same[k]`: sorted rows k and k + 1 tie on the first four.
    None when there are fewer than two rows."""
    n = len(chrom)
    if n < 2:
        return None
    pos = np.asarray(a, dtype=np.int64) >> 1
    order = np.lexsort((np.arange(n), read_id, b, pos, chrom))
    k = np.stack([np.asarray(chrom)[order], pos[order], np.asarray(b)[order], np.asarray(read_id)[order]])
    return order, np.all(k[:, 1:] == k[:, :-1], axis=0)


def ins_tie_rows(chrom, a, b, read_id):
    """Ascending INS rows that belong to a tie group of ins_tie_swaps (rows tying on (contig, int(pos), len, read)): the only rows
    whose sequence strings ins_tie_swaps reads, so a caller whose strings live on the device fetches just these."""
    runs = _tie_runs(chrom, a, b, read_id)
    if runs is None:
        return np.zeros(0, dtype=np.int64)
    order, same = runs
    member = np.zeros(len(order), dtype=bool)
    member[1:] |= same
    member[:-1] |= same
    return np.sort(order[member]).astype(np.int64)


def ins_tie_swaps(chrom, a, b, read_id, seqs):
    """Row swaps that put INS rows tying on (contig, int(pos), len, read) into the order of their sequence strings, the last
    field of the reference's INS sort key (cuteSV:774).  Vectorised search for tie groups (they need one read reporting two
    insertions of equal length at the same position: rare), selection sort inside a group.  Returns a list of (i, j)."""
    runs = _tie_runs(chrom, a, b, read_id)
    if runs is None:
        return []
    order, same = runs
    n = len(order)
    if not same.any():
        return []
    pairs = []
    starts = np.flatnonzero(same & ~np.concatenate([[False], same[:-1]]))
    for s0 in starts:
        e = s0 + 1
        while e < n - 1 and same[e]:
            e += 1
        rows = sorted(int(x) for x in order[s0:e + 1])          # input positions of the tie group, ascending
        want = sorted(rows, key=lambda r: (seqs[r], r))         # which row's content belongs at each position
        cur = list(rows)                                         # cur[p] = original row whose content sits at position rows[p]
        for p in range(len(rows)):
            if cur[p] != want[p]:
                q = cur.index(want[p])
                pairs.append((rows[p], rows[q]))
                cur[p], cur[q] = cur[q], cur[p]
    return pairs


def main_ctrl(args, argv, engine=None):
    tmp = args.work_dir if args.work_dir[-1] == "/" else args.work_dir + "/"
    if args.Ivcf is not None:
        raise ValueError("The force calling module has been disabled, please install cuteFC "
                         "(https://github.com/Meltpinkg/cuteFC) to achieve SV force calling/regenotyping.")
    if not os.path.isfile(args.reference):
        raise FileNotFoundError("[Errno 2] No such file: '%s'" % args.reference)
    if not os.path.exists(args.work_dir):
        raise FileNotFoundError("[Errno 2] No such directory: '%s'" % args.work_dir)
    if os.path.isdir("%sresults" % tmp):
        raise FileExistsError("[Errno 2] Directory exists: '%sresults'" % tmp)
    for t in workdir.TYPES:
        for ext in (".sigs", ".pickle"):
            if os.path.exists(tmp + t + ext):
                raise FileExistsError("[Errno 2] File exists: '%s'" % (tmp + t + ext))
    from .engine import Engine
    source = _open_source(args)
    stats = source.index_statistics()
    logging.info("The total number of chromsomes: %d" % len(stats))
    tasks, contig_info = task_windows(stats, source.get_reference_length, args.threads, args.batches)
    bed = load_bed(args.include_bed, tasks)
    chrom_names = sorted(c[0] for c in contig_info)
    chrom_id = {n: i for i, n in enumerate(chrom_names)}
    lens = {c[0]: c[1] for c in contig_info}
    params = params_from_args(args)
    eng = engine if engine is not None else Engine(int(os.environ.get("CUTESV_B200_DEVICE", "0")))
    eng.set_params(params)
    eng.set_contigs(np.array([lens[n] for n in chrom_names], dtype=np.int64))
    acc = _Accumulator(eng, args.min_siglength, args.merge_ins_threshold)
    want_seq = not args.ignore_sequence
    stages = {}
    t_stage = time.perf_counter()

    def lap(name):
        nonlocal t_stage
        now = time.perf_counter()
        stages[name] = stages.get(name, 0.0) + now - t_stage
        t_stage = now

    names_rank = source.scan(args, eng, acc, tasks, bed, chrom_id, want_seq)
    lap("scan")   # decode + pack + csv_extract_append per packet
    logging.info("Rebuilding signatures of structural variants.")
    read_names = acc.finish(*names_rank, want_seq=want_seq)   # the signatures never left the device
    lap("names_and_ties")
    logging.info("Clustering structural variants.")
    eng.upload_alignments(acc.alignments(acc.rank) if args.genotype else None)
    eng.cluster_device(0x1F)
    cands, genos, names = eng.fetch()
    eng.upload_alignments(None)
    lap("cluster_and_fetch")
    got = rows.records_to_rows(cands, genos, names, chrom_names, lambda k: read_names[k], lambda k: acc.ins_seq[k], bool(args.genotype))
    lap("rows")
    results = {}
    for t in ("DEL", "INS", "INV", "DUP", "TRA"):  # submission order of the reference, cuteSV:1116-1199
        for (tt, chrom), r in got.items():
            if tt == t:
                results.setdefault(chrom, []).extend(r)
    logging.info("Writing to your output file.")
    reference = vcf.IndexedFasta(args.reference)   # random access through <ref>.fai (built on the fly when missing)
    for name, n in contig_info:   # a stale .fai / another assembly would give wrong REF bases without any error
        have = reference.length_of(name)
        if have is not None and have != n:
            logging.warning("contig %s: %d bp in the BAM header but %d bp in %s (stale .fai or another assembly?)" % (name, n, have, args.reference))
    opts = dict(genotype=args.genotype, max_size=args.max_size, min_size=args.min_size, report_readid=args.report_readid,
                ignore_sequence=args.ignore_sequence)
    vcf.write_vcf(args.output, results, reference, contig_info, args.sample, argv, opts)
    lap("vcf")
    # stage split of the wall time (scan = BAM decode + packing + the device extraction, of which csv_extract_append and the
    # host rebuild of INS sequence strings are also given on their own)
    stages["scan.csv_extract_append"] = acc.t_extract
    stages["scan.ins_sequences"] = acc.t_ins_seq
    main_ctrl.last_stages = dict(stages)
    logging.info("Stage split (s): " + ", ".join("%s %.3f" % kv for kv in stages.items()))
    if args.retain_work_dir:   # the reference's pickle layout needs the signatures on the host: one D2H of the columns
        sigs = {t: eng.fetch_sig_cols(t) for t in _abi.TYPE_NAMES}
        _write_workdir(tmp, sigs, eng.fetch_read_rows(), chrom_names, read_names, acc.ins_seq, args.write_old_sigs)
    reference.close()
    source.close()
    return results


def _open_source(args):
    """BAM decoding backend: the native decoder (csrc/bam_reader.cpp) for BGZF BAM input, pysam for
    everything else (CRAM, SAM).  CUTESV_B200_BAM=native|pysam forces one."""
    from . import bamio
    want = os.environ.get("CUTESV_B200_BAM", "auto")
    if want == "native" or (want == "auto" and bamio.is_bam(args.input)):
        return _NativeSource(args)
    try:
        import pysam
    except ImportError:
        raise RuntimeError("pysam is required to decode this input (only BGZF-compressed BAM is decoded natively)")
    return _PysamSource(pysam.AlignmentFile(args.input, reference_filename=args.reference))


class _PysamSource(object):
    """Window-by-window pysam iteration, the reference's own access pattern (cuteSV:697-733)."""

    def __init__(self, sam):
        self.sam = sam

    def index_statistics(self):
        return self.sam.get_index_statistics()

    def get_reference_length(self, name):
        return self.sam.get_reference_length(name)

    def close(self):
        self.sam.close()

    def scan(self, args, eng, acc, tasks, bed, chrom_id, want_seq):
        def flush(packet):
            if not packet:
                return
            pk = packing.pack_alignments(packet, chrom_id, _NameIds(acc))
            acc.extract(pk, len(packet), lambda rec: packet[rec].query_sequence, want_seq,
                        lambda rec: (pk["cigar"][pk["cigar_off"][rec]:pk["cigar_off"][rec + 1]], int(pk["ref_start"][rec])))

        for i, task in enumerate(tasks):
            packet = []
            regions = None if bed is None else bed[i]
            for read in self.sam.fetch(task[0], task[1], task[2]):
                if args.genotype and read.reference_start >= task[1] and read.reference_end is not None:
                    acc.add_alignment(chrom_id[task[0]], read)  # EVERY record (no filter): input of the TRA genotyper
                if read.flag == 256 or read.flag == 272:  # cuteSV:711
                    continue
                if regions is not None and not any(not (read.reference_end <= r[0] or read.reference_start >= r[1]) for r in regions):
                    continue
                if not read.reference_start >= task[1]:    # window ownership, cuteSV:725
                    continue
                packet.append(read)
                if len(packet) >= PACKET_READS:
                    flush(packet)
                    packet = []
            flush(packet)
            logging.info("Finished %s:%d-%d." % (task[0], task[1], task[2]))
        return None, None


class _NativeSource(object):
    """One sequential pass over the BAM with the native decoder: every mapped record is seen once, in
    file order -- the same sequence the window loop above yields for a coordinate-sorted BAM, since a
    record is owned by the window its start falls in (cuteSV:725)."""

    def __init__(self, args):
        from . import bamio
        self.bamio = bamio
        self.rd = bamio.BamReader(args.input, threads=max(1, min(int(args.threads), 32)), keep_seq=not args.ignore_sequence)

    def index_statistics(self):
        return self.rd.index_statistics()

    def get_reference_length(self, name):
        return self.rd.get_reference_length(name)

    def close(self):
        self.rd.close()

    def scan(self, args, eng, acc, tasks, bed, chrom_id, want_seq):
        bamio, rd = self.bamio, self.rd
        rd.set_chrom_ids(chrom_id)
        starts, first_task = window_starts(tasks, chrom_id)
        n_seen = 0
        while True:
            pk = rd.next_packet(PACKET_READS, copy=False)   # views: everything kept beyond this iteration is copied below
            if pk is None:
                break
            has_cigar = pk["cigar_off"][1:] > pk["cigar_off"][:-1]   # reference_end is None otherwise
            if args.genotype:
                v = np.flatnonzero(has_cigar)
                acc.add_alignment_chunk(pk["chrom"][v], pk["ref_start"][v], pk["ref_end"][v], pk["read_id"][v],
                                        ((pk["flag"][v] == 0) | (pk["flag"][v] == 16)).astype(np.uint8))
            keep = has_cigar & (pk["flag"] != 256) & (pk["flag"] != 272) & (pk["chrom"] >= 0)
            if bed is not None:
                bed_filter(pk, keep, bed, starts, first_task)
            sub = bamio.subset_packet(pk, np.flatnonzero(keep))
            if len(sub["chrom"]):
                last = [-1, ""]   # the INS signatures of one record follow each other: decode its query once

                def query_of(rec, sub=sub, last=last):
                    if last[0] != rec:
                        last[0], last[1] = rec, bamio.decode_seq(sub, rec)
                    return last[1]
                acc.extract(sub, len(sub["chrom"]), query_of, want_seq,
                            lambda rec: (sub["cigar"][sub["cigar_off"][rec]:sub["cigar_off"][rec + 1]], int(sub["ref_start"][rec])))
            n_seen += len(keep)
            logging.info("Decoded %d records." % n_seen)
        return rd.names(), rd.name_ranks()


def window_starts(tasks, chrom_id):
    """Window starts per contig id and the index of each contig's first task: what bed_filter needs to find a record's window."""
    starts, first_task = {}, {}
    for i, t in enumerate(tasks):
        starts.setdefault(chrom_id[t[0]], []).append(t[1])
        first_task.setdefault(chrom_id[t[0]], i)
    return starts, first_task


def bed_filter(pk, keep, bed, starts, first_task):
    """-include_bed on one decoded packet: clears keep[i] of every kept record that overlaps no padded region of the window owning
    it, the last window of its contig starting at or before its ref_start (cuteSV:725)."""
    owner = np.zeros(len(keep), dtype=np.int64)
    for c in np.unique(pk["chrom"]):
        m = pk["chrom"] == c
        if int(c) in starts:
            owner[m] = first_task[int(c)] + np.searchsorted(np.asarray(starts[int(c)], dtype=np.float64), pk["ref_start"][m], side="right") - 1
    for ti in np.unique(owner[keep]):
        m = keep & (owner == ti)
        hit = np.zeros(len(keep), dtype=bool)
        for r in bed[int(ti)]:
            hit |= ~((pk["ref_end"] <= r[0]) | (pk["ref_start"] >= r[1]))
        keep[m & ~hit] = False


class _NameIds(object):
    """dict-like: read name -> provisional id (first-seen order); ranks are assigned at the end."""

    def __init__(self, acc):
        self.acc = acc

    def __getitem__(self, name):
        return self.acc.rid(name)


def _write_workdir(tmp, sigs, reads_cols, chrom_names, read_names, ins_seq, write_old_sigs):
    """--retain_work_dir: the reference's <TYPE>.pickle / sigindex.pickle layout (cuteSV:817-857)."""
    tuples = {t: workdir.columns_to_tuples(t, sigs[t], chrom_names, read_names, ins_seq) for t in workdir.TYPES}
    r = reads_cols
    tuples["reads"] = list(zip(r["start"].tolist(), r["end"].tolist(), r["is_primary"].tolist(), [read_names[i] for i in r["read_id"].tolist()],
                               [chrom_names[i] for i in r["chrom"].tolist()]))
    workdir.write_workdir(tmp, tuples)
    if write_old_sigs:  # legacy text dumps, cuteSV:766-816
        for t in workdir.TYPES:
            f = workdir.SIGS_LINE[t]
            with open("%s/%s.sigs" % (tmp, t), "w") as fh:
                for e in sorted(set(tuples[t]), key=workdir.sort_key(t)):
                    fh.write(f(e))


def setup_logging():
    logging.basicConfig(stream=sys.stderr, level=logging.INFO, format="%(asctime)s [%(levelname)s] %(message)s")
    logging.info("Running %s" % " ".join(sys.argv))


def run(argv):
    args = build_parser().parse_args(argv)
    setup_logging()
    t0 = time.time()
    main_ctrl(args, argv)
    logging.info("Finished in %0.2f seconds." % (time.time() - t0))


if __name__ == "__main__":
    run(sys.argv[1:])
