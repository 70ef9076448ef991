"""Drop-in for the reference's cuteSV_resolveTRA (resolveTRA.py:30-104,257-309).

Clustering and genotyping run on the GPU.  The reference's call_gt (resolveTRA.py:260-309) re-opens the BAM per
candidate and iterates bam.fetch() with an early exit; here pysam is used ONLY to decode the records around the
breakpoints into a packed all-alignments table (BAM order), which the device genotyper scans (csv_tra_call_gt ->
k_tra_call_gt, one warp per breakpoint pair).  No host genotype computation.

- resolution_TRA: csv_cluster, then, with action, csv_tra_call_gt on the candidates' own positions and supports.
- call_gt: the reference's signature and return tuple; call_gt_batch: many breakpoint pairs, one BAM pass and one device
  call.  Both raise ValueError for a clamped window with start > end, as pysam's fetch does; they check the second window
  up front, where the reference only reaches it when the first scan ran to its end."""
import numpy as np

from . import _abi, cuteSV_genotype, rows, runtime, workdir


def _fetch_alignments(bam_path, windows, chrom_id, name_id_of):
    """Decode every record overlapping the (merged) windows, per contig in BAM order."""
    import pysam
    bam = pysam.AlignmentFile(bam_path)
    cols = {k: [] for k in ("chrom", "start", "end", "read_id", "is_primary")}
    try:
        for chrom in sorted(windows, key=lambda c: chrom_id[c]):
            iv = sorted(windows[chrom])
            merged = []
            for s, e in iv:
                if merged and s <= merged[-1][1]:
                    merged[-1][1] = max(merged[-1][1], e)
                else:
                    merged.append([s, e])
            seen = set()
            recs = []
            for s, e in merged:
                for r in bam.fetch(chrom, s, e):
                    key = (r.reference_start, r.reference_end, r.query_name, r.flag)
                    if key in seen:  # a record spanning two disjoint windows is returned by both fetches
                        continue
                    seen.add(key)
                    recs.append(r)
            recs.sort(key=lambda r: r.reference_start)  # stable: BAM order inside one start
            for r in recs:
                cols["chrom"].append(chrom_id[chrom]); cols["start"].append(r.reference_start); cols["end"].append(r.reference_end)
                cols["read_id"].append(name_id_of(r.query_name)); cols["is_primary"].append(1 if r.flag in (0, 16) else 0)
        lens = {c: bam.get_reference_length(c) for c in windows}
    finally:
        bam.close()
    return {k: np.asarray(v, dtype=np.uint8 if k == "is_primary" else np.int32) for k, v in cols.items()}, lens


def resolution_TRA(path, chr_1, read_count, overlap_size, max_cluster_bias, bam_path, action, gt_round, sigs_index):
    if chr_1 not in sigs_index["TRA"]:
        return (chr_1, [])
    seqs = workdir.load_slice(path, "TRA", chr_1, sigs_index)
    name_id, names = workdir.name_index((seqs, 4))
    chroms = sorted(set([chr_1] + [t[2] for t in seqs]))
    chrom_id = {c: i for i, c in enumerate(chroms)}
    cols = workdir.tuples_to_columns("TRA", seqs, chrom_id, name_id)
    hi = max([1] + [int(cols[k].max()) for k in ("a", "b") if len(cols[k])])
    eng = runtime.get_engine()
    p = _abi.default_params(min_support=read_count, ratio_tra=overlap_size, bias_tra=max_cluster_bias, genotype=0, gt_round=gt_round)
    eng.set_params(p)
    eng.set_contigs(np.full(len(chroms), hi + max_cluster_bias + 2, dtype=np.int64))
    res = eng.cluster({"TRA": cols}, None, type_mask=1 << _abi.CSV_TRA)
    if action and len(res[0]):
        # windows of call_gt: [pos - bias, pos + bias] on both contigs (resolveTRA.py:264-265, 292-293)
        cands, _, names_buf = res
        windows = {}
        for c in cands:
            windows.setdefault(chroms[int(c["chrom"])], []).append((max(int(c["pos"]) - max_cluster_bias, 0), int(c["pos"]) + max_cluster_bias))
            windows.setdefault(chroms[int(c["aux"]) >> 2], []).append((max(int(c["pos2"]) - max_cluster_bias, 0), int(c["pos2"]) + max_cluster_bias))
        extra = {}

        def nid(name):  # names outside the signature set only need distinct ids
            i = name_id.get(name)
            if i is None:
                i = extra.get(name)
                if i is None:
                    i = len(names) + len(extra)
                    extra[name] = i
            return i
        aln, lens = _fetch_alignments(bam_path, windows, chrom_id, nid)
        eng.set_contigs(np.array([lens.get(c, hi + max_cluster_bias + 2) for c in chroms], dtype=np.int64))
        q = np.zeros(len(cands), _abi.TRA_QUERY_DTYPE)
        q["chr1"], q["pos1"], q["chr2"], q["pos2"] = cands["chrom"], cands["pos"], cands["aux"] >> 2, cands["pos2"]
        off = np.zeros(len(cands) + 1, np.int64)
        np.cumsum(cands["names_cnt"], out=off[1:])
        ids = np.concatenate([names_buf[o:o + k] for o, k in zip(cands["names_off"], cands["names_cnt"])])
        res = (cands, eng.tra_call_gt(q, off, ids, max_cluster_bias, gt_round, aln=aln), names_buf)
    out = rows.records_to_rows(res[0], res[1], res[2], chroms, lambda i: names[i], None, bool(action))
    return (chr_1, out.get(("TRA", chr_1), []))


def run_tra(args):
    return resolution_TRA(*args)


def _call_gt_genos(bam_path, queries, max_cluster_bias, gt_round):
    """queries: [(pos_1, pos_2, chr_1, chr_2, read_id_list), ...] -> one csv_geno per query (csv_tra_call_gt on the records
    fetched around all windows)."""
    import pysam
    chroms = sorted({q[2] for q in queries} | {q[3] for q in queries})
    bam = pysam.AlignmentFile(bam_path)
    try:
        lens = {c: bam.get_reference_length(c) for c in chroms}
    finally:
        bam.close()
    chrom_id = {c: i for i, c in enumerate(chroms)}
    windows = {}
    for pos_1, pos_2, chr_1, chr_2, _ in queries:
        for chrom, pos in ((chr_1, int(pos_1)), (chr_2, int(pos_2))):
            s, e = max(pos - max_cluster_bias, 0), min(pos + max_cluster_bias, lens[chrom])
            if s > e:   # pysam's fetch (resolveTRA.py:269, 294)
                raise ValueError("invalid coordinates: start (%d) > stop (%d)" % (s, e))
            windows.setdefault(chrom, []).append((s, e))
    name_id = {}

    def nid(name):   # supporting names absent from the BAM get ids of their own
        return name_id.setdefault(name, len(name_id))
    aln, _ = _fetch_alignments(bam_path, windows, chrom_id, nid)
    q = np.zeros(len(queries), _abi.TRA_QUERY_DTYPE)
    q["pos1"], q["pos2"] = [int(x[0]) for x in queries], [int(x[1]) for x in queries]
    q["chr1"], q["chr2"] = [chrom_id[x[2]] for x in queries], [chrom_id[x[3]] for x in queries]
    off = np.zeros(len(queries) + 1, np.int64)
    np.cumsum([len(x[4]) for x in queries], out=off[1:])
    ids = np.fromiter((nid(n) for x in queries for n in x[4]), dtype=np.int32, count=int(off[-1]))
    eng = runtime.get_engine()
    eng.set_contigs(np.array([lens[c] for c in chroms], dtype=np.int64))
    return eng.tra_call_gt(q, off, ids, max_cluster_bias, gt_round, aln=aln)


def _call_gt_tuple(g, dv):
    if int(g["status"]) == 2:   # count_coverage returned -1 (resolveTRA.py:277-282)
        return dv, ".", "./.", ".,.,.", ".", "."
    dr = int(g["dr"])
    return (dv, dr) + cuteSV_genotype._gl_tuple(g, dr, dv)


def call_gt(bam_path, pos_1, pos_2, chr_1, chr_2, read_id_list, max_cluster_bias, gt_round):
    """(DV, DR, GT, GL, GQ, QUAL) like resolveTRA.py:260-309: '.' strings where the first window is too noisy, otherwise
    ints and strings with QUAL typed as cal_GL types it."""
    g = _call_gt_genos(bam_path, [(pos_1, pos_2, chr_1, chr_2, read_id_list)], max_cluster_bias, gt_round)[0]
    return _call_gt_tuple(g, len(read_id_list))


def call_gt_batch(bam_path, queries, max_cluster_bias, gt_round):
    """[call_gt(bam_path, pos_1, pos_2, chr_1, chr_2, read_id_list, max_cluster_bias, gt_round) for each query] with
    queries = [(pos_1, pos_2, chr_1, chr_2, read_id_list), ...]: one pass over the BAM and one device call."""
    if not queries:
        return []
    genos = _call_gt_genos(bam_path, queries, max_cluster_bias, gt_round)
    return [_call_gt_tuple(g, len(x[4])) for g, x in zip(genos, queries)]
