"""Drop-ins for the reference's signature phases (Pool#1 and Pool#2 of main_ctrl, cuteSV:1058-1110):

- single_pipe (cuteSV:697-743): one task window through csv_extract (kernel (a)) instead of parse_read per record, appending
  the same six pickles to <temp_dir>signatures/<pid><TYPE>.pickle.
- process_process_sigs_type (cuteSV:750-857): the pid pickles of one type through csv_sort_sigs (sort + adjacent
  de-duplication on the device), written as <TYPE>.pickle with the reference's per-contig index.
- init_reading_process, cleanup, multi_run_wrapper, remove_duplicates_sorted: the reference's helpers around them.

The pickles interoperate with the reference's in both directions: the reference's process_process_sigs_type can rebuild
what this single_pipe wrote, and this process_process_sigs_type rebuilds what the reference's single_pipe wrote."""
import gc
import logging
import pickle
from multiprocessing import current_process

import numpy as np

from . import _abi, packing, runtime, workdir

SVTYPES = ["DEL", "INS", "DUP", "INV", "TRA"]
samfile = None
# field of the read name in every tuple type (cuteSV:520-531, 235-239, 55-60, 111-117, 733)
_NAME_FIELD = {"DEL": 2, "INS": 2, "DUP": 2, "INV": 3, "TRA": 4, "reads": 3}


def init_reading_process(sam_path, reference_path):
    global samfile
    import pysam
    samfile = pysam.AlignmentFile(sam_path, reference_filename=reference_path)


def cleanup():
    global samfile
    if samfile is not None:
        samfile.close()
        samfile = None


def _in_bed(read, bed_regions):
    if bed_regions is None:
        return True
    return any(not (read.reference_end <= r[0] or read.reference_start >= r[1]) for r in bed_regions)


def extract_window(records, chrom, params, eng=None):
    """parse_read (cuteSV:606-681) over `records` (the records single_pipe keeps, in fetch order) with ONE csv_extract.
    Returns (candidate dict, reads_info_list) with the lists in the reference's order: records in input order, inside a
    record the order in which parse_read appends."""
    eng = eng if eng is not None else runtime.get_engine()
    cand = {t: [] for t in SVTYPES}
    if not records:
        return cand, []
    # contig ids must be ranks in string order (the split-read rules compare contig names); only the names this window
    # touches are needed: its own contig and the contigs of the SA entries
    names = {chrom} | {r.reference_name for r in records}
    for r in records:
        for tag in r.get_tags():
            if tag[0] == "SA":
                names.update(ent.split(",")[0] for ent in tag[1].split(";")[:-1])
    chrom_names = sorted(names)
    chrom_id = {n: i for i, n in enumerate(chrom_names)}
    read_names = sorted({r.query_name for r in records})
    read_id = {n: i for i, n in enumerate(read_names)}
    pk = packing.pack_alignments(records, chrom_id, read_id)
    lens = []
    for n in chrom_names:
        try:
            lens.append(int(samfile.get_reference_length(n)) if samfile is not None else (1 << 31) - 1)
        except (KeyError, ValueError, AttributeError):
            lens.append((1 << 31) - 1)
    eng.set_params(params)
    eng.set_contigs(np.array(lens, dtype=np.int64))
    eng.set_extract_records(True)   # the record of every row: the key that restores the reference's list order
    try:
        eng.extract(pk)
    finally:
        eng.set_extract_records(False)
    ex = eng.fetch_extracted()

    def query_of(rec):
        return records[rec].query_sequence

    def cigar_of(rec):
        return pk["cigar"][pk["cigar_off"][rec]:pk["cigar_off"][rec + 1]], int(pk["ref_start"][rec])

    merge = (params.min_siglength, params.merge_ins_threshold)
    for t in SVTYPES:
        cols = ex["sigs"][t]
        if len(cols["chrom"]) == 0:
            continue
        # row slots come from atomics; one thread emits a record's rows in parse_read's order -> stable sort by record
        order = np.argsort(eng.fetch_records(t), kind="stable")
        cols = {k: v[order] for k, v in cols.items()}
        seqs = None
        if t == "INS":
            po, pc = ex["piece_off"][order], ex["piece_cnt"][order]
            seqs = [packing.ins_sequence(ex["pieces"], int(po[i]), int(pc[i]), query_of, cigar_of, merge) for i in range(len(order))]
        cand[t] = workdir.columns_to_tuples(t, cols, chrom_names, read_names, seqs)
    r = ex["rows"]
    order = np.argsort(eng.fetch_records("reads"), kind="stable")
    reads_info = list(zip(r["start"][order].tolist(), r["end"][order].tolist(), r["is_primary"][order].tolist(),
                          [read_names[i] for i in r["read_id"][order].tolist()], [chrom] * len(order)))
    return cand, reads_info


def single_pipe(sam_path, min_length, min_mapq, max_split_parts, min_read_len, temp_dir, task, min_siglength, merge_del_threshold,
                merge_ins_threshold, MaxSize, bed_regions):
    """cuteSV:697-743: the records of one task window (flag 256 / 272 skipped, -include_bed test, window ownership by start),
    their signatures from ONE csv_extract (not the append mode: a BAM-to-VCF accumulation on the same device is not touched
    beyond what csv_extract replaces), appended as one pickle.dump per type to <temp_dir>signatures/<pid><TYPE>.pickle."""
    Chr_name = task[0]
    records = []
    for read in samfile.fetch(Chr_name, task[1], task[2]):
        if read.flag == 256 or read.flag == 272:
            continue
        if read.reference_start >= task[1] and _in_bed(read, bed_regions):
            records.append(read)
    p = _abi.default_params(min_size=min_length, max_size=MaxSize, min_mapq=min_mapq, max_split_parts=max_split_parts,
                            min_read_len=min_read_len, min_siglength=min_siglength, merge_del_threshold=merge_del_threshold,
                            merge_ins_threshold=merge_ins_threshold)
    candidate, reads_info_list = extract_window(records, Chr_name, p)
    pid = current_process().pid
    for sv_type in SVTYPES:
        with open("%ssignatures/%s%s.pickle" % (temp_dir, pid, sv_type), "ab") as f:
            pickle.dump(candidate[sv_type], f)
    with open("%ssignatures/%sreads.pickle" % (temp_dir, pid), "ab") as f:
        pickle.dump(reads_info_list, f)
    logging.info("Finished %s:%d-%d." % (Chr_name, task[1], task[2]))
    gc.collect()
    return None


def multi_run_wrapper(args):
    return single_pipe(*args)


def remove_duplicates_sorted(sorted_list):
    """Adjacent equal tuples dropped (cuteSV:958-969)."""
    out = sorted_list[:1]
    for x in sorted_list[1:]:
        if x != out[-1]:
            out.append(x)
    return out


def finish_ins_ties(tuples, ins_tie):
    """INS rows in csv_sort_sigs order -> the reference's order and de-duplication: every group of rows that tie up to the
    sequence (ins_tie[k] = 1: row k ties with row k - 1) sorted stably by sequence, then adjacent duplicates dropped inside it.
    Returns (tuples, kept positions)."""
    tie = np.asarray(ins_tie, dtype=bool)
    if not tie.any():
        return tuples, np.arange(len(tuples), dtype=np.int64)
    out = list(tuples)
    keep = np.ones(len(out), dtype=bool)
    n = len(out)
    starts = np.flatnonzero(tie[1:] & ~tie[:-1]).tolist()   # k + 1 ties with k, k does not tie with k - 1
    for s in starts:
        e = s + 1
        while e + 1 < n and tie[e + 1]:
            e += 1
        grp = sorted(out[s:e + 1], key=lambda x: x[3])
        out[s:e + 1] = grp
        for j in range(s + 1, e + 1):   # remove_duplicates_sorted inside the group (rows outside it differ in the key)
            last = j - 1
            while not keep[last]:
                last -= 1
            if out[j] == out[last]:
                keep[j] = False
    pos = np.flatnonzero(keep)
    return [out[i] for i in pos.tolist()], pos


def _load_pid_lists(temporary_dir, pids, sv_type):
    out = []
    for pid in pids:
        with open("%ssignatures/%s%s.pickle" % (temporary_dir, pid, sv_type), "rb") as f:
            while True:
                try:
                    out.extend(pickle.load(f))
                except EOFError:
                    break
    return out


def rebuild_type(sv_type, type_candidates, eng=None):
    """Sort + de-duplication of process_process_sigs_type on the device.  Returns (sorted tuples, contig names in id order,
    per-contig row offsets into the sorted tuples)."""
    eng = eng if eng is not None else runtime.get_engine()
    if not type_candidates:
        return [], [], np.zeros(1, np.int64)
    f = list(zip(*type_candidates))   # ONE transpose: contig names, read names and columns all come from it
    names = set(f[-1])
    if sv_type == "TRA":
        names.update(f[2])
    chrom_names = sorted(names)
    chrom_id = {n: i for i, n in enumerate(chrom_names)}
    name_id = {n: i for i, n in enumerate(sorted(set(f[_NAME_FIELD[sv_type]])))}
    if sv_type == "reads":
        cols = workdir.reads_to_columns(type_candidates, chrom_id, name_id, fields=f)
        hi = int(max(cols["end"].max(), cols["start"].max(), 0))
        eng.set_contigs(np.full(len(chrom_names), min(hi + 2, (1 << 31) - 1), dtype=np.int64))
        eng.upload({}, cols)
    else:
        cols = workdir.tuples_to_columns(sv_type, type_candidates, chrom_id, name_id, fields=f)
        hi = int(max(cols["a"].max(), cols["b"].max(), 0))
        eng.set_contigs(np.full(len(chrom_names), min(hi + 2, (1 << 31) - 1), dtype=np.int64))
        eng.upload({sv_type: cols}, None)
    r = eng.sort_sigs(sv_type)
    order, off = r["order"], r["contig_off"]
    out = [type_candidates[i] for i in order.tolist()]
    if sv_type == "INS":
        out, pos = finish_ins_ties(out, r["ins_tie"])
        if len(pos) != len(order):   # rows dropped inside tie groups: shift the offsets
            off = np.searchsorted(pos, off, side="left").astype(np.int64)
    return out, chrom_names, off


def process_process_sigs_type(args):
    """cuteSV:750-857: concatenate the pid pickles of one type (pid order, then dump order), sort and de-duplicate them on the
    device, write <TYPE>.pickle as one pickle per contig with the byte offsets of the index (and reads_count for "reads"),
    and with write_old_sigs the legacy <TYPE>.sigs text.  Returns (sv_type, index, reads_count)."""
    sv_type, temporary_dir, pids, write_old_sigs = args
    type_candidates = _load_pid_lists(temporary_dir, pids, sv_type)
    out, chrom_names, off = rebuild_type(sv_type, type_candidates)
    if write_old_sigs:
        line = workdir.SIGS_LINE[sv_type]
        with open("%s/%s.sigs" % (temporary_dir, sv_type), "w") as f:
            f.write("".join(line(e) for e in out))
    index, reads_count = {}, {}
    with open("%s/%s.pickle" % (temporary_dir, sv_type), "wb") as f:
        start = 0
        for k, chrom in enumerate(chrom_names):
            lo, hi = int(off[k]), int(off[k + 1])
            if hi == lo:
                continue
            blob = pickle.dumps(out[lo:hi])
            f.write(blob)
            index[chrom] = start
            if sv_type == "reads":
                reads_count[chrom] = hi - lo
            start += len(blob)
    return (sv_type, index, reads_count)
