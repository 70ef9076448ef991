"""The reference's work-dir transport (cuteSV:817-857): <TYPE>.pickle = concatenated pickled
per-contig lists of signature tuples, sigindex = {type: {chr: byte offset}}.  Readers for the
drop-in resolution_* entry points, a writer for --retain_work_dir compatibility and tests, and the
tuple <-> column conversion (names -> ranks in Python string order)."""
import pickle

import numpy as np

from . import _abi

TYPES = ("DEL", "INS", "DUP", "INV", "TRA")
_TRA = {"A": 0, "B": 1, "C": 2, "D": 3}


def sort_key(svtype):
    """Sort keys of process_process_sigs_type (cuteSV:764,774,783,792,801)."""
    if svtype == "DEL":
        return lambda x: (x[-1], int(x[0]), x[1], x[2])
    if svtype == "INS":
        return lambda x: (x[-1], int(x[0]), x[1], x[2], x[3])
    if svtype == "DUP":
        return lambda x: (x[-1], int(x[0]), int(x[1]), x[2])
    if svtype == "INV":
        return lambda x: (x[-1], x[0], int(x[1]), x[2], x[3])
    if svtype == "TRA":
        return lambda x: (x[-1], x[2], x[0], int(x[1]), x[3], x[4], x[5])
    return lambda x: (x[-1])


# one line of the legacy --write_old_sigs text dumps (cuteSV:766-816)
SIGS_LINE = {"DEL": lambda e: "%s\t%s\t%d\t%d\t%s\n" % (e[-2], e[-1], e[0], e[1], e[2]),
             "INS": lambda e: "%s\t%s\t%d\t%d\t%s\t%s\n" % (e[-2], e[-1], e[0], e[1], e[2], e[3]),
             "DUP": lambda e: "%s\t%s\t%d\t%d\t%s\n" % (e[-2], e[-1], e[0], e[1], e[2]),
             "INV": lambda e: "%s\t%s\t%s\t%d\t%d\t%s\n" % (e[-2], e[-1], e[0], e[1], e[2], e[3]),
             "TRA": lambda e: "%s\t%s\t%s\t%d\t%s\t%d\t%s\n" % (e[-2], e[-1], e[0], e[1], e[2], e[3], e[4]),
             "reads": lambda e: "%s\t%d\t%d\t%d\t%s\n" % (e[-1], e[0], e[1], e[2], e[3])}


def write_type(path, svtype, tuples):
    """Write <path><svtype>.pickle in the reference layout; returns (index, reads_count)."""
    cand = sorted(tuples, key=sort_key(svtype))
    if svtype != "reads":  # remove_duplicates_sorted, cuteSV:958-969
        dedup = []
        for t in cand:
            if not dedup or dedup[-1] != t:
                dedup.append(t)
        cand = dedup
    index, counts = {}, {}
    with open("%s%s.pickle" % (path, svtype), "wb") as f:
        start = 0
        i = 0
        while i < len(cand):
            j = i
            while j < len(cand) and cand[j][-1] == cand[i][-1]:
                j += 1
            blob = pickle.dumps(cand[i:j])
            f.write(blob)
            index[cand[i][-1]] = start
            counts[cand[i][-1]] = j - i
            start += len(blob)
            i = j
    return index, counts


def write_workdir(path, tuples_by_type):
    """tuples_by_type: {"DEL": [...], ..., "reads": [...]} -> sigs_index (also pickled as sigindex.pickle)."""
    sigs_index = {}
    for t in TYPES + ("reads",):
        idx, cnt = write_type(path, t, tuples_by_type.get(t, []))
        sigs_index[t] = idx
        if t == "reads":
            sigs_index["reads_count"] = cnt
    with open("%ssigindex.pickle" % path, "wb") as f:
        pickle.dump(sigs_index, f)
    return sigs_index


def load_slice(path, svtype, chrom, sigs_index):
    with open("%s%s.pickle" % (path, svtype), "rb") as f:
        f.seek(sigs_index[svtype][chrom])
        return pickle.load(f)


def name_index(*tuple_lists_and_fields):
    """Rank of every read name in Python string order over several (list, field index) pairs."""
    names = set()
    for lst, k in tuple_lists_and_fields:
        if lst:
            names.update(list(zip(*lst))[k])
    ordered = sorted(names)
    return {n: i for i, n in enumerate(ordered)}, ordered


def _ids(values, index):
    return np.fromiter(map(index.__getitem__, values), dtype=np.int32, count=len(values))


def tuples_to_columns(svtype, tuples, chrom_id, name_id, fields=None):
    """Reference tuples -> int32 columns, column-wise (zip(*tuples) transposes at C speed; no per-tuple Python loop).
    fields: list(zip(*tuples)) when the caller already has it."""
    n = len(tuples)
    cols = dict(chrom=np.zeros(n, np.int32), a=np.zeros(n, np.int32), b=np.zeros(n, np.int32), read_id=np.zeros(n, np.int32),
                c=np.zeros(n, np.int32) if svtype in ("INS", "INV", "TRA") else None)
    if n == 0:
        return cols
    f = fields if fields is not None else list(zip(*tuples))
    cols["chrom"] = _ids(f[-1], chrom_id)
    if svtype == "DEL" or svtype == "DUP":
        cols["a"] = np.asarray(f[0], dtype=np.float64).astype(np.int32)   # int(): truncation
        cols["b"] = np.asarray(f[1], dtype=np.float64).astype(np.int32)
        cols["read_id"] = _ids(f[2], name_id)
    elif svtype == "INS":
        cols["a"] = np.rint(np.asarray(f[0], dtype=np.float64) * 2).astype(np.int32)  # positions from split reads can be x.5 (cuteSV:228,244)
        cols["b"] = np.asarray(f[1], dtype=np.int64).astype(np.int32)
        cols["read_id"] = _ids(f[2], name_id)
        cols["c"] = np.fromiter(map(len, f[3]), dtype=np.int32, count=n)
    elif svtype == "INV":
        cols["c"] = np.fromiter((0 if x == "++" else 1 for x in f[0]), dtype=np.int32, count=n)
        cols["a"] = np.asarray(f[1], dtype=np.float64).astype(np.int32)
        cols["b"] = np.asarray(f[2], dtype=np.float64).astype(np.int32)
        cols["read_id"] = _ids(f[3], name_id)
    elif svtype == "TRA":
        cols["a"] = np.asarray(f[1], dtype=np.float64).astype(np.int32)
        cols["b"] = np.asarray(f[3], dtype=np.float64).astype(np.int32)
        cols["read_id"] = _ids(f[4], name_id)
        cols["c"] = _ids(f[2], chrom_id) * 4 + np.fromiter(map(_TRA.__getitem__, f[0]), dtype=np.int32, count=n)
    return cols


def reads_to_columns(rows, chrom_id, name_id, fields=None):
    n = len(rows)
    if n == 0:
        return dict(chrom=np.zeros(0, np.int32), start=np.zeros(0, np.int32), end=np.zeros(0, np.int32), read_id=np.zeros(0, np.int32),
                    is_primary=np.zeros(0, np.uint8))
    f = fields if fields is not None else list(zip(*rows))
    return dict(chrom=_ids(f[4], chrom_id), start=np.asarray(f[0], dtype=np.int64).astype(np.int32),
                end=np.asarray(f[1], dtype=np.int64).astype(np.int32), read_id=_ids(f[3], name_id),
                is_primary=np.asarray(f[2], dtype=np.int64).astype(np.uint8))


def columns_to_tuples(svtype, cols, chrom_names, read_names, ins_seq=None):
    """int32 columns -> the reference's tuple lists (--retain_work_dir), column-wise."""
    n = len(cols["chrom"])
    if n == 0:
        return []
    ch = [chrom_names[i] for i in cols["chrom"].tolist()]
    nm = [read_names[i] for i in cols["read_id"].tolist()]
    a, b = cols["a"].tolist(), cols["b"].tolist()
    if svtype == "DEL" or svtype == "DUP":
        return list(zip(a, b, nm, [svtype] * n, ch))
    if svtype == "INS":
        pos = [(x // 2 if x % 2 == 0 else x / 2) for x in a]
        return list(zip(pos, b, nm, ins_seq, ["INS"] * n, ch))
    c = cols["c"].tolist()
    if svtype == "INV":
        return list(zip([("++" if x == 0 else "--") for x in c], a, b, nm, ["INV"] * n, ch))
    if svtype == "TRA":
        return list(zip(["ABCD"[x & 3] for x in c], a, [chrom_names[x >> 2] for x in c], b, nm, ["TRA"] * n, ch))
    raise ValueError(svtype)
