"""ctypes / numpy mirrors of include/cutesv_b200.h (struct layouts only, no library loading).

Shared by the product binding (cutesv_b200/_lib.py) and by the test-only oracle binding
(the oracle wrapper under oracle/); the header is the single source of truth for the layouts.
"""
import ctypes as C

import numpy as np

CSV_DEL, CSV_INS, CSV_INV, CSV_DUP, CSV_TRA, CSV_NTYPES = 0, 1, 2, 3, 4, 5
TYPE_NAMES = ("DEL", "INS", "INV", "DUP", "TRA")
TYPE_IDS = {n: i for i, n in enumerate(TYPE_NAMES)}

CSV_OK, CSV_E_INVALID, CSV_E_CUDA, CSV_E_CAPACITY, CSV_E_NODEVICE, CSV_E_INPUT, CSV_E_STATE = (
    0, -1, -2, -3, -4, -5, -6)
CSV_F_NO_READS, CSV_F_GT_HOST = 1, 2
CSV_SORT_READS = 5   # csv_sort_sigs / csv_fetch_records: the reads table instead of one SV type

STAGES = ("h2d", "keys", "sort", "segment", "cluster", "order", "genotype", "d2h", "extract")
CSV_ST_COUNT = len(STAGES)


class csv_params(C.Structure):
    _fields_ = [
        ("min_support", C.c_int32), ("min_support_allele", C.c_int32),
        ("min_size", C.c_int32), ("max_size", C.c_int32),
        ("bias_del", C.c_int32), ("bias_ins", C.c_int32), ("bias_inv", C.c_int32),
        ("bias_dup", C.c_int32), ("bias_tra", C.c_int32),
        ("genotype", C.c_int32), ("gt_round", C.c_int32), ("gt_bias_ins", C.c_int32),
        ("ratio_del", C.c_double), ("ratio_ins", C.c_double), ("ratio_tra", C.c_double),
        ("remain_reads_ratio", C.c_double),
        ("min_mapq", C.c_int32), ("max_split_parts", C.c_int32), ("min_read_len", C.c_int32),
        ("min_siglength", C.c_int32), ("merge_del_threshold", C.c_int32),
        ("merge_ins_threshold", C.c_int32), ("reserved", C.c_int32 * 2),
    ]


_I32P = C.POINTER(C.c_int32)
_I64P = C.POINTER(C.c_int64)
_U8P = C.POINTER(C.c_uint8)
_U32P = C.POINTER(C.c_uint32)


class csv_sig_cols(C.Structure):
    _fields_ = [("n", C.c_int64), ("chrom", _I32P), ("a", _I32P), ("b", _I32P),
                ("read_id", _I32P), ("c", _I32P)]


class csv_reads_cols(C.Structure):
    _fields_ = [("n", C.c_int64), ("chrom", _I32P), ("start", _I32P), ("end", _I32P),
                ("read_id", _I32P), ("is_primary", _U8P)]


class csv_read_cols(C.Structure):
    _fields_ = [("n", C.c_int64), ("chrom", _I32P), ("ref_start", _I32P), ("ref_end", _I32P),
                ("flag", _I32P), ("mapq", _I32P), ("query_len", _I32P), ("read_id", _I32P),
                ("cigar_off", _I64P), ("sa_off", _I64P)]


class csv_sa_cols(C.Structure):
    _fields_ = [("n", C.c_int64), ("chrom", _I32P), ("pos0", _I32P), ("strand", _I32P),
                ("mapq", _I32P), ("first_clip", _I32P), ("last_clip", _I32P), ("ref_span", _I32P)]


class csv_seq_cols(C.Structure):
    _fields_ = [("n_bytes", C.c_int64), ("seq_off", _I64P), ("seq4", _U8P)]


class csv_name_cols(C.Structure):
    _fields_ = [("n_bytes", C.c_int64), ("name_off", _I64P), ("names", _U8P)]


class csv_sa_text(C.Structure):
    _fields_ = [("n_records", C.c_int64), ("n_bytes", C.c_int64), ("text_off", _I64P), ("text", _U8P)]


CAND_DTYPE = np.dtype([
    ("svtype", "<i4"), ("chrom", "<i4"), ("pos", "<i4"), ("len", "<i4"), ("support", "<i4"),
    ("cipos", "<i4"), ("cilen", "<i4"), ("search_pos", "<i4"), ("pos2", "<i4"), ("aux", "<i4"),
    ("names_off", "<i4"), ("names_cnt", "<i4"), ("cluster", "<i4"), ("flags", "<i4"),
    ("reserved", "<i4", (2,)),
])
GENO_DTYPE = np.dtype([
    ("dr", "<i4"), ("dv", "<i4"), ("gt", "<i4"), ("pl", "<i4", (3,)), ("gq", "<i4"),
    ("status", "<i4"), ("qual", "<f8"),
])
WINDOW_DTYPE = np.dtype([("chrom", "<i4"), ("reserved", "<i4"), ("s2", "<i8"), ("e2", "<i8")])   # csv_window, half units
TRA_QUERY_DTYPE = np.dtype([("chr1", "<i4"), ("chr2", "<i4"), ("pos1", "<i8"), ("pos2", "<i8")])   # csv_tra_query
assert CAND_DTYPE.itemsize == 64 and GENO_DTYPE.itemsize == 40 and WINDOW_DTYPE.itemsize == 24 and TRA_QUERY_DTYPE.itemsize == 24


def make_windows(chrom, s2, e2):
    """csv_window array from contig ids and half-unit bounds."""
    w = np.zeros(len(s2), dtype=WINDOW_DTYPE)
    w["chrom"], w["s2"], w["e2"] = chrom, s2, e2
    return w


def i32(a):
    """Contiguous int32 view/copy of `a` (None passes through)."""
    if a is None:
        return None
    return np.ascontiguousarray(a, dtype=np.int32)


def ptr(a, ctype=C.c_int32):
    if a is None:
        return C.cast(None, C.POINTER(ctype))
    return a.ctypes.data_as(C.POINTER(ctype))


def make_sig_cols(cols):
    """cols: dict(chrom, a, b, read_id[, c]) of int32 arrays (or None) -> (struct, keepalive)."""
    if cols is None or len(cols["chrom"]) == 0:
        return csv_sig_cols(0, None, None, None, None, None), ()
    keep = tuple(i32(cols.get(k)) for k in ("chrom", "a", "b", "read_id", "c"))
    n = len(keep[0])
    for k in keep:
        assert k is None or len(k) == n
    return csv_sig_cols(n, *[ptr(k) for k in keep]), keep


def make_sig_cols_grouped(cols):
    """cols: dict(contig_off, a, b, read_id[, c]) (rows grouped by contig) -> (struct, offsets array, keepalive)."""
    if cols is None or len(cols["a"]) == 0:
        return csv_sig_cols(0, None, None, None, None, None), None, ()
    keep = tuple(i32(cols.get(k)) for k in ("a", "b", "read_id", "c"))
    off = np.ascontiguousarray(cols["contig_off"], dtype=np.int64)
    n = len(keep[0])
    for k in keep:
        assert k is None or len(k) == n
    return csv_sig_cols(n, None, *[ptr(k) for k in keep]), off, keep + (off,)


def make_reads_cols_grouped(reads):
    if reads is None or len(reads["start"]) == 0:
        return csv_reads_cols(0, None, None, None, None, None), None, ()
    keep = [i32(reads[k]) for k in ("start", "end", "read_id")]
    prim = np.ascontiguousarray(reads["is_primary"], dtype=np.uint8)
    off = np.ascontiguousarray(reads["contig_off"], dtype=np.int64)
    s = csv_reads_cols(len(keep[0]), None, *[ptr(k) for k in keep], ptr(prim, C.c_uint8))
    return s, off, tuple(keep) + (prim, off)


def group_by_contig(cols, n_contigs):
    """Stable regrouping of a column dict by its `chrom` column: returns the dict without `chrom`, with
    `contig_off` (n_contigs + 1 row offsets).  The order inside a contig is kept, so every tie-break on
    the input order gives the same result as for the ungrouped columns."""
    chrom = np.asarray(cols["chrom"])
    order = np.argsort(chrom, kind="stable")
    out = {k: (None if v is None else np.ascontiguousarray(np.asarray(v)[order])) for k, v in cols.items() if k != "chrom"}
    off = np.zeros(n_contigs + 1, dtype=np.int64)
    np.cumsum(np.bincount(chrom, minlength=n_contigs)[:n_contigs], out=off[1:])
    out["contig_off"] = off
    return out


def make_reads_cols(reads):
    """reads: dict(chrom, start, end, read_id, is_primary) -> (struct, keepalive)."""
    if reads is None or len(reads["chrom"]) == 0:
        return csv_reads_cols(0, None, None, None, None, None), ()
    keep = [i32(reads[k]) for k in ("chrom", "start", "end", "read_id")]
    prim = np.ascontiguousarray(reads["is_primary"], dtype=np.uint8)
    n = len(keep[0])
    s = csv_reads_cols(n, *[ptr(k) for k in keep], ptr(prim, C.c_uint8))
    return s, tuple(keep) + (prim,)


SIG_FIELDS = ("chrom", "a", "b", "read_id", "c")
READS_FIELDS = ("chrom", "start", "end", "read_id", "is_primary")
_TYPESTR = {"is_primary": "|u1", "contig_off": "<i8"}   # every other column is int32 ("<i4")
_ITEMSIZE = {"<i4": 4, "|u1": 1, "<i8": 8, "<u4": 4, "<u1": 1}


def is_device_array(x):
    """True for objects that expose __cuda_array_interface__ (torch CUDA tensors, CuPy / Numba device arrays)."""
    try:
        return hasattr(x, "__cuda_array_interface__")
    except Exception:   # e.g. torch raises for a CPU tensor
        return False


def _device_index(x):
    """Device ordinal an array reports (torch: .device.index, CuPy: .device.id), or None."""
    d = getattr(x, "device", None)
    for attr in ("index", "id"):
        v = getattr(d, attr, None)
        if isinstance(v, int):
            return v
    return None


def device_cols(cols, fields, device, grouped=False, n_contigs=None):
    """Normalises the columns of ONE upload (a signature dict of SIG_FIELDS or a reads dict of READS_FIELDS) whose columns live in
    GPU memory.  Needs no GPU: it reads __cuda_array_interface__ and the arrays' device attribute only.

    Returns None when the dict is None / empty or holds host columns only (the numpy path).  Otherwise (struct, contig_off address
    or None): the csv_sig_cols / csv_reads_cols of device addresses for csv_upload_*_device.  grouped=True: the dict holds
    `contig_off` (int64, n_contigs + 1) instead of `chrom`.
    Raises TypeError for a column of the wrong dtype (int32; uint8 is_primary; int64 contig_off), not 1-D or not contiguous,
    ValueError when host and device columns are mixed, when a column is on another device than `device`, or when lengths disagree.
    Whether the addresses really are device memory of `device` is checked again by the library."""
    if cols is None:
        return None
    names = [f for f in fields if not (grouped and f == "chrom")] + (["contig_off"] if grouped else [])
    present = {f: cols.get(f) for f in names if cols.get(f) is not None}
    on_dev = {f: is_device_array(v) for f, v in present.items()}
    if not any(on_dev.values()):
        return None
    if not all(on_dev.values()):
        raise ValueError("columns of one upload must be all device or all host arrays: host %s, device %s"
                         % (sorted(f for f, d in on_dev.items() if not d), sorted(f for f, d in on_dev.items() if d)))
    ptrs, lens = {}, {}
    for f, v in present.items():
        ptrs[f], lens[f] = _cai_check(f, v, (_TYPESTR.get(f, "<i4"),), device)
    row_cols = {f: n for f, n in lens.items() if f != "contig_off"}
    if len(set(row_cols.values())) > 1:
        raise ValueError("column lengths disagree: %s" % row_cols)
    n = next(iter(row_cols.values()), 0)
    for f in ("chrom", "a", "b", "read_id") if fields == SIG_FIELDS else ("chrom", "start", "end", "read_id", "is_primary"):
        if f in names and f not in present and n:
            raise ValueError("column %s is missing" % f)
    off = None
    if grouped and n:
        if "contig_off" not in present:
            raise ValueError("grouped columns need contig_off")
        if n_contigs is not None and lens["contig_off"] != n_contigs + 1:
            raise ValueError("contig_off has %d entries, expected n_contigs + 1 = %d" % (lens["contig_off"], n_contigs + 1))
        off = C.cast(C.c_void_p(ptrs["contig_off"]), _I64P)
    if fields == SIG_FIELDS:
        s = csv_sig_cols(n, *[C.cast(C.c_void_p(ptrs.get(f) if n else None), _I32P) for f in SIG_FIELDS])
    else:
        s = csv_reads_cols(n, *[C.cast(C.c_void_p(ptrs.get(f) if n else None), _U8P if f == "is_primary" else _I32P) for f in READS_FIELDS])
    return s, off


READ_FIELDS = ("chrom", "ref_start", "ref_end", "flag", "mapq", "query_len", "read_id")
SA_FIELDS = ("chrom", "pos0", "strand", "mapq", "first_clip", "last_clip", "ref_span")


def _cai_check(name, v, typestrs, device):
    """(address or None, length) of one device array; raises TypeError / ValueError like device_cols."""
    cai = v.__cuda_array_interface__
    if cai["typestr"] not in typestrs:
        raise TypeError("column %s: dtype %s, expected %s" % (name, cai["typestr"], " or ".join(typestrs)))
    shape = tuple(cai["shape"])
    if len(shape) != 1:
        raise TypeError("column %s: shape %s, expected one dimension" % (name, shape))
    strides = cai.get("strides")
    if strides is not None and shape[0] > 1 and tuple(strides) != (_ITEMSIZE[typestrs[0]],):
        raise TypeError("column %s is not contiguous (strides %s)" % (name, tuple(strides)))
    idx = _device_index(v)
    if idx is not None and idx != device:
        raise ValueError("column %s is on device %d, the engine on device %d" % (name, idx, device))
    return (int(cai["data"][0]) if shape[0] else None), shape[0]



class DevicePacket(tuple):
    """device_packet's result: unpacks as (csv_read_cols, cigar address, n_cigar, csv_sa_cols, csv_seq_cols or None); `names` is
    the csv_name_cols of a named packet (csv_extract*_named_device), else None; `sa_text` the csv_sa_text of a packet that carries
    its SA:Z tags as text (csv_reduce_sa_device fills sa_off and the csv_sa_cols), else None."""
    names = None
    sa_text = None


def device_packet(packet, device):
    """Normalises an alignment packet (the keys of packing.pack_alignments, plus optional seq_off / seq4: BAM's 4-bit packed bases,
    and optional names / name_off: the records' read names as bytes) whose arrays live in GPU memory.  Needs no GPU: it reads
    __cuda_array_interface__ and the arrays' device attribute only.

    Returns None when every array is a host array (the numpy path of csv_extract).  Otherwise a DevicePacket: (csv_read_cols,
    cigar address, n_cigar, csv_sa_cols, csv_seq_cols or None) of device addresses for csv_extract*_device, with `.names` the
    csv_name_cols of a named packet (record i's name is names[name_off[i]:name_off[i + 1]]; such a packet has no read_id).
    Raises TypeError for an array of the wrong dtype (int32 record and SA columns, int64 offsets, uint32 or int32 CIGAR, uint8
    bases and names), not 1-D or not contiguous; ValueError when host and device arrays are mixed (names on a host packet
    included), an array is on another device than `device`, lengths disagree (n record columns, n + 1 offsets, equal SA
    columns), only one of seq_off / seq4 or of names / name_off is given, or read_id comes with names.
    Whether the addresses really are device memory of `device` is checked again by the library, the offsets' values on the device.
    A device packet may carry its records' SA:Z values as text instead of sa / sa_off: sa_text (uint8) and sa_text_off (int64, n + 1;
    record i's value is sa_text[sa_text_off[i]:sa_text_off[i + 1]], no tag prefix, no NUL).  The result's `sa_text` then holds
    them, and its csv_read_cols::sa_off and csv_sa_cols are empty until csv_reduce_sa_device fills them; ValueError for a packet
    with both forms, one of sa_text / sa_text_off only, or text on a host packet."""
    sa = packet.get("sa") or {}
    named = packet.get("names") is not None or packet.get("name_off") is not None
    text = packet.get("sa_text") is not None or packet.get("sa_text_off") is not None
    if text and (sa or packet.get("sa_off") is not None):
        raise ValueError("a packet carries sa / sa_off or sa_text / sa_text_off: one or the other")
    arrays = [(f, packet.get(f), ("<i4",)) for f in READ_FIELDS] + [(f, packet.get(f), ("<i8",)) for f in ("cigar_off", "sa_off")]
    arrays += [("cigar", packet.get("cigar"), ("<u4", "<i4"))] + [("sa." + f, sa.get(f), ("<i4",)) for f in SA_FIELDS]
    arrays += [("seq_off", packet.get("seq_off"), ("<i8",)), ("seq4", packet.get("seq4"), ("|u1", "<u1"))]
    arrays += [("name_off", packet.get("name_off"), ("<i8",)), ("names", packet.get("names"), ("|u1", "<u1"))]
    arrays += [("sa_text_off", packet.get("sa_text_off"), ("<i8",)), ("sa_text", packet.get("sa_text"), ("|u1", "<u1"))]
    present = [(f, v, t) for f, v, t in arrays if v is not None]
    on_dev = {f: is_device_array(v) for f, v, _ in present}
    if not any(on_dev.values()):
        if named:
            raise ValueError("names / name_off are accepted on device packets only (a host packet carries read_id)")
        if text:
            raise ValueError("sa_text / sa_text_off are accepted on device packets only (a host packet carries sa / sa_off)")
        return None
    if not all(on_dev.values()):
        raise ValueError("arrays of one packet must be all device or all host arrays: host %s, device %s"
                         % (sorted(f for f, d in on_dev.items() if not d), sorted(f for f, d in on_dev.items() if d)))
    if named and packet.get("read_id") is not None:
        raise ValueError("a named packet carries no read_id: the library numbers its records and ranks their names")
    missing = [f for f, v, _ in arrays[:len(READ_FIELDS) + 3 + len(SA_FIELDS)]
               if v is None and not (named and f == "read_id") and not (text and (f == "sa_off" or f.startswith("sa.")))]
    if missing:
        raise ValueError("packet arrays missing: %s" % missing)
    if (packet.get("seq_off") is None) != (packet.get("seq4") is None):
        raise ValueError("seq_off and seq4 go together: give both or neither")
    if (packet.get("name_off") is None) != (packet.get("names") is None):
        raise ValueError("name_off and names go together: give both or neither")
    if (packet.get("sa_text_off") is None) != (packet.get("sa_text") is None):
        raise ValueError("sa_text_off and sa_text go together: give both or neither")
    ptrs, lens = {}, {}
    for f, v, t in present:
        ptrs[f], lens[f] = _cai_check(f, v, t, device)
    n = lens["chrom"]
    rfields = [f for f in READ_FIELDS if f in lens]
    for f in rfields:
        if lens[f] != n:
            raise ValueError("column lengths disagree: %s" % {g: lens[g] for g in rfields})
    for f in ("cigar_off", "sa_text_off" if text else "sa_off") + tuple(f for f in ("seq_off", "name_off") if f in lens):
        if lens[f] != n + 1:
            raise ValueError("%s has %d entries, expected n + 1 = %d" % (f, lens[f], n + 1))
    n_sa = 0 if text else lens["sa.chrom"]
    if not text and any(lens["sa." + f] != n_sa for f in SA_FIELDS):
        raise ValueError("SA column lengths disagree: %s" % {f: lens["sa." + f] for f in SA_FIELDS})

    def p(f, ctype=_I32P):
        return C.cast(C.c_void_p(ptrs.get(f)), ctype)
    reads = csv_read_cols(n, *[p(f) for f in READ_FIELDS], p("cigar_off", _I64P), p("sa_off", _I64P))
    sa_cols = csv_sa_cols(n_sa, *[p("sa." + f) for f in SA_FIELDS])
    seq = None
    if "seq_off" in lens:
        seq = csv_seq_cols(lens["seq4"], p("seq_off", _I64P), p("seq4", _U8P))
    out = DevicePacket((reads, C.cast(C.c_void_p(ptrs["cigar"]), _U32P), lens["cigar"], sa_cols, seq))
    if named:
        out.names = csv_name_cols(lens["names"], p("name_off", _I64P), p("names", _U8P))
    if text:
        out.sa_text = csv_sa_text(n, lens["sa_text"], p("sa_text_off", _I64P), p("sa_text", _U8P))
    return out


def scan_packet(packet, device):
    """device_packet of a scanned packet (csv_scan_append_named_device): every decoded record of a BAM packet, in GPU memory and
    with names / name_off.  Raises what device_packet raises, and ValueError for a host packet or a packet without names."""
    d = device_packet(packet, device)
    if d is None:
        raise ValueError("a scanned packet lives in GPU memory (torch CUDA tensors); host packets go through extract()")
    if d.names is None:
        raise ValueError("a scanned packet carries names / name_off: the library numbers its records and ranks their names")
    return d


def scan_regions(tasks, bed, chrom_id):
    """Arrays of csv_set_scan_regions from cli.task_windows' tasks ([contig, start, end], start may be a float), cli.load_bed's
    region lists (one list of (lo, hi) per task, or None: no table) and the contig ids: (n_contigs, win_off int64, win_start float64,
    reg_off int64, reg int64 [n_regions, 2]).  n_contigs is 0 without a BED file.  A contig's windows keep their task order."""
    if bed is None:
        return 0, None, None, None, None
    if len(bed) != len(tasks):
        raise ValueError("bed has %d region lists for %d tasks" % (len(bed), len(tasks)))
    n_contigs = max(chrom_id.values()) + 1 if chrom_id else 0
    cid = np.array([chrom_id[t[0]] for t in tasks], dtype=np.int64)
    order = np.argsort(cid, kind="stable")
    win_off = np.zeros(n_contigs + 1, dtype=np.int64)
    np.cumsum(np.bincount(cid, minlength=n_contigs), out=win_off[1:])
    win_start = np.array([tasks[i][1] for i in order.tolist()], dtype=np.float64)
    regs = [bed[i] for i in order.tolist()]
    reg_off = np.zeros(len(tasks) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in regs], out=reg_off[1:])
    reg = np.array([x for r in regs for x in r], dtype=np.int64).reshape(-1, 2)
    return n_contigs, win_off, win_start, reg_off, reg


def default_params(**kw):
    """Reference defaults (cuteSV_Description.py:78-262; wiring cuteSV:1116-1189)."""
    p = csv_params()
    p.min_support = 10
    p.min_size = 30
    p.max_size = 100000
    p.bias_del, p.bias_ins, p.bias_inv, p.bias_dup, p.bias_tra = 200, 100, 500, 500, 50
    p.genotype = 0
    p.gt_round = 500
    p.gt_bias_ins = 1000
    p.ratio_del, p.ratio_ins, p.ratio_tra = 0.5, 0.3, 0.6
    p.remain_reads_ratio = 1.0
    p.min_mapq, p.max_split_parts, p.min_read_len, p.min_siglength = 20, 7, 500, 10
    p.merge_del_threshold, p.merge_ins_threshold = 0, 100
    explicit_allele = "min_support_allele" in kw
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError("unknown parameter %r" % k)
        setattr(p, k, v)
    if not explicit_allele:
        p.min_support_allele = min(p.min_support, 5)  # cuteSV:1124,1141
    return p
