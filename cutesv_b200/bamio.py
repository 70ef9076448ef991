"""Native BAM decoder binding (libcutesv_bam.so, csrc/bam_reader.cpp): BGZF/BAM -> the columnar packet
`Engine.extract` consumes, without a Python loop over reads (replaces the pysam iteration of
cuteSV:709-733 and the per-read packing of packing.pack_alignments for plain BAM input).

Sequential decode only; the .bai (or .csi) is read just for the per-contig mapped counts that size the task
windows (get_index_statistics, cuteSV:1015-1025).
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "bam_reader.cpp")
SO = os.path.join(HERE, "libcutesv_bam.so")
_lib = None

_I32P, _I64P = C.POINTER(C.c_int32), C.POINTER(C.c_int64)


class _Packet(C.Structure):
    _fields_ = ([("n", C.c_int64)] + [(k, _I32P) for k in ("chrom", "ref_start", "ref_end", "flag", "mapq", "query_len", "read_id")]
                + [("cigar_off", _I64P), ("sa_off", _I64P), ("n_cigar", C.c_int64), ("cigar", C.POINTER(C.c_uint32)), ("n_sa", C.c_int64)]
                + [(k, _I32P) for k in ("sa_chrom", "sa_pos0", "sa_strand", "sa_mapq", "sa_first", "sa_last", "sa_span")]
                + [("seq_off", _I64P), ("seq4", C.POINTER(C.c_uint8))])


def build(force=False):
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < os.path.getmtime(SRC):
        subprocess.check_call([os.environ.get("CXX_HOST", "/usr/bin/g++"), "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC, "-lz", "-pthread"])
    return SO


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            raise RuntimeError("libcutesv_bam.so is not built; run `python -m cutesv_b200.build`")
        L = C.CDLL(SO)
        L.bamr_error.restype = C.c_char_p
        L.bamr_open.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]
        L.bamr_close.argtypes = [C.c_void_p]
        L.bamr_n_ref.argtypes = [C.c_void_p]
        L.bamr_ref_name.argtypes = [C.c_void_p, C.c_int32]
        L.bamr_ref_name.restype = C.c_char_p
        L.bamr_ref_len.argtypes = [C.c_void_p, C.c_int32]
        L.bamr_ref_len.restype = C.c_int64
        L.bamr_set_chrom_ids.argtypes = [C.c_void_p, _I32P]
        L.bamr_keep_seq.argtypes = [C.c_void_p, C.c_int]
        L.bamr_tune.argtypes = [C.c_void_p, C.c_int, C.c_int64]
        L.bamr_next.argtypes = [C.c_void_p, C.c_int64, C.POINTER(_Packet)]
        L.bamr_next.restype = C.c_int64
        L.bamr_n_names.argtypes = [C.c_void_p]
        L.bamr_n_names.restype = C.c_int64
        L.bamr_name.argtypes = [C.c_void_p, C.c_int64]
        L.bamr_name.restype = C.c_char_p
        L.bamr_name_ranks.argtypes = [C.c_void_p, _I32P]
        L.bamr_decode_seq.argtypes = [C.c_void_p, C.c_int64, C.c_char_p]
        L.bamr_index_stats.argtypes = [C.c_char_p, C.c_int32, _I64P]
        L.bamr_unpack_ranges.argtypes = [C.c_void_p, C.c_int64, _I64P, _I64P, _I64P, C.c_void_p]
        L.bamr_unpack_ranges.restype = None
        _lib = L
    return _lib


def _arr(ptr, n, dtype, copy=True):
    if n == 0:
        return np.zeros(0, dtype=dtype)
    a = np.ctypeslib.as_array(ptr, shape=(n,))
    return a.astype(dtype, copy=True) if copy else a


def is_bam(path):
    """True for a BGZF file (gzip magic + FEXTRA): the native decoder's input."""
    with open(path, "rb") as f:
        h = f.read(4)
    return len(h) == 4 and h[0] == 31 and h[1] == 139 and h[2] == 8 and (h[3] & 4) != 0


class BamReader(object):
    def __init__(self, path, threads=4, keep_seq=True):
        self._h = C.c_void_p()
        self.path = path
        if lib().bamr_open(os.fsencode(path), int(threads), C.byref(self._h)) != 0:
            raise IOError(lib().bamr_error().decode())
        L = lib()
        n = L.bamr_n_ref(self._h)
        self.references = [L.bamr_ref_name(self._h, i).decode() for i in range(n)]
        self.lengths = [int(L.bamr_ref_len(self._h, i)) for i in range(n)]
        L.bamr_keep_seq(self._h, 1 if keep_seq else 0)

    def tune(self, batch_blocks=0, headroom=-1):
        """Chunking knobs (tests): BGZF blocks per chunk, bytes reserved in front of a chunk for a straddling record."""
        lib().bamr_tune(self._h, int(batch_blocks), int(headroom))

    def close(self):
        if self._h:
            lib().bamr_close(self._h)
            self._h = C.c_void_p()

    def get_reference_length(self, name):
        return self.lengths[self.references.index(name)]

    def index_statistics(self):
        """[(contig, mapped)] in header order, like pysam's get_index_statistics().  Reads <bam>.bai or <stem>.bai, else the
        CSI index <bam>.csi or <stem>.csi (`samtools index -c`, which contigs longer than 2^29 bp need)."""
        stem = os.path.splitext(self.path)[0]
        cands = [self.path + ".bai", stem + ".bai", self.path + ".csi", stem + ".csi"]
        idx = next((p for p in cands if os.path.exists(p)), cands[1])
        mapped = np.zeros(max(len(self.references), 1), dtype=np.int64)
        if lib().bamr_index_stats(os.fsencode(idx), len(self.references), mapped.ctypes.data_as(_I64P)) != 0:
            raise IOError(lib().bamr_error().decode())
        return [(n, int(mapped[i])) for i, n in enumerate(self.references)]

    def set_chrom_ids(self, chrom_id):
        ids = np.array([chrom_id.get(n, -1) for n in self.references], dtype=np.int32)
        lib().bamr_set_chrom_ids(self._h, ids.ctypes.data_as(_I32P))

    def next_packet(self, max_records, copy=True):
        """Next packet (dict like packing.pack_alignments + 'seq_off'/'seq4'), or None at EOF.
        read_id holds provisional ids (first-seen order); see name_ranks().
        copy=False returns views of the decoder's own buffers, valid until the next call."""
        p = _Packet()
        n = lib().bamr_next(self._h, int(max_records), C.byref(p))
        if n < 0:
            raise IOError(lib().bamr_error().decode())
        if n == 0:
            return None
        out = {k: _arr(getattr(p, k), n, np.int32, copy) for k in ("chrom", "ref_start", "ref_end", "flag", "mapq", "query_len", "read_id")}
        out["cigar_off"] = _arr(p.cigar_off, n + 1, np.int64, copy)
        out["sa_off"] = _arr(p.sa_off, n + 1, np.int64, copy)
        out["cigar"] = _arr(p.cigar, p.n_cigar, np.uint32, copy)
        out["sa"] = {k: _arr(getattr(p, "sa_" + s), p.n_sa, np.int32, copy) for k, s in
                     (("chrom", "chrom"), ("pos0", "pos0"), ("strand", "strand"), ("mapq", "mapq"), ("first_clip", "first"),
                      ("last_clip", "last"), ("ref_span", "span"))}
        out["seq_off"] = _arr(p.seq_off, n + 1, np.int64, copy)
        out["seq4"] = _arr(p.seq4, int(out["seq_off"][-1]), np.uint8, copy)
        return out

    def names(self):
        L = lib()
        return [L.bamr_name(self._h, i).decode() for i in range(L.bamr_n_names(self._h))]

    def name_ranks(self):
        n = lib().bamr_n_names(self._h)
        r = np.zeros(max(n, 1), dtype=np.int32)
        lib().bamr_name_ranks(self._h, r.ctypes.data_as(_I32P))
        return r


# BAM packs two bases per byte (high nibble first, "=ACMGRSVTWYHKDBN"): one 16-bit table look-up per byte
_NIB = "=ACMGRSVTWYHKDBN"
_LUT16 = np.array([ord(_NIB[b >> 4]) | (ord(_NIB[b & 15]) << 8) for b in range(256)], dtype="<u2")


def decode_seq(packet, rec):
    """Query sequence (ASCII) of record `rec` of a packet."""
    l_seq = int(packet["query_len"][rec])
    if "seq_lo" in packet:   # a subset that still refers to the bases of its parent packet (subset_packet)
        o, end = int(packet["seq_lo"][rec]), int(packet["seq_hi"][rec])
    else:
        o, end = int(packet["seq_off"][rec]), int(packet["seq_off"][rec + 1])
    if end - o < (l_seq + 1) // 2:
        return ""
    return _LUT16[packet["seq4"][o:o + (l_seq + 1) // 2]].view(np.uint8)[:l_seq].tobytes().decode("ascii")


def unpack_ranges(seq4, nib0, length, out_off, total):
    """ASCII bases of many ranges of BAM's 4-bit packed bases in one C call (range i: `length[i]` bases from nibble `nib0[i]`)."""
    out = np.empty(int(total), dtype=np.uint8)
    n = len(nib0)
    if n and total:
        seq4 = np.ascontiguousarray(seq4, dtype=np.uint8)
        nib0, length, out_off = (np.ascontiguousarray(x, dtype=np.int64) for x in (nib0, length, out_off))
        lib().bamr_unpack_ranges(seq4.ctypes.data_as(C.c_void_p), n, nib0.ctypes.data_as(_I64P), length.ctypes.data_as(_I64P),
                                 out_off.ctypes.data_as(_I64P), out.ctypes.data_as(C.c_void_p))
    return out


def subset_packet(pk, keep):
    """Rows `keep` (index array, ascending) of a packet, CSR arrays rebuilt.  The kept rows form few long runs (the scan drops
    a few percent of the records), so the variable-length parts are copied run by run, not element by element."""
    keep = np.asarray(keep, dtype=np.int64)
    n = len(pk["chrom"])
    if len(keep) == n:
        return pk
    out = {k: pk[k][keep] for k in ("chrom", "ref_start", "ref_end", "flag", "mapq", "query_len", "read_id")}
    if len(keep):
        brk = np.flatnonzero(np.diff(keep) != 1)
        run_a = keep[np.concatenate([[0], brk + 1])]
        run_b = keep[np.concatenate([brk, [len(keep) - 1]])] + 1
    else:
        run_a = run_b = np.zeros(0, dtype=np.int64)

    def regather(off, arrays):
        lens = (off[1:] - off[:-1])[keep]
        new_off = np.zeros(len(keep) + 1, dtype=np.int64)
        np.cumsum(lens, out=new_off[1:])
        lo, hi = off[run_a].tolist(), off[run_b].tolist()
        return new_off, [np.concatenate([v[x:y] for x, y in zip(lo, hi)]) if len(lo) else v[:0] for v in arrays]
    out["cigar_off"], (out["cigar"],) = regather(pk["cigar_off"], [pk["cigar"]])
    keys = list(pk["sa"].keys())
    out["sa_off"], vals = regather(pk["sa_off"], [pk["sa"][k] for k in keys])
    out["sa"] = dict(zip(keys, vals))
    if "seq_off" in pk:   # the packed bases are not copied: only the host reads them (decode_seq), through the parent's offsets
        out["seq4"] = pk["seq4"]
        out["seq_lo"] = pk["seq_off"][:-1][keep]
        out["seq_hi"] = pk["seq_off"][1:][keep]
    return out
