"""Host side of the boundary: decoded alignment records -> pinned-friendly columnar int32 buffers.

Packs the fields the reference reads at cuteSV:606-733 from duck-typed read objects (pysam records for CRAM / SAM
input, test doubles; plain BAM goes through the native decoder in bamio.py instead) (.flag .mapq .query_length
.query_name .reference_start .reference_end .cigartuples .get_tags()).
"""
import re

import numpy as np

_CIG = re.compile(r"(\d+)([MIDNSHP=X])")
_REFSPAN_OPS = frozenset("MD=X")


def acquire_clip_pos(cigar_string):
    """(first S length, last S length, ref span) of an SA-tag CIGAR string -- the three numbers the
    reference derives at cuteSV:466-481 (clips from a leading / trailing 'S' only; span = M+D+=+X)."""
    items = _CIG.findall(cigar_string)
    first = int(items[0][0]) if items and items[0][1] == "S" else 0
    last = int(items[-1][0]) if items and items[-1][1] == "S" else 0
    span = sum(int(n) for n, op in items if op in _REFSPAN_OPS)
    return first, last, span


def name_ranks(names):
    """Rank of every name in Python string order (the reference's tuple sorts break ties on the
    read-name string, cuteSV:764-801).  Returns (rank array, sorted unique names)."""
    uniq = sorted(set(names))
    index = {n: i for i, n in enumerate(uniq)}
    return np.fromiter((index[n] for n in names), dtype=np.int32, count=len(names)), uniq


def pack_alignments(reads, chrom_id, read_id):
    """reads: sequence of read objects; chrom_id: dict name -> contig id; read_id: dict name -> id;
    each read object needs `.reference_name`.  Returns dict(read_cols..., cigar, sa_cols...)."""
    n = len(reads)
    cols = {k: np.zeros(n, dtype=np.int32) for k in ("chrom", "ref_start", "ref_end", "flag", "mapq", "query_len", "read_id")}
    cigar_off = np.zeros(n + 1, dtype=np.int64)
    sa_off = np.zeros(n + 1, dtype=np.int64)
    cig = []
    sa = {k: [] for k in ("chrom", "pos0", "strand", "mapq", "first_clip", "last_clip", "ref_span")}
    for i, r in enumerate(reads):
        cols["chrom"][i] = chrom_id[r.reference_name]
        cols["ref_start"][i] = r.reference_start
        cols["ref_end"][i] = r.reference_end
        cols["flag"][i] = r.flag
        cols["mapq"][i] = r.mapq
        cols["query_len"][i] = r.query_length
        cols["read_id"][i] = read_id[r.query_name]
        for op, ln in r.cigartuples:
            cig.append((ln << 4) | op)
        cigar_off[i + 1] = len(cig)
        for tag in r.get_tags():
            if tag[0] == "SA":
                for ent in tag[1].split(";")[:-1]:  # cuteSV:678
                    f = ent.split(",")
                    first, last, span = acquire_clip_pos(f[3])
                    sa["chrom"].append(chrom_id[f[0]])
                    sa["pos0"].append(int(f[1]) - 1)  # SA pos is 1-based, cuteSV:497
                    sa["strand"].append(0 if f[2] == "+" else 1)
                    sa["mapq"].append(int(f[4]))
                    sa["first_clip"].append(first)
                    sa["last_clip"].append(last)
                    sa["ref_span"].append(span)
        sa_off[i + 1] = len(sa["chrom"])
    out = dict(cols)
    out["cigar_off"] = cigar_off
    out["sa_off"] = sa_off
    out["cigar"] = np.array(cig, dtype=np.uint32)
    out["sa"] = {k: np.array(v, dtype=np.int32) for k, v in sa.items()}
    return out


_COMP = str.maketrans("ACGTNacgtn", "TGCANtgcan")
_NIB_CODE = np.full(256, 15, dtype=np.uint8)   # BAM's 4-bit base codes, "=ACMGRSVTWYHKDBN"; any other character packs as N
for _i, _ch in enumerate("=ACMGRSVTWYHKDBN"):
    _NIB_CODE[ord(_ch)] = _i
    _NIB_CODE[ord(_ch.lower())] = _i


def pack_bases(strings):
    """BAM's 4-bit packed form of query sequences (high nibble first, "=ACMGRSVTWYHKDBN"; lower case packs as upper case):
    returns (seq4 uint8, seq_off int64 [n + 1]), the layout of bamio.BamReader.next_packet.  None or "" stores no bases
    (BAM '*')."""
    lens = np.fromiter((len(s) if s else 0 for s in strings), dtype=np.int64, count=len(strings))
    nb = (lens + 1) // 2
    seq_off = np.zeros(len(strings) + 1, dtype=np.int64)
    np.cumsum(nb, out=seq_off[1:])
    seq4 = np.zeros(int(seq_off[-1]), dtype=np.uint8)
    for i, s in enumerate(strings):
        if not s:
            continue
        code = _NIB_CODE[np.frombuffer(s.encode("ascii"), dtype=np.uint8)]
        if len(code) & 1:
            code = np.append(code, np.uint8(0))
        seq4[seq_off[i]:seq_off[i + 1]] = (code[0::2] << 4) | code[1::2]
    return seq4, seq_off


def revcomp(s):
    return s.translate(_COMP)[::-1]


def merged_ins_from_cigar(cigar, ref_start, query, pos, min_siglength, merge_ins_threshold):
    """Sequence of the merged insertion signature that starts at reference position `pos`: parse_read's CIGAR walk
    (cuteSV:616-645) + generate_combine_sigs' INS chain (cuteSV:530-545) on one record.  Only for signatures that merge more
    insertions than the device buffers (piece flag 2)."""
    ref = int(ref_start)
    first = int(cigar[0]) if len(cigar) else 0
    q = -(first >> 4) if (first & 15) == 5 else 0          # shift_ins_read starts at -hardclip_left
    groups = []                                              # [first pos, last pos, [slices]]
    for cg in cigar:
        op, ln = int(cg) & 15, int(cg) >> 4
        if op != 2:
            q += ln                                          # every op except D advances the query cursor (cuteSV:631-632)
        if ln >= min_siglength and op in (1, 2):
            if op == 2:
                ref += ln
            else:
                piece = query[q - ln:q]   # Python slice semantics, as the reference (cuteSV:639)
                if groups and ref - groups[-1][1] <= merge_ins_threshold:
                    groups[-1][1] = ref
                    groups[-1][2].append(piece)
                else:
                    groups.append([ref, ref, [piece]])
        elif op in (0, 2, 3, 7, 8):
            ref += ln
    for g in groups:
        if g[0] == pos:
            return "".join(g[2])
    raise ValueError("merged insertion at %d not found in the record's CIGAR" % pos)


def ins_sequence(pieces, off, cnt, query_of, cigar_of=None, merge=None):
    """Rebuild an INS signature's sequence from its piece list; query_of(rec) -> query string.
    A piece with flag 2 (more merged insertions than the device buffers) is rebuilt from the record's CIGAR:
    cigar_of(rec) -> (uint32 CIGAR array, reference_start), merge = (min_siglength, merge_ins_threshold)."""
    out = []
    for p in range(off, off + cnt):
        rec, a, b, rc = (int(x) for x in pieces[p])
        q = query_of(rec)
        if rc == 2:
            cig, ref_start = cigar_of(rec)
            out.append(merged_ins_from_cigar(cig, ref_start, q, a, merge[0], merge[1]))
            continue
        if rc:
            q = revcomp(q)
        out.append(q[a:b])
    return "".join(out)


class InsStore(object):
    """INS signature sequences by input index, kept as a few large ASCII buffers (one block per packet: uint8 bases +
    offsets) instead of one Python string per signature; a string is only materialised for the rows that need one (the
    representative signature of an emitted candidate, members of a tie group, the work-dir writer).  Sequences the
    vectorised builder does not cover, and rows moved by the tie ordering, live in an override table."""

    def __init__(self):
        self._first = []     # first input index of every block
        self._blocks = []    # (bases uint8, offsets int64 [k + 1])
        self._over = {}
        self._n = 0

    def __len__(self):
        return self._n

    def add_block(self, bases, offsets):
        self._first.append(self._n)
        self._blocks.append((bases, offsets))
        self._n += len(offsets) - 1

    def add_strings(self, strings):
        off = np.zeros(len(strings) + 1, dtype=np.int64)
        if len(strings):
            np.cumsum(np.fromiter(map(len, strings), dtype=np.int64, count=len(strings)), out=off[1:])
        self.add_block(np.frombuffer("".join(strings).encode("ascii"), dtype=np.uint8), off)

    def add_empty(self, k):
        self.add_block(np.zeros(0, dtype=np.uint8), np.zeros(k + 1, dtype=np.int64))

    def __getitem__(self, k):
        k = int(k)
        v = self._over.get(k)
        if v is not None:
            return v
        if not 0 <= k < self._n:
            raise IndexError(k)
        import bisect
        b = bisect.bisect_right(self._first, k) - 1
        bases, off = self._blocks[b]
        j = k - self._first[b]
        return bases[off[j]:off[j + 1]].tobytes().decode("ascii")

    def __setitem__(self, k, v):
        self._over[int(k)] = v

    def __iter__(self):
        for first, (bases, off) in zip(self._first, self._blocks):
            whole = bases.tobytes().decode("ascii")
            o = off.tolist()
            for j in range(len(o) - 1):
                v = self._over.get(first + j)
                yield whole[o[j]:o[j + 1]] if v is None else v


def ins_block_from_packed(pieces, po, pc, seq4, seq_lo, seq_hi, query_len):
    """Vectorised rebuild of the INS sequences of one packet from BAM's 4-bit packed bases.
    pieces: int32 [m, 4] = (packet record, a, b, rc); signature i = pieces po[i] .. po[i] + pc[i] (consecutive).
    Covers forward-strand pieces with non-negative slice bounds (q[a:b], clamped like a Python slice); returns
    (bases uint8, offsets int64 [n + 1], slow) where `slow` lists the signatures that need packing.ins_sequence
    (reverse complement, merged-from-CIGAR marker pieces, negative slice indices): they take no room in `bases`."""
    n = len(po)
    m = len(pieces)
    po = np.asarray(po, dtype=np.int64)
    pc = np.asarray(pc, dtype=np.int64)
    if n == 0:
        return np.zeros(0, dtype=np.uint8), np.zeros(1, dtype=np.int64), np.zeros(0, dtype=np.int64)
    contiguous = po[0] == 0 and bool(np.all(po[1:] == po[:-1] + pc[:-1])) and po[-1] + pc[-1] == m
    if not contiguous:
        # the device hands out piece slots with atomics: a signature's pieces are consecutive, the signatures are in no
        # particular order -> bring the pieces into signature order first
        start = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(pc, out=start[1:])
        order = np.repeat(po - start[:-1], pc) + np.arange(int(start[-1]), dtype=np.int64)
        if len(order) and (order.min() < 0 or order.max() >= m):
            return np.zeros(0, dtype=np.uint8), np.zeros(n + 1, dtype=np.int64), np.arange(n, dtype=np.int64)
        pieces = np.asarray(pieces)[order]
        po = start[:-1]
        m = len(pieces)
    rec = pieces[:, 0].astype(np.int64)
    a = pieces[:, 1].astype(np.int64)
    b = pieces[:, 2].astype(np.int64)
    ql = np.asarray(query_len, dtype=np.int64)[rec]
    lo = np.asarray(seq_lo, dtype=np.int64)[rec]
    have = (np.asarray(seq_hi, dtype=np.int64)[rec] - lo) >= (ql + 1) // 2      # '*' query: every slice is empty
    simple_piece = (pieces[:, 3] == 0) & (a >= 0) & (b >= 0)
    sig_of_piece = np.repeat(np.arange(n, dtype=np.int64), pc)
    bad_sig = np.zeros(n, dtype=bool)
    bad_sig[sig_of_piece[~simple_piece]] = True
    a2 = np.minimum(a, ql)
    plen = np.where(have, np.maximum(np.minimum(b, ql) - a2, 0), 0)
    plen[bad_sig[sig_of_piece]] = 0
    pstart = np.zeros(m + 1, dtype=np.int64)
    np.cumsum(plen, out=pstart[1:])
    from . import bamio   # the unpacking loop is C (libcutesv_bam.so, the library the packed bases come from)
    bases = bamio.unpack_ranges(seq4, 2 * lo + a2, plen, pstart[:-1], pstart[-1])
    offsets = np.concatenate([pstart[po], pstart[-1:]])
    return bases, offsets, np.flatnonzero(bad_sig)
