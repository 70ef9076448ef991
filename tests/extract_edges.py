"""Planted layouts for k_extract (cutesv_b200/csrc/extract.cuh) at the edges of its CIGAR walk, which the CPU emulator does not
share: the 256-op tiles (8 consecutive ops per lane), the 512-op chunks fetched by one bulk copy from `c_lo & ~3` and picked
out at `d0 = c_lo & 3`, the two-slot ring, the lazy offsets of tiles without a qualifying op, the serial hand-over to lane 0,
the 64-piece buffer of an open merged insertion (MAX_OPEN_PIECES, extract_core.h) and the output-capacity reruns of
extract_api.inl.

Every case is a packet of SynthRead records built from explicit op lists, with query sequences, so that the reference's
parse_read can run on them (oracle/gen_extract_edges_golden.py).  Filler records of 1-3 ops (some skipped by mapq,
min_read_len or flag 256 / 272) set each planted record's d0.  For every qualifying op the builder records where the kernel
meets it (index, tile, lane, item, chunk, ring slot, d0) and what it must yield (reference position, length, query slice), and
`expected` states parse_read's output for a parameter set from those literals.  Nothing here calls the library."""
import numpy as np

from cutesv_b200 import _abi, packing
from cutesv_b200.synth import SynthRead

# k_extract's walk (extract.cuh) and the open-piece buffer (extract_core.h)
EX_ITEMS, EX_TILE, EX_CHUNK, EX_RING = 8, 256, 512, 2
MAX_OPEN_PIECES = 64
M, I, D, N, S, H, P, EQ, X = 0, 1, 2, 3, 4, 5, 6, 7, 8
MIN_SIG = 10   # min_siglength of every parameter set
CONTIG, CONTIG_LEN = "chr1", 1 << 30

# the parameter sets the golden holds: the defaults, no merging (and no min_read_len, so one-op D / H records are parsed), and
# thresholds at which the merge cases' DEL pairs join (first-signature rule) and INS chains run long
PARAMS = {
    "defaults": {},
    "zero": dict(merge_del_threshold=0, merge_ins_threshold=0, min_read_len=0),
    "merge": dict(merge_del_threshold=100, merge_ins_threshold=300),
}
LENGTHS = (1, 8, 9, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 1536, 1537, 2048, 2049)
EDGE_IDX = (7, 8, 255, 256, 511, 512, 1023, 1024, 1535, 1536)
CHAINS = (63, 64, 65, 66)
_QUERY_OPS = (M, I, S, EQ, X)   # what query_length counts
_REF_OPS = (M, D, N, EQ, X)     # what advances the reference (cuteSV:592-603)


def params(name):
    return _abi.default_params(**PARAMS[name])


def name_of(rec):
    """Read names sort in record order, so a record's read id (its name's rank) is its index in the packet."""
    return "r%05d" % rec


def where(i, d0):
    """Where k_extract meets op i of a record whose CIGAR starts d0 words past a 16 B boundary."""
    return dict(i=i, tile=i // EX_TILE, lane=(i % EX_TILE) // EX_ITEMS, item=i % EX_ITEMS, chunk=i // EX_CHUNK,
                slot=(i // EX_CHUNK) % EX_RING, d0=d0)


def walk(ops, ref_start, query, min_sig=MIN_SIG):
    """Every qualifying op of a record: parse_read's walk (cuteSV:616-645) stated on the op list.  The query cursor starts at
    minus a leading hard clip and advances on every op but D (also on H, S, N and P), the reference on M D N = X."""
    ref = ref_start
    q = -ops[0][1] if ops and ops[0][0] == H else 0
    out = []
    for i, (op, ln) in enumerate(ops):
        if op != D:
            q += ln
        if ln >= min_sig and op in (I, D):
            if op == D:
                out.append(dict(idx=i, kind="DEL", pos=ref, len=ln))
                ref += ln
            else:
                out.append(dict(idx=i, kind="INS", pos=ref, len=ln, seq=query[q - ln:q]))   # Python slice, as cuteSV:639
        elif op in _REF_OPS:
            ref += ln
    return out


def combine(sigs, merge_del, merge_ins):
    """generate_combine_sigs (cuteSV:515-575) on one record's qualifying ops: INS joins when its position is within merge_ins
    of the last joined insertion; DEL compares with the END of the first signature and, after a flush, with the START of the
    new one."""
    ins, dels = [], []
    cur = None
    for s in (x for x in sigs if x["kind"] == "INS"):
        if cur is not None and s["pos"] - cur["last"] <= merge_ins:
            cur["len"] += s["len"]; cur["seq"] += s["seq"]; cur["last"] = s["pos"]; cur["n"] += 1
            continue
        if cur is not None:
            ins.append(cur)
        cur = dict(pos=s["pos"], len=s["len"], seq=s["seq"], last=s["pos"], n=1)
    if cur is not None:
        ins.append(cur)
    cur = None
    for s in (x for x in sigs if x["kind"] == "DEL"):
        if cur is not None and s["pos"] - cur["cmp"] <= merge_del:
            cur["len"] += s["len"]; cur["cmp"] = s["pos"] + s["len"]
            continue
        first = cur is None
        if cur is not None:
            dels.append(cur)
        cur = dict(pos=s["pos"], len=s["len"], cmp=s["pos"] + s["len"] if first else s["pos"])
    if cur is not None:
        dels.append(cur)
    return [(d["pos"], d["len"]) for d in dels], [(x["pos"], x["len"], x["seq"], x["n"]) for x in ins]


class _Packet(object):
    def __init__(self, name, seed):
        self.name = name
        self.rng = np.random.default_rng(seed)
        self.reads, self.info = [], []
        self.n_ops = 0
        self.pos = 10_000
        self.n_fill = 0

    def _query(self, ops):
        n = sum(ln for op, ln in ops if op in _QUERY_OPS)
        return "".join(self.rng.choice(list("ACGT"), n)) if n else ""

    def add(self, ops, flag=0, mapq=60, label=None, **meta):
        rec = len(self.reads)
        r = SynthRead()
        r.flag, r.mapq, r.query_name, r.reference_name = flag, mapq, name_of(rec), CONTIG
        r.query_sequence = self._query(ops)
        r.query_length = len(r.query_sequence)
        r.reference_start = self.pos
        r.reference_end = self.pos + sum(ln for op, ln in ops if op in _REF_OPS)
        r.cigartuples = [(int(op), int(ln)) for op, ln in ops]
        r.cigar = r.cigartuples
        r.tags = []
        self.pos = r.reference_end + 5_000
        d0 = self.n_ops % 4
        sigs = walk(r.cigartuples, r.reference_start, r.query_sequence) if label else []
        for s in sigs:
            s.update(where(s["idx"], d0))
        self.info.append(dict(rec=rec, label=label, n_ops=len(ops), d0=d0, cigar_off=self.n_ops, flag=flag, mapq=mapq, sigs=sigs, **meta))
        self.reads.append(r)
        self.n_ops += len(ops)
        return rec

    def filler(self, k):
        """A record of k (1-3) ops that yields no signature: by turns one the reference skips for flag 256 / 272, for mapq, for
        min_read_len, or parses to nothing."""
        kind = self.n_fill % 5
        self.n_fill += 1
        if kind == 3:   # query_len < min_read_len (500)
            ops = [(S, 20), (M, 100), (S, 20)][:k] if k > 1 else [(M, 100)]
        else:
            ops = [(S, 30), (M, 600), (S, 30)][:k] if k > 1 else [(M, 600)]
            if k == 2:
                ops = [(M, 300), (EQ, 300)]
        flag, mapq = (256, 60) if kind == 0 else (272, 60) if kind == 1 else (0, 3) if kind == 2 else (16, 60)
        self.add(ops, flag=flag, mapq=mapq)

    def align(self, d0):
        """Fillers so that the next record's CIGAR starts at d0 (mod 4); at least one filler precedes every planted record."""
        need = (d0 - self.n_ops) % 4
        for k in {0: (1, 3), 1: (1,), 2: (2,), 3: (3,)}[need]:
            self.filler(k)

    def m(self):
        return int(self.rng.integers(20, 61))

    def ins(self):
        return int(self.rng.integers(MIN_SIG, 41))

    def dele(self):
        return int(self.rng.integers(MIN_SIG, 61))

    def body(self, n):
        """n ops that advance reference and query and never qualify (M, = and X)."""
        code = self.rng.choice([M, M, M, EQ, X], n)
        return [(int(c), self.m()) for c in code]

    def packet(self):
        cid = {CONTIG: 0}
        rid = {name_of(i): i for i in range(len(self.reads))}
        return packing.pack_alignments(self.reads, cid, rid)

    def case(self):
        pk = self.packet()
        assert [int(x["cigar_off"]) for x in self.info] == pk["cigar_off"][:-1].tolist()
        return dict(name=self.name, reads=self.reads, names=[CONTIG], lens=[CONTIG_LEN], rnames=[name_of(i) for i in range(len(self.reads))],
                    pk=pk, records=self.info)


def _plant(ops, idx, kinds, b):
    for i, k in zip(idx, kinds):
        ops[i] = (I, b.ins()) if k == "I" else (D, b.dele())
    return ops


def case_lengths():
    """Records of L ops at every d0, in two shapes: soft clips at both ends (qualifying ops on the first op after the clip and
    the last op before the trailing clip), and a leading hard clip with the record's last op qualifying.  Both carry
    qualifying ops at EDGE_IDX; I and D alternate, starting with I or D by turns, so that adjacent indices never merge."""
    b = _Packet("lengths", 11)
    turn = 0
    for L in LENGTHS:
        for d0 in range(4):
            for shape in ("clip", "open"):
                if L == 1:
                    if shape == "clip":
                        continue
                    ops, idx = [(I, 600)], [0]
                elif shape == "clip":
                    ops = [(S, 40)] + b.body(L - 2) + [(S, 40)]
                    idx = sorted({1, L - 2} | {i for i in EDGE_IDX if 1 <= i <= L - 2})
                else:
                    ops = [(H, 40)] + b.body(L - 1)
                    idx = sorted({1, L - 1} | {i for i in EDGE_IDX if 1 <= i <= L - 1})
                kinds = ["ID"[(j + turn) % 2] for j in range(len(idx))] if L > 1 else ["I"]
                turn += 1
                if L == 1:
                    ops[0] = (I, 600)   # the whole query is the insertion (query_len >= min_read_len)
                else:
                    ops = _plant(ops, idx, kinds, b)
                b.align(d0)
                b.add(ops, label="L%d_d%d_%s" % (L, d0, shape), L=L, shape=shape)
    return b.case()


def case_lanes():
    """Tile 1 of the first record: every lane has a qualifying op at item 0 and at item 7.  Tile 2 of the second: lane 5
    holds four (I M I M D M D M), the first two within merge_ins_threshold of each other."""
    b = _Packet("lanes", 12)
    for d0 in (1, 3):
        ops = [(S, 40)] + b.body(600)
        for lane in range(32):
            ops[EX_TILE + 8 * lane] = (I, b.ins()) if lane % 2 == 0 else (D, b.dele())
            ops[EX_TILE + 8 * lane + 7] = (D, b.dele()) if lane % 2 == 0 else (I, b.ins())
        b.align(d0)
        b.add(ops, label="every_lane_d%d" % d0)
        ops = [(S, 40)] + b.body(800)
        base = 2 * EX_TILE + 5 * EX_ITEMS
        for j, k in enumerate("IMIMDMDM"):
            ops[base + j] = (I, b.ins()) if k == "I" else (D, b.dele()) if k == "D" else (M, 15)
        b.align(3 - d0)
        b.add(ops, label="one_lane_d%d" % (3 - d0))
    return b.case()


def _gap_ops(b, n):
    """n ops that never qualify, of every class that advances something: M, =, X, N, P of nonzero length (the reference advances
    the query on P and N too), and I / D of min_siglength - 1."""
    code = b.rng.choice([M, EQ, X, N, P, I, D], n)
    out = []
    for c in code:
        c = int(c)
        out.append((c, MIN_SIG - 1) if c in (I, D) else (c, b.m()))
    return out


def case_gaps():
    """Qualifying ops 1, 2, 3 and 5 tiles apart with none between (the lazy per-lane offsets fold them in), behind three kinds
    of leading clip in front of an early INS: hard + soft, soft only, hard only."""
    b = _Packet("gaps", 13)
    tiles = [0, 1, 3, 6, 11]
    for d0, lead in ((0, [(H, 50), (S, 30)]), (2, [(S, 30)]), (1, [(H, 70)]), (3, [(H, 20), (S, 10)])):
        ops = lead + [(I, b.ins())] + _gap_ops(b, 12 * EX_TILE)
        for j, t in enumerate(tiles[1:]):
            i = t * EX_TILE + int(b.rng.integers(0, EX_TILE))
            ops[i] = (I, b.ins()) if (j + d0) % 2 == 0 else (D, b.dele())
        ops[tiles[0] * EX_TILE + 200] = (D, b.dele())
        b.align(d0)
        b.add(ops, label="gaps_d%d" % d0)
    return b.case()


def case_thresholds():
    """I and D of min_siglength - 1 and min_siglength on the last op of a tile and the first op of the next (255 / 256 and the
    chunk edge 511 / 512)."""
    b = _Packet("thresholds", 14)
    r = 0
    for k_last, k_first in (("I", "I"), ("I", "D"), ("D", "I"), ("D", "D")):
        for short_last in (True, False):
            ops = [(S, 40)] + b.body(700)
            for e in (EX_TILE, EX_CHUNK):
                ops[e - 1] = (I if k_last == "I" else D, MIN_SIG - 1 if short_last else MIN_SIG)
                ops[e] = (I if k_first == "I" else D, MIN_SIG if short_last else MIN_SIG - 1)
            b.align(r % 4)
            b.add(ops, label="thr_%s%s_%s" % (k_last, k_first, "short_last" if short_last else "short_first"))
            r += 1
    return b.case()


def case_merges():
    """DEL pairs that merge_del_threshold joins: the first at op 255 / 511 / 1023 and the second two ops later, D 80 and M 40 so
    that the pair joins under the first-signature rule (compared with the first DEL's END) and not under the later one (its
    START).  INS chains of 63-66 insertions 20-60 bp apart, starting on op 511 (last op of tile 1 and of chunk 0); the last
    one ends on the record's last op."""
    b = _Packet("merges", 15)
    for j, first in enumerate((EX_TILE - 1, EX_CHUNK - 1, 2 * EX_CHUNK - 1)):
        ops = [(S, 40)] + b.body(1100)
        for k, e in enumerate((EX_TILE - 1, EX_CHUNK - 1, 2 * EX_CHUNK - 1)):
            if e < first:
                continue
            ops[e], ops[e + 1], ops[e + 2] = (D, 80), (M, 40), (D, 60)
        b.align(j)
        b.add(ops, label="del_pairs_from_%d" % first)
    for j, k in enumerate(CHAINS):
        last = j == len(CHAINS) - 1
        n = EX_CHUNK - 1 + 2 * k - 1 + (0 if last else 300)
        ops = [(S, 40)] + b.body(n - 1)
        for c in range(k):
            ops[EX_CHUNK - 1 + 2 * c] = (I, b.ins())
        b.align((j + 1) % 4)
        b.add(ops, label="ins_chain_%d" % k, chain=k)
    return b.case()


def case_one_op():
    """Records whose whole CIGAR is one M, I, D, S or H op, between longer records."""
    b = _Packet("one_op", 16)
    for j, op in enumerate((M, I, D, S, H)):
        ops = [(S, 40)] + b.body(300)
        ops[100] = (I, b.ins())
        b.align(j % 4)
        b.add(ops, label="before_%d" % op)
        b.add([(op, 600 if op in (M, I, S) else 50 if op == D else 600)], label="one_op_%d" % op)
    b.add([(S, 40)] + b.body(20) + [(D, 30)] + b.body(20), label="after")
    return b.case()


CASES = ("lengths", "lanes", "gaps", "thresholds", "merges", "one_op")
_BUILD = dict(lengths=case_lengths, lanes=case_lanes, gaps=case_gaps, thresholds=case_thresholds, merges=case_merges, one_op=case_one_op)
_CACHE = {}


def case(name):
    if name not in _CACHE:
        _CACHE[name] = _BUILD[name]()
    return _CACHE[name]


def expected(c, pname):
    """parse_read's DEL and INS signatures of every record of case c under parameter set pname, from the planted literals:
    {rec: (dels [(pos, len)], ins [(pos, len, seq, n_pieces)])}, only for records the reference parses."""
    p = params(pname)
    out = {}
    for info, r in zip(c["records"], c["reads"]):
        if info["flag"] in (256, 272) or r.query_length < p.min_read_len or r.mapq < p.min_mapq:
            continue
        out[info["rec"]] = combine(info["sigs"], p.merge_del_threshold, p.merge_ins_threshold)
    return out


def expected_rows(c, pname):
    """reads_info_list rows (cuteSV:729-733) in record order: (start, end, is_primary, name, contig)."""
    p = params(pname)
    return [(r.reference_start, r.reference_end, 1 if r.flag in (0, 16) else 0, r.query_name, CONTIG)
            for r in c["reads"] if r.flag not in (256, 272) and r.mapq >= p.min_mapq]


def planted(c):
    """Every qualifying op of the case with its record's label: the table the edge assertions read."""
    return [dict(s, rec=info["rec"], label=info["label"]) for info in c["records"] for s in info["sigs"]]


# ---------------------------------------------------------------------------------------------------------------------
# packets built as numpy columns (no SynthRead): the ring-parity case and the output-capacity reruns
# ---------------------------------------------------------------------------------------------------------------------
def parity_packet(n=32768, seed=21):
    """n records of 257-2049 ops (1-5 chunks, odd and even counts): several records per resident warp, so the ring's mbarrier
    parity carries from record to record.  Mostly M / = / X ops with N, P and sub-threshold I / D, and about six qualifying
    I / D ops per record at random indices."""
    rng = np.random.default_rng(seed)
    L = rng.integers(257, 2050, n).astype(np.int64)
    off = np.zeros(n + 1, np.int64)
    np.cumsum(L, out=off[1:])
    tot = int(off[-1])
    op = rng.choice(np.array([M, M, M, M, EQ, X, N, P, I, D], np.uint32), tot)
    ln = rng.integers(20, 61, tot).astype(np.uint32)
    ln[(op == I) | (op == D)] = MIN_SIG - 1
    q = rng.random(tot) < 6.0 / 1150
    op[q] = np.where(rng.random(int(q.sum())) < 0.5, I, D).astype(np.uint32)
    ln[q] = rng.integers(MIN_SIG, 80, int(q.sum())).astype(np.uint32)
    first = off[:-1]
    op[first] = np.where(rng.random(n) < 0.3, H, S).astype(np.uint32)   # leading clips: the query cursor starts at -H
    cigar = (ln << 4) | op
    rec_of = np.repeat(np.arange(n), L)
    qlen = np.bincount(rec_of, weights=np.where(np.isin(op, _QUERY_OPS), ln, 0), minlength=n).astype(np.int32)
    span = np.bincount(rec_of, weights=np.where(np.isin(op, _REF_OPS), ln, 0), minlength=n).astype(np.int64)
    start = (np.arange(n, dtype=np.int64) * 1000 % (CONTIG_LEN - 200_000)).astype(np.int32)
    z = np.zeros(0, np.int32)
    return dict(chrom=np.zeros(n, np.int32), ref_start=start, ref_end=(start + span).astype(np.int32), flag=np.zeros(n, np.int32),
                mapq=np.full(n, 60, np.int32), query_len=qlen, read_id=np.arange(n, dtype=np.int32), cigar_off=off,
                sa_off=np.zeros(n + 1, np.int64), cigar=cigar.astype(np.uint32), sa={k: z for k in ("chrom", "pos0", "strand", "mapq", "first_clip",
                                                                                                   "last_clip", "ref_span")})


def rerun_packet(n, dels=0, ins=0, pieces=1, seed=0, rec0=0):
    """n records with `dels` DEL rows and `ins` INS rows of `pieces` merged insertions each, spread over the records as evenly
    as possible, under the default parameters: DELs 30 bp apart (merge_del_threshold 0), insertions of one row 20 bp apart and
    rows 200 bp apart (merge_ins_threshold 100).  Returns (reads, names, packet); names continue from rec0."""
    b = _Packet("rerun", seed)
    for r in range(n):
        nd = dels // n + (1 if r < dels % n else 0)
        ni = ins // n + (1 if r < ins % n else 0)
        ops = [(S, 20), (M, 600)]
        for _ in range(nd):
            ops += [(D, 20), (M, 30)]
        for _ in range(ni):
            for k in range(pieces):
                ops += [(I, 12), (M, 20 if k < pieces - 1 else 200)]
        r_ = b.add(ops, label="rerun")
        b.reads[r_].query_name = name_of(rec0 + r_)
    rid = {name_of(rec0 + i): rec0 + i for i in range(n)}
    return b.reads, [x.query_name for x in b.reads], packing.pack_alignments(b.reads, {CONTIG: 0}, rid)


# ---------------------------------------------------------------------------------------------------------------------
# per-record views of the reference's tuple lists
# ---------------------------------------------------------------------------------------------------------------------
def ordered(cand):
    """{read name: ([(pos, len)] DEL, [(pos, len, seq)] INS)} in list order (parse_read's emission order within a record) from
    the reference's candidate tuples (cuteSV:520-575) or compare_extract.tuples_from_columns."""
    out = {}
    for t in cand["DEL"]:
        out.setdefault(t[2], ([], []))[0].append((float(t[0]), int(t[1])))
    for t in cand["INS"]:
        out.setdefault(t[2], ([], []))[1].append((float(t[0]), int(t[1]), t[3]))
    return out


def expected_ordered(c, pname):
    """expected() in the shape of ordered(), records without a signature left out."""
    out = {}
    for rec, (dels, ins) in expected(c, pname).items():
        if dels or ins:
            out[name_of(rec)] = ([(float(a), b) for a, b in dels], [(float(a), b, s) for a, b, s, _ in ins])
    return out
