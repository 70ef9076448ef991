"""CPU: extraction packets from GPU memory.  _abi.device_packet's normalisation with stand-in __cuda_array_interface__ objects;
packing.pack_bases; and the device's INS sequence routines (extract_core.h, compiled for the host from
tests/emul/emul_ins_seq.cpp) reproducing the REAL reference's INS strings from the emulator's piece lists."""
import collections
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import device_packet_util as dpu
import emul_lib
import golden_util
from cutesv_b200 import _abi, bamio, cli, packing
from oracle import compare_extract
from test_device_inputs_cpu import FakeDev
from test_extract_cpu import EXTRACT_GOLDENS, _run, _seed_golden

# ---- _abi.device_packet ----


def fake_packet(n=5, n_cigar=40, n_sa=3, n_bytes=30, seq=True, **over):
    pk = {f: FakeDev(n, addr=0x1000 * (k + 1)) for k, f in enumerate(_abi.READ_FIELDS)}
    pk["cigar_off"] = FakeDev(n + 1, "<i8", addr=0x10000)
    pk["sa_off"] = FakeDev(n + 1, "<i8", addr=0x20000)
    pk["cigar"] = FakeDev(n_cigar, "<u4", addr=0x30000)
    pk["sa"] = {f: FakeDev(n_sa, addr=0x40000 + 0x100 * k) for k, f in enumerate(_abi.SA_FIELDS)}
    if seq:
        pk["seq_off"] = FakeDev(n + 1, "<i8", addr=0x50000)
        pk["seq4"] = FakeDev(n_bytes, "|u1", addr=0x60000)
    for k, v in over.items():
        if k.startswith("sa."):
            pk["sa"] = dict(pk["sa"], **{k[3:]: v})
        else:
            pk[k] = v
    return pk


def addr(p):
    return C.cast(p, C.c_void_p).value


def test_device_packet_structs_carry_the_addresses():
    reads, cig, n_cig, sa, seq = _abi.device_packet(fake_packet(), 0)
    assert reads.n == 5 and [addr(getattr(reads, f)) for f in _abi.READ_FIELDS] == [0x1000 * (k + 1) for k in range(7)]
    assert addr(reads.cigar_off) == 0x10000 and addr(reads.sa_off) == 0x20000
    assert addr(cig) == 0x30000 and n_cig == 40
    assert sa.n == 3 and addr(sa.chrom) == 0x40000 and addr(sa.ref_span) == 0x40600
    assert seq.n_bytes == 30 and addr(seq.seq_off) == 0x50000 and addr(seq.seq4) == 0x60000
    assert _abi.device_packet(fake_packet(seq=False), 0)[4] is None
    assert _abi.device_packet(fake_packet(cigar=FakeDev(40, "<i4")), 0)[2] == 40   # int32 CIGAR (torch) is accepted


def test_host_packets_take_the_numpy_path():
    pk = packing.pack_alignments([], {}, {})
    assert _abi.device_packet(pk, 0) is None
    assert _abi.device_packet(dpu.with_bases(pk, []), 0) is None


def test_empty_device_packet():
    reads, cig, n_cig, sa, seq = _abi.device_packet(fake_packet(n=0, n_cigar=0, n_sa=0, n_bytes=0), 0)
    assert reads.n == 0 and n_cig == 0 and addr(cig) is None and sa.n == 0 and seq.n_bytes == 0 and addr(reads.cigar_off) == 0x10000


@pytest.mark.parametrize("field,bad", [("flag", FakeDev(5, "<i8")), ("cigar_off", FakeDev(6, "<i4")), ("cigar", FakeDev(40, "<i8")),
                                       ("seq4", FakeDev(30, "<i4")), ("seq_off", FakeDev(6, "<u8")), ("sa.mapq", FakeDev(3, "<f4"))])
def test_wrong_dtype_raises_type_error(field, bad):
    with pytest.raises(TypeError, match=field):
        _abi.device_packet(fake_packet(**{field: bad}), 0)


def test_shape_and_contiguity():
    with pytest.raises(TypeError, match="one dimension"):
        _abi.device_packet(fake_packet(cigar=FakeDev(40, "<u4", shape=(20, 2))), 0)
    with pytest.raises(TypeError, match="contiguous"):
        _abi.device_packet(fake_packet(mapq=FakeDev(5, strides=(8,))), 0)
    _abi.device_packet(fake_packet(mapq=FakeDev(5, strides=(4,))), 0)


@pytest.mark.parametrize("field,bad,msg", [("read_id", FakeDev(4), "lengths"), ("cigar_off", FakeDev(5, "<i8"), "cigar_off"),
                                           ("sa_off", FakeDev(7, "<i8"), "sa_off"), ("seq_off", FakeDev(5, "<i8"), "seq_off"),
                                           ("sa.strand", FakeDev(2), "SA column")])
def test_lengths_must_agree(field, bad, msg):
    with pytest.raises(ValueError, match=msg):
        _abi.device_packet(fake_packet(**{field: bad}), 0)


def test_mixing_host_and_device_raises():
    with pytest.raises(ValueError, match="all device or all host"):
        _abi.device_packet(fake_packet(query_len=np.zeros(5, np.int32)), 0)
    with pytest.raises(ValueError, match="all device or all host"):
        _abi.device_packet(fake_packet(seq4=np.zeros(30, np.uint8)), 0)


def test_seq_columns_go_together_and_required_columns_exist():
    pk = fake_packet()
    del pk["seq4"]
    with pytest.raises(ValueError, match="seq_off and seq4"):
        _abi.device_packet(pk, 0)
    pk = fake_packet()
    del pk["ref_end"]
    with pytest.raises(ValueError, match="ref_end"):
        _abi.device_packet(pk, 0)


def test_other_device_raises():
    with pytest.raises(ValueError, match="device 1"):
        _abi.device_packet(fake_packet(seq4=FakeDev(30, "|u1", device=1)), 0)


# ---- pack_bases ----

def test_pack_bases_round_trips_through_decode_seq():
    rng = np.random.default_rng(3)
    strings = ["", None, "A", "=ACMGRSVTWYHKDBN", "ACGTN" * 7 + "G"] + ["".join(rng.choice(list("ACGTN"), k)) for k in rng.integers(1, 300, 40)]
    seq4, seq_off = packing.pack_bases(strings)
    assert seq_off[0] == 0 and len(seq4) == seq_off[-1]
    assert (np.diff(seq_off) == [(len(s or "") + 1) // 2 for s in strings]).all()
    pk = dict(query_len=np.array([len(s or "") for s in strings], np.int32), seq_off=seq_off, seq4=seq4)
    assert [bamio.decode_seq(pk, i) for i in range(len(strings))] == [s or "" for s in strings]


# ---- the device's sequence routines, compiled for the host ----

@pytest.fixture(scope="module")
def ins_lib(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "emul_ins_seq.cpp")
    so = str(tmp_path_factory.mktemp("emul") / "libemul_ins_seq.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-fPIC", "-shared", "-o", so, src])
    L = C.CDLL(so)
    L.emul_ins_seqs.restype = C.c_int
    L.emul_fetch_offsets.restype = C.c_int64
    return L


def emul_strings(L, pk, pieces, po, pc, p, rec_base=0):
    """INS strings of rows (po, pc) over `pieces`, built by the device routines on the packet's packed bases."""
    keep = [np.ascontiguousarray(a, dtype=t) for a, t in ((pieces, np.int32), (po, np.int32), (pc, np.int32), (pk["query_len"], np.int32),
                                                          (pk["seq_off"], np.int64), (pk["seq4"], np.uint8), (pk["cigar_off"], np.int64),
                                                          (pk["cigar"], np.uint32), (pk["ref_start"], np.int32))]
    P = [a.ctypes.data_as(C.c_void_p) if a.size else None for a in keep]
    n = len(po)
    out_off = np.zeros(n + 1, np.int64)
    cap = 1 << 16
    while True:
        out = np.zeros(cap, np.uint8)
        rc = L.emul_ins_seqs(P[0], P[1], P[2], C.c_int64(n), C.c_int32(rec_base), P[3], P[4], P[5], P[6], P[7], P[8], C.c_int32(p.min_siglength),
                             C.c_int32(p.merge_ins_threshold), out.ctypes.data_as(C.c_void_p), C.c_int64(cap), out_off.ctypes.data_as(C.c_void_p))
        if rc != -3:
            break
        cap = int(out_off[n])
    assert rc == 0, rc
    o = out_off.tolist()
    whole = out[:o[-1]].tobytes().decode("ascii")
    return [whole[o[i]:o[i + 1]] for i in range(n)]


def _emulated_tuples(L, seed, n_reads, p, kind):
    reads, (gc, gr), ex = _run(seed, n_reads, p, kind)
    # the packet _run extracted (contig / read ids do not matter for bases, CIGARs and reference starts)
    pk = dpu.with_bases(packing.pack_alignments(reads, collections.defaultdict(int), collections.defaultdict(int)),
                        [r.query_sequence for r in reads])
    seqs = emul_strings(L, pk, ex["pieces"], ex["piece_off"], ex["piece_cnt"], p)
    assert [len(s) for s in seqs] == ex["sigs"]["INS"]["c"].tolist()   # every synthetic record stores its bases
    # INS tuples come out in row order: swap in the device-built strings
    gc = dict(gc, INS=[t[:3] + (s,) + t[4:] for t, s in zip(gc["INS"], seqs)])
    return gc, gr, ex


@pytest.mark.parametrize("name", EXTRACT_GOLDENS)
def test_device_routines_reproduce_reference_ins_strings(ins_lib, name):
    meta = json.load(open(os.path.join(golden_util.GOLDEN, name + ".json")))
    p = _abi.default_params(**meta["params"])
    gc, gr, ex = _emulated_tuples(ins_lib, meta["seed"], meta["n_reads"], p, meta.get("kind", "short"))
    if name in ("extract_l0", "extract_l1", "extract_l4"):
        assert (ex["pieces"][:, 3] == 2).any(), "marker pieces should be exercised"
    ref_c = {k: [tuple(t) for t in v] for k, v in meta["candidate"].items()}
    assert not compare_extract.diff_extract(ref_c, [tuple(t) for t in meta["rows"]], gc, gr)


@pytest.mark.parametrize("seed", range(500, 520))
def test_device_routines_reproduce_reference_digests(ins_lib, seed):
    meta = _seed_golden(seed)
    p = _abi.default_params(**meta["params"])
    gc, gr, _ = _emulated_tuples(ins_lib, seed, meta["n_reads"], p, "short")
    gc = dict(gc, INS=[golden_util.seq_digest(t) for t in gc["INS"]])
    ref_c = {k: [tuple(t) for t in v] for k, v in meta["candidate"].items()}
    assert not compare_extract.diff_extract(ref_c, [tuple(t) for t in meta["rows"]], gc, gr)


def test_hand_made_pieces(ins_lib):
    """Reverse-strand pieces (only ACGTN / acgtn complemented), negative and out-of-range slice bounds, a record without stored
    bases (its column c says 12 bases, the string is empty), and a marker piece rebuilt from the CIGAR."""
    q0 = "ACGTNRYKM=ACGTTGCA"                          # 18 bases, IUPAC codes kept by the complement
    q2 = "TTTTACGGGGCCCCAAAATTTTGGGGCCCCAAAAT"         # 35 bases, the CIGAR below with a hard clip in front
    queries = [q0, None, q2]
    # record 2 at 7: 5H 4M 4I 3M 4I 3M 2D 4I 9M 3D 2I 2M; min_siglength 2, merge 3: merged groups at 11 (two insertions), 19, 31
    ops = [(5, 5), (4, 0), (4, 1), (3, 0), (4, 1), (3, 0), (2, 2), (4, 1), (9, 0), (3, 2), (2, 1), (2, 0)]
    cig2 = np.array([(ln << 4) | op for ln, op in ops], np.uint32)
    pk = dict(query_len=np.array([18, 12, 35], np.int32), ref_start=np.array([0, 0, 7], np.int32),
              cigar_off=np.array([0, 0, 0, len(cig2)], np.int64), cigar=cig2)
    pk["seq4"], pk["seq_off"] = packing.pack_bases(queries)
    pieces = np.array([[0, 2, 9, 0], [0, 2, 9, 1], [0, -5, -1, 0], [0, -5, -1, 1], [0, -40, 3, 1], [0, 15, 99, 0], [0, 9, 2, 0],
                       [1, 0, 12, 0], [1, -3, 12, 1],
                       [2, 11, 0, 2], [2, 19, 0, 2], [0, 0, 4, 1]], np.int32)
    po = np.array([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 0], np.int32)
    pc = np.array([1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 3], np.int32)
    p = _abi.default_params(min_siglength=2, merge_ins_threshold=3)
    got = emul_strings(ins_lib, pk, pieces, po, pc, p)
    query_of = lambda rec: queries[rec] or ""
    cigar_of = dpu.cigar_of_packet(pk)
    want = [packing.ins_sequence(pieces, int(o), int(c), query_of, cigar_of, (2, 3)) for o, c in zip(po, pc)]
    assert got == want
    assert got[1] == packing.revcomp(q0)[2:9] and "R" in packing.revcomp(q0)
    assert got[7] == got[8] == ""                                   # no stored bases
    assert got[9] == q2[4:8] + q2[11:15] and got[10] == q2[18:22]   # merged groups of record 2
    assert got[9] == packing.merged_ins_from_cigar(cig2, 7, q2, 11, 2, 3)


def test_fetch_offsets_are_64_bit(ins_lib):
    """csv_fetch_ins_seqs may be asked for rows whose strings add up past 4 GiB (the arena spans the whole accumulation, and rows may
    repeat): the output offsets are summed in 64 bits, so none wraps and the total is the size the caller must provide."""
    big = 2 ** 31 - 1
    lens = np.array([big, 7, big, big, 0, 5], np.int32)   # the same long row asked for three times
    off = np.zeros(len(lens) + 1, np.int64)
    total = ins_lib.emul_fetch_offsets(lens.ctypes.data_as(C.c_void_p), C.c_int64(len(lens)), off.ctypes.data_as(C.c_void_p))
    want = np.concatenate([[0], np.cumsum(lens.astype(np.int64))])
    assert total == want[-1] == 3 * big + 12 and total > 2 ** 32
    assert (off == want).all()


def test_tie_rows_are_the_rows_tie_swaps_reads():
    """cli.ins_tie_rows and cli.ins_tie_swaps share one tie-group search: the strings of the rows ins_tie_rows returns are the only
    ones ins_tie_swaps reads, and with just those it makes the same swaps as with every row's string."""
    rng = np.random.default_rng(4)
    n = 400
    chrom, a = rng.integers(0, 3, n).astype(np.int32), (2 * rng.integers(0, 40, n) + rng.integers(0, 2, n)).astype(np.int32)
    b, rid = rng.integers(30, 33, n).astype(np.int32), rng.integers(0, 4, n).astype(np.int32)
    seqs = ["".join(rng.choice(list("ACGT"), 3)) for _ in range(n)]
    rows = cli.ins_tie_rows(chrom, a, b, rid)
    assert len(rows) and (np.diff(rows) > 0).all()

    class Only(dict):
        def __getitem__(self, k):
            assert k in self, "ins_tie_swaps read the string of row %d, outside ins_tie_rows" % k
            return dict.__getitem__(self, k)
    pairs = cli.ins_tie_swaps(chrom, a, b, rid, Only((int(r), seqs[r]) for r in rows))
    assert len(pairs) and pairs == cli.ins_tie_swaps(chrom, a, b, rid, seqs)
    assert set(np.ravel(pairs).tolist()) <= set(rows.tolist())
