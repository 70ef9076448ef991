"""-m gpu: k_extract on the planted edge layouts of tests/extract_edges.py (tiles, lanes, items, chunks, d0, the ring, the lazy
offsets, the hand-over, the 64-piece INS buffer) through every packet route: host packets, device packets with bases (INS
strings built on the device), packets appended at cuts beside a planted record, and named device packets.  Each result is
compared three ways: with the emulator row by row in emission order within every record, with the reference's golden, and
with the builder's literals.  Then the ring parity across many records per warp, and the output-capacity reruns."""
import collections

import numpy as np
import pytest

import device_packet_util as dpu
import emul_lib
import extract_edges as E
import name_util
from cutesv_b200 import _abi, packing
from cutesv_b200.engine import Engine
from oracle import compare_extract
from test_extract_edges_cpu import golden

pytestmark = pytest.mark.gpu
TYPES = _abi.TYPE_NAMES


# ---------------------------------------------------------------------------------------------------------------------
# comparisons
# ---------------------------------------------------------------------------------------------------------------------
def per_record(ex, seqs=None):
    """{(type, read id): [row, ...]} in slot order, which within one record and type is parse_read's emission order.  An INS row
    carries its piece list, or its string when `seqs` (by INS row) is given."""
    out = {}
    for t in TYPES:
        s = ex["sigs"][t]
        for i in range(len(s["chrom"])):
            row = (int(s["chrom"][i]), int(s["a"][i]), int(s["b"][i]), int(s["c"][i]) if t in ("INS", "INV", "TRA") else 0)
            if t == "INS":
                po, pc = int(ex["piece_off"][i]), int(ex["piece_cnt"][i])
                row += (seqs[i] if seqs is not None else tuple(map(tuple, ex["pieces"][po:po + pc].tolist())),)
            out.setdefault((t, int(s["read_id"][i])), []).append(row)
    r = ex["rows"]
    out["rows"] = collections.Counter(zip(r["chrom"].tolist(), r["start"].tolist(), r["end"].tolist(), r["read_id"].tolist(), r["is_primary"].tolist()))
    return out


def check_records(engine, ex):
    """The record column (csv_fetch_records) names every row's record; the builders give record k the read id k."""
    for t in TYPES:
        assert np.array_equal(engine.fetch_records(t), ex["sigs"][t]["read_id"]), t
    assert np.array_equal(engine.fetch_records("reads"), ex["rows"]["read_id"])


def tuples(c, ex, p, seqs=None):
    """The reference's tuple shapes; INS strings from the piece table (host) or the device arena (`seqs`, by INS row)."""
    gc, gr = compare_extract.tuples_from_columns(ex, c["names"], c["rnames"], lambda rec: c["reads"][rec].query_sequence,
                                                 dpu.cigar_of_packet(c["pk"]), (p.min_siglength, p.merge_ins_threshold))
    if seqs is not None:
        assert [len(x) for x in seqs] == ex["sigs"]["INS"]["c"].tolist()
        gc = dict(gc, INS=[t[:3] + (s,) + t[4:] for t, s in zip(gc["INS"], seqs)])
    return gc, gr


def three_ways(c, pname, ex, seqs=None):
    """ex equals the emulator row by row within each record, the reference's golden, and the planted literals."""
    p = E.params(pname)
    ref = emul_lib.extract(p, c["pk"])
    assert per_record(ex) == per_record(ref)
    gc, gr = tuples(c, ex, p, seqs)
    cand, rows = golden(c["name"], pname)
    assert not compare_extract.diff_extract(cand, rows, gc, gr)
    assert E.ordered(gc) == E.ordered(cand)
    assert E.ordered(gc) == E.expected_ordered(c, pname)
    assert sorted(gr) == sorted(E.expected_rows(c, pname))


def dev_strings(engine):
    return engine.fetch_ins_seqs(np.arange(engine._ex_counts[_abi.CSV_INS]))


def queries(c):
    return [r.query_sequence for r in c["reads"]]


@pytest.fixture
def rec_engine(engine):
    engine.set_extract_records(True)
    yield engine
    engine.set_extract_records(False)


def _setup(engine, c, pname):
    engine.set_params(E.params(pname))
    engine.set_contigs(c["lens"])


# ---------------------------------------------------------------------------------------------------------------------
# the routes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pname", list(E.PARAMS))
@pytest.mark.parametrize("name", E.CASES)
def test_host_packet(rec_engine, name, pname):
    c = E.case(name)
    _setup(rec_engine, c, pname)
    rec_engine.extract(c["pk"])
    ex = rec_engine.fetch_extracted()
    check_records(rec_engine, ex)
    three_ways(c, pname, ex)


@pytest.mark.parametrize("pname", list(E.PARAMS))
@pytest.mark.parametrize("name", E.CASES)
def test_device_packet_with_bases(engine, name, pname):
    """INS strings from the device arena: the marker walk (k_ins_len / k_ins_fill) runs on the 65- and 66-insertion chains."""
    c = E.case(name)
    _setup(engine, c, pname)
    engine.extract(dpu.to_device(dpu.with_bases(c["pk"], queries(c))))
    three_ways(c, pname, engine.fetch_extracted(), dev_strings(engine))


def _slice(pk, lo, hi):
    out = {k: pk[k][lo:hi] for k in _abi.READ_FIELDS}
    keys = ["cigar_off", "sa_off"] + (["seq_off"] if "seq_off" in pk else [])
    b = {k: (int(pk[k][lo]), int(pk[k][hi])) for k in keys}
    for k in keys:
        out[k] = pk[k][lo:hi + 1] - b[k][0]
    out["cigar"] = pk["cigar"][b["cigar_off"][0]:b["cigar_off"][1]]
    if "seq_off" in pk:
        out["seq4"] = pk["seq4"][b["seq_off"][0]:b["seq_off"][1]]
    out["sa"] = {k: v[b["sa_off"][0]:b["sa_off"][1]] for k, v in pk["sa"].items()}
    return out


def _cut_records(c):
    """The planted record with the most ops and the last planted record: cuts fall just before and just after each."""
    planted = [x for x in c["records"] if x["label"]]
    return sorted({max(planted, key=lambda x: x["n_ops"])["rec"], planted[-1]["rec"]})


@pytest.mark.parametrize("route", ["host", "device"])
@pytest.mark.parametrize("name", E.CASES)
def test_append_at_cuts_beside_planted_records(engine, name, route):
    """Packets cut just before and just after planted records (which moves the d0 of every later record) give the one-call
    result record by record, INS strings included."""
    c = E.case(name)
    pname = "defaults" if name != "merges" else "merge"
    _setup(engine, c, pname)
    pk = dpu.with_bases(c["pk"], queries(c)) if route == "device" else c["pk"]
    wrap = dpu.to_device if route == "device" else (lambda x: x)
    engine.extract(wrap(pk))
    one = engine.fetch_extracted()
    one_seqs = dev_strings(engine) if route == "device" else None
    n = len(c["reads"])
    cuts = sorted({0, n} | {k for r in _cut_records(c) for k in (r, r + 1)})
    engine.extract_reset()
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        engine.extract(wrap(_slice(pk, lo, hi)), append=True)
    many = engine.fetch_extracted()
    if route == "device":
        assert per_record(many, dev_strings(engine)) == per_record(one, one_seqs)
        three_ways(c, pname, many, dev_strings(engine))
    else:
        three_ways(c, pname, many)
    assert per_record(many) == per_record(one)


@pytest.mark.parametrize("pname", ["defaults", "zero"])
@pytest.mark.parametrize("name", E.CASES)
def test_named_device_packet(engine, name, pname):
    c = E.case(name)
    _setup(engine, c, pname)
    engine.extract(name_util.named(dpu.to_device(dpu.with_bases(c["pk"], queries(c))), c["rnames"]))
    assert engine.rank_names() == len(c["rnames"])   # names sort in record order: ranks are the host packets' read ids
    ex = engine.fetch_extracted()
    three_ways(c, pname, ex, dev_strings(engine))


@pytest.mark.parametrize("route", ["host", "device"])
def test_piece_table_at_the_open_piece_limit(engine, route):
    """64 merged insertions fill the open-piece buffer: 64 pieces, no marker; 65 and 66 become one marker piece (rc 2) whose
    string the host (packing.merged_ins_from_cigar) or the device (ins_marker) rebuilds from the record's CIGAR."""
    c = E.case("merges")
    _setup(engine, c, "defaults")
    pk = c["pk"] if route == "host" else dpu.to_device(dpu.with_bases(c["pk"], queries(c)))
    engine.extract(pk)
    ex = engine.fetch_extracted()
    s = ex["sigs"]["INS"]
    want = E.expected(c, "defaults")
    by_label = {x["label"]: x["rec"] for x in c["records"] if x["label"]}
    seqs = dev_strings(engine) if route == "device" else None
    for k in E.CHAINS:
        rec = by_label["ins_chain_%d" % k]
        rows = np.flatnonzero(s["read_id"] == rec)
        assert len(rows) == 1
        i = int(rows[0])
        po, pc = int(ex["piece_off"][i]), int(ex["piece_cnt"][i])
        pieces = ex["pieces"][po:po + pc]
        if k <= E.MAX_OPEN_PIECES:
            assert pc == k and (pieces[:, 3] == 0).all() and (pieces[:, 0] == rec).all()
        else:
            assert pc == 1 and pieces[0].tolist() == [rec, int(s["a"][i]) // 2, 0, 2]
        (pos, ln, seq, n_ins), = want[rec][1]
        assert (int(s["a"][i]), int(s["b"][i]), int(s["c"][i]), n_ins) == (2 * pos, ln, len(seq), k)
        if seqs is not None:
            assert seqs[i] == seq


# ---------------------------------------------------------------------------------------------------------------------
# the ring parity across records
# ---------------------------------------------------------------------------------------------------------------------
def _rows_in_record_order(ex, rec=None):
    """Every type's columns, and the INS rows' pieces, with the rows put in record order (stable: slot order within a record)."""
    out = {}
    for t in TYPES:
        s = ex["sigs"][t]
        o = np.argsort(s["read_id"] if rec is None else rec[t], kind="stable")
        cols = [s[k][o] for k in ("chrom", "a", "b", "read_id")] + ([s["c"][o]] if t in ("INS", "INV", "TRA") else [])
        out[t] = np.stack(cols) if len(o) else np.zeros((len(cols), 0), np.int32)
        if t == "INS":
            po, pc = ex["piece_off"][o].astype(np.int64), ex["piece_cnt"][o].astype(np.int64)
            first = np.repeat(po - (np.cumsum(pc) - pc), pc)
            out["pieces"] = ex["pieces"][first + np.arange(int(pc.sum()))]
            out["piece_cnt"] = pc
    return out


def _emulated_in_record_order(p, pk, step=2048):
    """_rows_in_record_order of the emulator, run on slices of `step` records (its output buffers scale with the CIGAR length)."""
    parts = []
    n = len(pk["chrom"])
    for lo in range(0, n, step):
        r = _rows_in_record_order(emul_lib.extract(p, _slice(pk, lo, min(lo + step, n))))
        r["pieces"][:, 0] += lo   # record indices of the whole packet
        parts.append(r)
    return {k: np.concatenate([x[k] for x in parts], axis=-1 if k in TYPES else 0) for k in parts[0]}


def test_ring_parity_across_records(rec_engine):
    """32 768 records of 257-2049 ops (1 to 5 chunks: the ring's slots change parity an odd or even number of times per
    record) on 132 SMs x 24 resident warps: every warp walks several records, carrying its mbarrier phase from one to the
    next.  Row by row against the emulator, in emission order within every record."""
    pk = E.parity_packet()
    L = np.diff(pk["cigar_off"])
    chunks = (L + E.EX_CHUNK - 1) // E.EX_CHUNK
    assert set(chunks.tolist()) == {1, 2, 3, 4, 5}
    p = _abi.default_params()
    rec_engine.set_params(p)
    rec_engine.set_contigs([E.CONTIG_LEN])
    rec_engine.extract(pk)
    ex = rec_engine.fetch_extracted()
    rec = {t: rec_engine.fetch_records(t) for t in TYPES}
    for t in TYPES:
        assert np.array_equal(rec[t], ex["sigs"][t]["read_id"]), t
    got, ref = _rows_in_record_order(ex, rec), _emulated_in_record_order(p, pk)
    assert got["DEL"].shape[1] > 50_000 and got["INS"].shape[1] > 50_000
    for k in ref:
        assert np.array_equal(got[k], ref[k]), k
    assert len(ex["rows"]["chrom"]) == len(L)


# ---------------------------------------------------------------------------------------------------------------------
# output-capacity reruns
# ---------------------------------------------------------------------------------------------------------------------
N_RERUN = 64   # first guesses: DEL / INS rows 4n + 1024 = 1280, pieces 8n + 2048 = 2560


def _profiled_engine(lens):
    eng = Engine(0, contig_lens=lens)
    eng.set_profiling(True)
    return eng


def _launches(eng):
    return eng.kernel_times()["k_extract"][0]


@pytest.mark.parametrize("dels,ins,pieces,launches", [
    (1280, 0, 1, 1), (1281, 0, 1, 2),          # DEL rows at and one past the first guess
    (0, 1281, 1, 2), (0, 2560, 1, 2),          # INS rows past it, their pieces within the first piece guess
    (0, 2561, 1, 3),                           # the INS rows that found no slot reserved no pieces: the second run overflows them
    (0, 1000, 3, 2),                           # 3000 pieces of 1000 rows
])
def test_rerun_launches(engine, dels, ins, pieces, launches):
    """A fresh context per case (the densest packet so far raises later first guesses for the context's lifetime)."""
    reads, names, pk = E.rerun_packet(N_RERUN, dels, ins, pieces)
    eng = _profiled_engine([E.CONTIG_LEN])
    try:
        eng.set_extract_records(True)
        eng.extract(pk)
        assert _launches(eng) == launches
        ex = eng.fetch_extracted()
        check_records(eng, ex)
        assert len(ex["sigs"]["DEL"]["chrom"]) == dels and len(ex["sigs"]["INS"]["chrom"]) == ins and len(ex["pieces"]) == ins * pieces
        assert per_record(ex) == per_record(emul_lib.extract(_abi.default_params(), pk))
    finally:
        eng.close()


def _append_packets():
    """A sparse packet, a dense one past the first guess (its rerun must keep the sparse packet's rows), a sparse one."""
    out, rec0 = [], 0
    for dels, ins in ((64, 64), (1500, 1400), (64, 64)):
        reads, names, pk = E.rerun_packet(N_RERUN, dels, ins, 1, seed=rec0, rec0=rec0)
        out.append((reads, names, pk))
        rec0 += N_RERUN
    return out


@pytest.mark.parametrize("route", ["host", "named_device"])
def test_rerun_in_append_mode_keeps_earlier_rows(engine, route):
    parts = _append_packets()
    reads = [r for x in parts for r in x[0]]
    names = [nm for x in parts for nm in x[1]]
    whole = packing.pack_alignments(reads, {E.CONTIG: 0}, {nm: i for i, nm in enumerate(names)})

    def wrap(pk, nm, rs):
        return pk if route == "host" else name_util.named(dpu.to_device(dpu.with_bases(pk, [r.query_sequence for r in rs])), nm)

    results = []
    for append_mode in (True, False):
        eng = _profiled_engine([E.CONTIG_LEN])
        try:
            eng.set_extract_records(route == "host")
            if append_mode:
                runs = []
                for rs, nm, pk in parts:
                    eng.extract(wrap(pk, nm, rs), append=True)
                    runs.append(_launches(eng))
                assert runs == [1, 2, 1]
            else:
                eng.extract(wrap(whole, names, reads))
            seqs = None
            if route == "named_device":
                assert eng.rank_names() == len(names)
            ex = eng.fetch_extracted()
            if route == "host":
                check_records(eng, ex)
            else:
                seqs = dev_strings(eng)
                ranks = sorted(set(ex["sigs"]["DEL"]["read_id"].tolist()) | set(ex["rows"]["read_id"].tolist()))
                assert eng.fetch_names(ranks) == [names[k] for k in ranks]
            results.append((per_record(ex), per_record(ex, seqs) if seqs is not None else None, ex))
        finally:
            eng.close()
    (app, app_s, app_ex), (one, one_s, one_ex) = results
    assert app == one == per_record(emul_lib.extract(_abi.default_params(), whole))
    assert app_s == one_s
    assert len(app_ex["sigs"]["DEL"]["chrom"]) == 1628 and len(app_ex["sigs"]["INS"]["chrom"]) == 1528
    if route == "named_device":
        want = {}
        for i, r in enumerate(reads):
            for s in E.walk(r.cigartuples, r.reference_start, r.query_sequence):
                if s["kind"] == "INS":
                    want.setdefault(i, []).append(s["seq"])
        got = {k[1]: [row[4] for row in v] for k, v in app_s.items() if k != "rows" and k[0] == "INS"}
        assert got == want
