"""-m gpu: the state rules of an extraction accumulation.  Every (state, call) pair: the states an accumulation can be in (fresh
engine, open plain / named / named and ranked / scanned / scanned-with-alignments accumulation, an upload after an open named
accumulation, a reset) against the seven extraction entry points and the calls that read the accumulation.  Each case pins
the return code, the message and what happened to the library's row counts: unchanged, replaced by the packet's, or the
packet's appended."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import device_packet_util as dpu
import golden_util
import name_util
from cutesv_b200 import _abi, _lib
from cutesv_b200.engine import Engine
from test_gpu_device_extract import _host, _packet

pytestmark = pytest.mark.gpu

RANKED = "the accumulation's names were ranked: csv_extract_reset (or a fresh extraction) starts a new one"
WITHOUT_NAMES = "a packet without names cannot join an accumulation of named packets"
WITH_NAMES = "a named packet cannot join an accumulation of packets without names"
ONLY_SCANNED = "only scanned packets (csv_scan_append_named_device) can join a scanned accumulation"
NOT_SCANNED = "a scanned packet cannot join an accumulation of extracted packets"
ALN = "every packet of a scanned accumulation asks for alignment rows, or none does"
REGIONS = "a scanned accumulation is open: the region table may change after csv_rank_names or csv_extract_reset"
NO_NAMES = "no read names: the device-resident rows do not come from csv_extract*_named_device calls"
NO_NAME_TABLE = "no name table: csv_rank_names has not ranked a named accumulation"
NO_ARENA = "no INS sequence arena: the device-resident rows do not come from csv_extract*_device calls that all carried bases"
NOT_RANKS = "the read ids are not ranks yet: call csv_rank_names first"

STATES = ("fresh", "plain", "named", "ranked", "scanned", "scanned_aln", "uploaded", "reset")
OPEN = {"plain": "plain", "named": "named", "ranked": "named", "scanned": "scanned", "scanned_aln": "scanned_aln", "uploaded": "plain"}
WITH_ARENA = ("plain", "named", "ranked", "scanned", "scanned_aln")
# extraction calls: (packet kind, append)
EXTRACT = {"extract": ("host", False), "extract_append": ("host", True), "extract_device": ("plain", False),
           "extract_append_device": ("plain", True), "extract_named_device": ("named", False),
           "extract_append_named_device": ("named", True), "scan": ("scanned", True), "scan_alignments": ("scanned_aln", True)}
CALLS = tuple(EXTRACT) + ("set_scan_regions", "rank_names", "order_ins_ties", "fetch_names", "fetch_ins_seqs")


def _expect(state, call):
    """(message of the CSV_E_STATE error or None, counts after the call: "same", "fresh" or "append")."""
    if call in EXTRACT:
        kind, append = EXTRACT[call]
        if not append or state not in OPEN:
            return None, "fresh"
        if state == "ranked":
            return RANKED, "same"
        have, kind = OPEN[state], "plain" if kind == "host" else kind
        named, scanned = have != "plain", have.startswith("scanned")
        if have == kind:
            return None, "append"
        if named != (kind != "plain"):
            return (WITHOUT_NAMES if named else WITH_NAMES), "same"
        if scanned != kind.startswith("scanned"):
            return (ONLY_SCANNED if scanned else NOT_SCANNED), "same"
        return ALN, "same"
    if call == "set_scan_regions":
        return (REGIONS if state in ("scanned", "scanned_aln") else None), "same"
    if call == "rank_names":
        return (None if state in ("named", "ranked", "scanned", "scanned_aln") else NO_NAMES), "same"
    if call == "fetch_names":
        return (None if state == "ranked" else NO_NAME_TABLE), "same"
    if call == "fetch_ins_seqs":
        return (None if state in WITH_ARENA else NO_ARENA), "same"
    assert call == "order_ins_ties"
    if state not in WITH_ARENA:
        return NO_ARENA, "same"
    return (NOT_RANKS if state in ("named", "scanned", "scanned_aln") else None), "same"


def _take(pk, idx):
    """The packet of records idx, in that order."""
    out = {k: pk[k][idx] for k in _abi.READ_FIELDS}

    def gather(off_key, cols):
        lo, hi = pk[off_key][idx].astype(np.int64), pk[off_key][idx + 1].astype(np.int64)
        off = np.zeros(len(idx) + 1, dtype=np.int64)
        np.cumsum(hi - lo, out=off[1:])
        sel = np.concatenate([np.arange(a, b) for a, b in zip(lo.tolist(), hi.tolist())] + [np.zeros(0, np.int64)])
        return off, [c[sel] for c in cols]
    out["cigar_off"], (out["cigar"],) = gather("cigar_off", [pk["cigar"]])
    out["seq_off"], (out["seq4"],) = gather("seq_off", [pk["seq4"]])
    keys = sorted(pk["sa"])
    out["sa_off"], sa = gather("sa_off", [pk["sa"][k] for k in keys])
    out["sa"] = dict(zip(keys, sa))
    return out


@pytest.fixture(scope="module")
def packets(engine):
    """(params, contig lengths, first packet, second packet, record names of each): an extraction golden's records in BAM order."""
    meta = json.load(open(os.path.join(golden_util.GOLDEN, "extract_s0.json")))
    reads, names, lens, rnames, pk = _packet(meta["seed"], meta["n_reads"])
    order = np.lexsort((pk["ref_start"], pk["chrom"]))
    pk = _take(pk, order)
    rec_names = [rnames[i] for i in pk["read_id"].tolist()]
    cut = len(order) * 3 // 5
    p1, p2 = _take(pk, np.arange(cut)), _take(pk, np.arange(cut, len(order)))
    return _abi.default_params(**meta["params"]), lens, p1, p2, rec_names[:cut], rec_names[cut:]


@pytest.fixture(autouse=True)
def _nothing_left(engine):
    yield
    engine.extract_reset()
    engine.set_scan_regions([], None, {})
    engine.upload_alignments(None)


def _counts(e):
    """The library's row counts: signatures per type, reads rows, INS pieces.  A capacity of -1 makes the size probes report
    what they need."""
    def need(rc):
        assert rc == _abi.CSV_E_CAPACITY
        return int(e.L.csv_last_error().decode().rsplit(" ", 1)[1])
    out = [need(e.L.csv_fetch_sigs(e.h, t, C.c_int64(-1), None, None, None, None, None, None, None)) for t in range(_abi.CSV_NTYPES)]
    out.append(need(e.L.csv_fetch_read_rows(e.h, C.c_int64(-1), None, None, None, None, None)))
    npz = C.c_int64(0)
    _lib.check(e.L.csv_fetch_pieces(e.h, C.c_int64(0), None, C.byref(npz)))
    return np.array(out + [npz.value], dtype=np.int64)


def _call(e, call, pk, names):
    if call in EXTRACT:
        kind, append = EXTRACT[call]
        if kind == "host":
            return e.extract(_host(pk), append=append)
        dev = dpu.to_device(pk)
        if kind == "plain":
            return e.extract(dev, append=append)
        dev = name_util.named(dev, names)
        if kind == "named":
            return e.extract(dev, append=append)
        return e.scan(dev, alignments=kind == "scanned_aln")
    if call == "set_scan_regions":
        return e.set_scan_regions([], None, {})
    if call == "fetch_names":
        return e.fetch_names([0])
    if call == "fetch_ins_seqs":
        return e.fetch_ins_seqs([0])
    return getattr(e, call)()


def _enter(e, state, pk, names):
    """Brings e (for "fresh": a new engine) into `state` with packet pk."""
    if state == "fresh":
        return
    e.extract_reset()
    if state in ("plain", "named", "scanned", "scanned_aln"):
        _call(e, {"plain": "extract_append_device", "named": "extract_append_named_device", "scanned": "scan",
                  "scanned_aln": "scan_alignments"}[state], pk, names)
    elif state in ("ranked", "uploaded", "reset"):
        _call(e, "extract_append_named_device", pk, names)
        if state == "ranked":
            e.rank_names()
        elif state == "uploaded":
            i = np.arange(3, dtype=np.int32)
            e.upload({"DEL": dict(chrom=i * 0, a=i * 10, b=i * 10 + 60, read_id=i)},
                     dict(chrom=i * 0, start=i * 10, end=i * 10 + 500, read_id=i, is_primary=np.ones(3, np.uint8)))
        else:
            e.extract_reset()


@pytest.mark.parametrize("call", CALLS)
@pytest.mark.parametrize("state", STATES)
def test_state_call(engine, packets, state, call):
    params, lens, p1, p2, n1, n2 = packets
    engine.set_params(params)
    engine.set_contigs(lens)
    alone = None
    if call in EXTRACT:   # the packet's own counts: the call on an empty accumulation
        _enter(engine, "reset", p1, n1)
        _call(engine, call, p2, n2)
        alone = _counts(engine)
    e = Engine(0, params=params, contig_lens=lens) if state == "fresh" else engine
    try:
        _enter(e, state, p1, n1)
        before = _counts(e)
        msg, counts = _expect(state, call)
        if msg is None:
            _call(e, call, p2, n2)
        else:
            with pytest.raises(_lib.CuteSVError) as err:
                _call(e, call, p2, n2)
            assert err.value.code == _abi.CSV_E_STATE
            assert str(err.value) == "cutesv_b200 error %d: %s" % (_abi.CSV_E_STATE, msg)
        after = _counts(e)
        want = before if counts == "same" else alone if counts == "fresh" else before + alone
        assert np.array_equal(after, want), (before, after, alone)
    finally:
        if e is not engine:
            e.close()


def test_packets_tell_fresh_from_append(engine, packets):
    """The second packet yields rows, INS rows with sequences and pieces, and counts unlike the first's, so that every count
    check above can tell a replaced accumulation from an appended one."""
    params, lens, p1, p2, n1, n2 = packets
    engine.set_params(params)
    engine.set_contigs(lens)
    got = []
    for pk, names in ((p1, n1), (p2, n2)):
        engine.extract_reset()
        engine.scan(name_util.named(dpu.to_device(pk), names))
        scanned = _counts(engine)
        engine.extract(dpu.to_device(pk))
        got.append(_counts(engine))
        assert np.all(scanned[[_abi.CSV_INS, _abi.CSV_NTYPES]] > 0)
    assert np.all(got[0][[_abi.CSV_INS, _abi.CSV_NTYPES, _abi.CSV_NTYPES + 1]] > 0)
    assert not np.array_equal(got[0], got[1])
