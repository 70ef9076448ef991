"""-m gpu: the signature-phase drop-ins (cutesv_b200.cuteSV_signatures) on the CUDA library against the reference's own
single_pipe / process_process_sigs_type / run_* output (tests/golden/sigs_dropin.json.gz), and csv_sort_sigs against a numpy
statement of its order on random columns."""
import os
import sys

import numpy as np
import pytest

import sigs_dropin_data as D
from cutesv_b200 import _abi, cuteSV_resolveDUP, cuteSV_resolveINDEL, cuteSV_resolveINV, cuteSV_resolveTRA, cuteSV_signatures as S, runtime, synth
from cutesv_b200._resolve_common import clear_cache
from oracle import compare_records

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return D.load()


@pytest.fixture
def dropin(engine, monkeypatch):
    monkeypatch.setattr(runtime, "_engine", engine)
    monkeypatch.syspath_prepend(os.path.join(os.path.dirname(os.path.abspath(__file__)), "fake_pysam"))   # stands in for pysam
    monkeypatch.delitem(sys.modules, "pysam", raising=False)
    clear_cache()
    yield engine
    clear_cache()


def _tuples(lst):
    return [tuple(x) for x in lst]


def _run_single_pipe(case, g, d, monkeypatch):
    ds, tasks, bed = D.dataset(case)
    assert tasks == g["tasks"]
    os.makedirs(d + "signatures")
    D.write_fake_bam(d + "in.bam", ds)
    S.init_reading_process(d + "in.bam", None)
    proc = type("P", (), {})()
    monkeypatch.setattr(S, "current_process", lambda: proc)
    for i, task in enumerate(tasks):
        proc.pid = g["task_pid"][i]
        S.multi_run_wrapper(D.task_args(case, d, task, None if bed is None else [tuple(r) for r in bed[i]]))
        for t in D.TYPES:
            got = D.read_pid_dumps("%ssignatures/%s%s.pickle" % (d, proc.pid, t))[-1]
            assert got == _tuples(g["windows"][i][t]), (case["name"], i, t)
    S.cleanup()


@pytest.mark.parametrize("k", range(len(D.CASES)))
def test_single_pipe_matches_reference(golden, dropin, tmp_path, monkeypatch, k):
    """Every window's pid-pickle lists equal the reference's, in order (record order, parse_read's order inside a record)."""
    _run_single_pipe(D.CASES[k], golden["cases"][k], str(tmp_path) + "/", monkeypatch)


@pytest.mark.parametrize("k", range(len(D.CASES)))
def test_rebuild_on_reference_pid_pickles(golden, dropin, tmp_path, k):
    """process_process_sigs_type on the reference-written pid pickles: lists, index keys, reads_count and .sigs text."""
    g = golden["cases"][k]
    d = str(tmp_path) + "/"
    D.write_pid_pickles(d, g)
    for t in D.TYPES:
        sv, index, rc = S.process_process_sigs_type((t, d, list(D.PIDS), True))
        assert sv == t and list(index) == g["index_keys"][t]
        assert rc == (g["reads_count"][t] if t == "reads" else {})
        for chrom, rows in g["rebuilt"][t]:
            assert S.workdir.load_slice(d, t, chrom, {t: index}) == _tuples(rows), (g["name"], t, chrom)
        with open("%s/%s.sigs" % (d, t)) as f:
            assert f.read() == g["sigs_text"][t]


def _row(svtype, r):
    """A resolution row as strings; TRA's read names are ','.join(set(...)) in the reference (resolveTRA.py:182), an order that
    depends on the string hash seed, so they compare as a sorted list."""
    r = list(map(str, r))
    if svtype == "TRA":
        r[-1] = sorted(r[-1].split(","))
    return r


@pytest.mark.parametrize("k", range(len(D.CASES)))
def test_chain_to_resolution(golden, dropin, tmp_path, monkeypatch, k):
    """Drop-in single_pipe -> drop-in rebuild -> the resolution_* drop-ins give the reference's rows for the seed."""
    case, g = D.CASES[k], golden["cases"][k]
    d = str(tmp_path) + "/"
    _run_single_pipe(case, g, d, monkeypatch)
    sigs_index = {}
    for t in D.TYPES:
        sv, index, rc = S.process_process_sigs_type((t, d, list(D.PIDS), False))
        sigs_index[t] = index
        if t == "reads":
            sigs_index["reads_count"] = rc
    run = {"DEL": cuteSV_resolveINDEL.run_del, "INS": cuteSV_resolveINDEL.run_ins, "INV": cuteSV_resolveINV.run_inv,
           "DUP": cuteSV_resolveDUP.run_dup, "TRA": cuteSV_resolveTRA.run_tra}
    got = [[t, chrom, list(run[t](args))] for t, chrom, args in D.resolve_calls(d, sigs_index)]
    want = [[t, c, list(r)] for t, c, r in g["resolved"]]
    assert len(got) == len(want)
    n = 0
    for a, b in zip(got, want):
        assert a[:2] == b[:2]
        assert a[2][0] == b[2][0]
        assert [_row(a[0], r) for r in a[2][1]] == [_row(b[0], r) for r in b[2][1]], a[:2]
        n += len(b[2][1])
    assert n > 0


def _random_cols(rng, svtype, n, n_contigs, a_max, rid_max, b_max):
    chrom = rng.integers(0, n_contigs, n).astype(np.int32)
    if n_contigs > 8:   # heavy ties: few distinct values per field
        chrom = rng.choice(rng.integers(0, n_contigs, 6), n).astype(np.int32)
    a = rng.choice(rng.integers(0, a_max - 1, 5), n).astype(np.int32)
    if svtype == "INS":
        a = a + rng.integers(0, 2, n).astype(np.int32)   # x.5 and integer positions of one int(pos)
    b = rng.choice(rng.integers(0, b_max, 4), n).astype(np.int32) if b_max > 4 else rng.integers(0, 4, n).astype(np.int32)
    rid = rng.choice(rng.integers(0, rid_max, 50), n) if rid_max > (1 << 30) else rng.integers(0, rid_max, n)
    if rid_max > (1 << 30):
        rid[rng.integers(0, n, 3)] = rid_max - 1   # the widest read rank
    if b_max > 4:   # every field at its full width, so that the key really has the rounds the case is for
        chrom[0], a[0], b[1] = n_contigs - 1, a_max - 2, b_max - 1
    cols = dict(chrom=chrom, a=a, b=b, read_id=rid.astype(np.int32))
    if svtype == "INV":
        cols["c"] = rng.integers(0, 2, n).astype(np.int32)
    elif svtype == "TRA":
        cols["c"] = (rng.choice(rng.integers(0, n_contigs, 3), n) * 4 + rng.integers(0, 4, n)).astype(np.int32)
        if b_max > 4:
            cols["c"][2] = (n_contigs - 1) * 4 + 3
    elif svtype == "INS":
        cols["c"] = rng.integers(0, 100, n).astype(np.int32)
    else:
        cols["c"] = None
    return cols


def _reads_cols(rng, n, n_contigs):
    chrom = rng.integers(0, min(n_contigs, 40), n).astype(np.int32) * max(n_contigs // 40, 1)
    s = rng.integers(0, 1 << 20, n).astype(np.int32)
    return dict(chrom=chrom, start=s, end=s + 5, read_id=rng.integers(0, 50, n).astype(np.int32), is_primary=np.ones(n, np.uint8))


def _check_sort(engine, svtype, cols, n_contigs):
    want = D.np_sort_sigs(svtype, cols, n_contigs)
    got = engine.sort_sigs(svtype)
    assert np.array_equal(got["order"], want["order"]), svtype
    assert np.array_equal(got["contig_off"], want["contig_off"]), svtype
    assert np.array_equal(got["ins_tie"], want["ins_tie"]), svtype


@pytest.mark.parametrize("n,n_contigs,a_max,rid_max,b_max", [(0, 3, 10, 5, 4), (1, 3, 10, 5, 4), (5000, 3, 40, 7, 4),
                                                             (300000, 25, 1 << 30, 1 << 20, 4), (70000, 40000, 1 << 31, 3000, 4),
                                                             (70000, 40000, 1 << 31, (1 << 31) - 1, 1 << 31),
                                                             (60000, 1000000, 1 << 31, (1 << 31) - 1, 1 << 31)])
def test_sort_sigs_matches_lexsort(engine, n, n_contigs, a_max, rid_max, b_max):
    """Every type and the reads table against a stable numpy lexsort + adjacent de-duplication: empty, one row, heavy ties,
    more than 32 768 contigs with positions up to 2^31 - 1 (a linear span above 2^32), and keys of every round shape: a
    32-bit second round, a 64-bit second round (> 96 key bits: wide lengths and read ranks) and a third round (TRA on
    10^6 contigs: 20 + 22 + 3 * 31 = 135 bits)."""
    rng = np.random.default_rng(n + n_contigs + (b_max > 4))
    lens = np.full(n_contigs, (1 << 31) - 1, np.int64)
    engine.set_contigs(lens)
    assert int(lens.sum()) > (1 << 32)
    for svtype in _abi.TYPE_NAMES:
        cols = _random_cols(rng, svtype, n, n_contigs, a_max, rid_max, b_max)
        engine.upload({svtype: cols}, None)
        _check_sort(engine, svtype, cols, n_contigs)
    reads = _reads_cols(rng, n, n_contigs)
    engine.upload({}, reads)
    _check_sort(engine, "reads", reads, n_contigs)


def test_sort_sigs_all_duplicates(engine):
    engine.set_contigs(np.full(4, 1000, np.int64))
    for svtype in ("DEL", "DUP", "INV", "TRA"):
        n = 4097
        cols = dict(chrom=np.full(n, 2, np.int32), a=np.full(n, 7, np.int32), b=np.full(n, 9, np.int32), read_id=np.full(n, 3, np.int32),
                    c=None if svtype in ("DEL", "DUP") else np.full(n, 1, np.int32))
        engine.upload({svtype: cols}, None)
        got = engine.sort_sigs(svtype)
        assert got["order"].tolist() == [0] and got["contig_off"].tolist() == [0, 0, 0, 1, 1]
    cols = dict(chrom=np.zeros(3, np.int32), a=np.array([20, 21, 20], np.int32), b=np.ones(3, np.int32), read_id=np.ones(3, np.int32),
                c=np.ones(3, np.int32))
    engine.upload({"INS": cols}, None)
    got = engine.sort_sigs("INS")
    assert got["order"].tolist() == [0, 1, 2] and got["ins_tie"].tolist() == [0, 1, 1]


def test_sort_sigs_rejects_bad_input(engine):
    engine.set_contigs(np.full(2, 1000, np.int64))
    engine.upload({"DEL": dict(chrom=np.array([0, 2], np.int32), a=np.zeros(2, np.int32), b=np.zeros(2, np.int32),
                               read_id=np.zeros(2, np.int32), c=None)}, None)
    with pytest.raises(Exception) as e:
        engine.sort_sigs("DEL")
    assert e.value.code == _abi.CSV_E_INPUT


def test_sort_sigs_leaves_cluster_results_alone(engine):
    """csv_cluster -> csv_sort_sigs (every type and the reads table) -> csv_fetch returns what csv_cluster -> csv_fetch returns,
    and a following csv_cluster gives the same records."""
    cfg = synth.make_config(3, 0.02)
    engine.set_params(_abi.default_params(**cfg["params"]))
    engine.set_contigs(cfg["lens"])
    engine.upload(cfg["sigs"], cfg["reads"])
    engine.cluster_device(0x1F)
    ref = engine.fetch()
    engine.upload(cfg["sigs"], cfg["reads"])
    engine.cluster_device(0x1F)
    for t in list(_abi.TYPE_NAMES) + ["reads"]:
        engine.sort_sigs(t)
    got = engine.fetch()
    assert not compare_records.diff_records(ref, got)
    engine.cluster_device(0x1F)
    assert not compare_records.diff_records(ref, engine.fetch())
    assert len(ref[0]) > 0


def test_records_follow_extraction(engine):
    """csv_fetch_records: with csv_extract_records on, every extracted row carries its record; without it, or after an upload
    since the extraction, there is no column to fetch.  The extracted rows themselves do not depend on the switch."""
    reads, names, lens = synth.synth_alignments(4, 200)
    rn = sorted({r.query_name for r in reads})
    pk = S.packing.pack_alignments(reads, {n: i for i, n in enumerate(names)}, {n: i for i, n in enumerate(rn)})
    engine.set_params(_abi.default_params(min_mapq=0, min_read_len=100))
    engine.set_contigs(lens)
    engine.extract(pk)
    plain = engine.fetch_extracted()
    with pytest.raises(Exception) as e:
        engine.fetch_records("DEL", 0, 0)
    assert e.value.code == _abi.CSV_E_STATE
    engine.set_extract_records(True)
    try:
        engine.extract(pk)
    finally:
        engine.set_extract_records(False)
    got = engine.fetch_extracted()
    for t in _abi.TYPE_NAMES:
        assert sorted(zip(*[got["sigs"][t][k].tolist() for k in ("chrom", "a", "b", "read_id")])) == \
            sorted(zip(*[plain["sigs"][t][k].tolist() for k in ("chrom", "a", "b", "read_id")]))
    rows = engine.fetch_extracted()["rows"]
    rec = engine.fetch_records("reads")
    assert np.array_equal(rows["read_id"], pk["read_id"][rec]) and np.array_equal(rows["start"], pk["ref_start"][rec])
    for t in _abi.TYPE_NAMES:
        r = engine.fetch_records(t)
        assert np.array_equal(engine.fetch_extracted()["sigs"][t]["read_id"], pk["read_id"][r])
    engine.upload({}, None)
    with pytest.raises(Exception) as e:
        engine.fetch_records("DEL", 0, 0)
    assert e.value.code == _abi.CSV_E_STATE
