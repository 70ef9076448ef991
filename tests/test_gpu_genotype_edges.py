"""-m gpu: csv_cluster's genotype pass (k_permute -> k_scan_excl<4> -> k_windows<1> -> k_reads_pass -> k_pairs_test ->
k_finalize) on the planted layouts of tests/genotype_edges.py.  Every case is checked against three references: the oracle's
records, the numpy statement of the rule with cal_GL from the oracle, and the standalone call_gt (pinned to the reference by
its goldens) on the candidates' windows; and against the DR it plants.  Also: both pair routes, the inline path past the pair
buffer's capacity, graph replays with alternating reads tables, rows that end before they start, and the TRA genotyper's
warp-cooperative count_coverage at its step edges."""
import numpy as np
import pytest

import genotype_edges as ge
from cutesv_b200 import _abi
from cutesv_b200._lib import CuteSVError
from cutesv_b200.engine import Engine
from oracle import compare_records, oracle_lib

pytestmark = pytest.mark.gpu

CASES = {c.name: c for c in ge.all_cases()}


def cluster_fn(eng):
    def fn(p, lens, sigs, reads):
        eng.set_params(p)
        eng.set_contigs(lens)
        return eng.cluster(sigs, reads)
    return fn


def check(eng, case, reads, got):
    ref = oracle_lib.cluster(case.params, case.lens, case.sigs, reads)
    d = compare_records.diff_records(ref, got)
    assert not d, "\n".join(d[:5])
    cands, genos, names = got
    want, no_reads = ge.rule_genos(cands, names, reads, case.params, oracle_lib.cal_gl)
    windowed = ge.n_windows(cands) > 0
    d = ge.diff_genos(want[windowed], genos[windowed])
    assert not d, "\n".join(d)
    assert np.array_equal((cands["flags"] & _abi.CSV_F_NO_READS) != 0, no_reads)
    dr = ge.dr_by_contig(cands, genos)
    for c, n in case.planted.items():
        assert dr[c] == (-1 if n == -2 else n), (c, dr[c], n)
    # the standalone call_gt on the same windows
    win = ge.windows_of_candidates(cands, case.params)
    checked = 0
    for per, types in ((1, (_abi.CSV_DEL, _abi.CSV_INS)), (2, (_abi.CSV_DUP, _abi.CSV_INV))):
        sel = np.flatnonzero(np.isin(cands["svtype"], types) & (genos["status"] == 0))
        if not len(sel):
            continue
        off = np.zeros(len(sel) + 1, np.int64)
        np.cumsum(cands["names_cnt"][sel], out=off[1:])
        ids = np.concatenate([ge.supporters(cands, names, i) for i in sel]).astype(np.int32)
        g = eng.call_gt(win[sel][:, :per].reshape(-1), per, off, ids, reads)
        for k in ("dr", "dv", "gt", "pl", "gq", "qual"):
            assert np.array_equal(g[k], genos[sel][k]), (per, k)
        checked += len(sel)
    assert checked > 0


def run(eng, case):
    reads = ge.build(case, cluster_fn(eng))
    got = eng.cluster(case.sigs, reads)
    return reads, got


def route_names(eng):
    return {n for n in eng.kernel_times() if "k_reads_pass" in n or "k_pairs_test" in n}


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_matches_three_references(engine, name):
    case = CASES[name]
    engine.set_profiling(True)
    try:
        reads, got = run(engine, case)
        names = route_names(engine)   # (before call_gt replaces the collected intervals)
        check(engine, case, reads, got)
    finally:
        engine.set_profiling(False)
    lin32 = case.lay()["lin32"]
    want = "<true>" if lin32 else "<false>"
    assert names and all(want in n for n in names), names


@pytest.mark.parametrize("n_reads", ge.TILE_SIZES)
def test_tiles(engine, n_reads):
    case = ge.tiles(n_reads)
    reads, got = run(engine, case)
    assert len(reads["chrom"]) == n_reads
    check(engine, case, reads, got)


@pytest.mark.parametrize("name", ["window_bounds", "lin64_bottom"])
def test_pair_buffer_capacity(engine, monkeypatch, name):
    """The same DR whatever the pair buffer holds: every pair inline (cap 1), a CTA's reservation straddling the cap
    (P // 2 + 1), one pair inline (P - 1), none (P, P + 1)."""
    case = CASES[name]
    reads, got = run(engine, case)
    check(engine, case, reads, got)
    pairs = engine.counters()["pairs"]
    assert pairs > 8
    for cap in (1, pairs // 2 + 1, pairs - 1, pairs, pairs + 1):
        monkeypatch.setenv("CUTESV_B200_PAIR_CAP", str(cap))
        eng = Engine(0, params=case.params, contig_lens=case.lens)
        try:
            g = eng.cluster(case.sigs, reads)
            assert eng.counters()["pairs"] == pairs
        finally:
            eng.close()
        assert np.array_equal(g[1]["dr"], got[1]["dr"]), cap
        d = compare_records.diff_records(got, g)
        assert not d, (cap, d[:3])


def test_graph_replays_alternating_reads(engine):
    """Two reads tables of the same size, resident on the device, alternated over five calls: the second call captures a
    graph and the later ones replay it; each result is its own table's answer (no bins, bit map or has_rows carried over)."""
    torch = pytest.importorskip("torch")
    case = ge.window_bounds()
    reads_a = ge.build(case, cluster_fn(engine))
    planted = dict(case.planted)
    # table B: the same rows moved 2 bases later (fewer cover), contig 0's rows moved to contig 9 (contig 0: NO_READS)
    reads_b = {k: v.copy() for k, v in reads_a.items()}
    reads_b["start"] += 2
    reads_b["end"] += 2
    reads_b["chrom"][reads_b["chrom"] == 0] = 9
    answers = []
    for reads in (reads_a, reads_b):
        cands, genos, names = oracle_lib.cluster(case.params, case.lens, case.sigs, reads)
        want, no_reads = ge.rule_genos(cands, names, reads, case.params, oracle_lib.cal_gl)
        answers.append((cands, genos, names, want, no_reads))
    assert not np.array_equal(answers[0][3]["dr"], answers[1][3]["dr"])
    assert answers[1][4].any() and not answers[0][4].any()
    assert ge.dr_by_contig(answers[0][0], answers[0][3]) == {c: n for c, n in planted.items()}
    engine.set_params(case.params)
    engine.set_contigs(case.lens)
    dev = [{k: torch.as_tensor(v).cuda() for k, v in r.items()} for r in (reads_a, reads_b)]
    sigs = {k: {f: torch.as_tensor(x).cuda() for f, x in v.items() if x is not None} for k, v in case.sigs.items()}
    r0 = engine.graph_replays()
    for call in range(5):
        which = call % 2
        engine.upload(sigs, dev[which])
        engine.cluster_device()
        got = engine.fetch()
        cands, genos, names, want, no_reads = answers[which]
        d = compare_records.diff_records((cands, genos, names), got)
        assert not d, (call, d[:3])
        windowed = ge.n_windows(got[0]) > 0
        d = ge.diff_genos(want[windowed], got[1][windowed])
        assert not d, (call, d)
    torch.cuda.synchronize()
    assert engine.graph_replays() - r0 >= 2


@pytest.mark.parametrize("name,cap", [("window_bounds", 0), ("lin64_bottom", 0), ("lin64_bottom", 1)])
def test_rows_ending_before_they_start_are_rejected(engine, monkeypatch, name, cap):
    """end < start and start < 0, on both pair routes, with the pair buffer and (cap 1) inline: an input error."""
    case = CASES[name]
    reads = ge.build(case, cluster_fn(engine))
    if cap:
        monkeypatch.setenv("CUTESV_B200_PAIR_CAP", str(cap))
    eng = Engine(0, params=case.params, contig_lens=case.lens)
    try:
        for col, v in (("end", int(reads["start"][0]) - 1), ("start", -1)):
            bad = {k: x.copy() for k, x in reads.items()}
            bad[col][0] = v
            with pytest.raises(CuteSVError) as e:
                eng.cluster(case.sigs, bad)
            assert e.value.code == _abi.CSV_E_INPUT
        got = eng.cluster(case.sigs, reads)   # the engine still works
        check(eng, case, reads, got)
    finally:
        eng.close()


@pytest.mark.parametrize("name", ["tra_steps", "tra_rounds"])
def test_tra_warp_steps(engine, name):
    """k_tra_genotype's warp-cooperative count_coverage against the plain Python loop, the oracle and the planted DR: up_bound
    reached at lanes 31 and 0 of consecutive 32-record steps, the round reached on a secondary record, primary / iteration
    exactly 0.2, both returns on one record, an intra-contig pair, windows clamped at 0 and at the contig length, and the
    max_span lower bound."""
    case = {c.name: c for c in ge.tra_cases()}[name]
    aln = ge.build_tra(case, cluster_fn(engine))
    engine.upload_alignments(aln)
    try:
        got = engine.cluster(case.sigs, ge.EMPTY_READS)
    finally:
        engine.upload_alignments(None)
    ref = oracle_lib.cluster(case.params, case.lens, case.sigs, ge.EMPTY_READS, aln=aln)
    d = compare_records.diff_records(ref, got)
    assert not d, "\n".join(d[:5])
    assert not (got[0]["flags"] & _abi.CSV_F_GT_HOST).any()
    sel, want, by = ge.tra_genos(got[0], got[2], aln, case.params, case.lens, oracle_lib.cal_gl)
    d = ge.diff_genos(want, got[1][sel])
    assert not d, "\n".join(d)
    assert by == case.planted
