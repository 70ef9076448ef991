"""csv_cluster's genotype pass at its window, bin, tile and contig edges, without a GPU: every planted layout of
tests/genotype_edges.py hits the edge it is named for, and the emulator (which mirrors the kernels' linear-coordinate pass)
equals the oracle (per-contig cover counts), the numpy statement of the rule and the planted DR."""
import numpy as np
import pytest

import emul_lib
import genotype_edges as ge
from cutesv_b200 import _abi
from oracle import compare_records, oracle_lib

CASES = {c.name: c for c in ge.all_cases()}


def check_case(case, reads, got):
    """`got` (cands, genos, names) against the oracle, the rule and the planted DR of every planted contig."""
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


@pytest.mark.parametrize("name", sorted(CASES))
def test_layout_hits_its_edges(name):
    case = CASES[name]
    reads = ge.build(case, oracle_lib.cluster)
    cands, _, names = oracle_lib.cluster(case.params, case.lens, case.sigs, reads)
    assert case.planted and set(case.planted) <= set(ge.dr_by_contig(cands, np.zeros(len(cands), _abi.GENO_DTYPE)))
    edges = case.edges(cands, names, reads)
    missed = [k for k, v in edges.items() if not v]
    assert not missed, missed
    if name in ge.ROUTES:
        total, shift, lin32 = ge.ROUTES[name]
        lay = case.lay()
        assert (lay["total"], lay["shift"], lay["lin32"]) == (total, shift, lin32)
    if name == "bin_edges":
        assert case.lay()["shift"] == 10


def test_route_thresholds_are_exact():
    """The totals sit on the threshold itself: one base less changes the shift or the route."""
    for name, (total, shift, lin32) in ge.ROUTES.items():
        lay = ge.route_case(name).lay()
        assert (lay["shift"], lay["lin32"]) == (shift, lin32)
    p = ge.params()
    for total in ((1 << 30) + 1024, (1 << 31) + 2048):
        assert ge.layout(p, [total - ge.pad_of(p)])["shift"] == ge.layout(p, [total - 1 - ge.pad_of(p)])["shift"] + 1
    assert not ge.layout(p, [(1 << 31) - 1] * 2)["lin32"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_emulator_matches_oracle_and_rule(name):
    case = CASES[name]
    reads = ge.build(case, emul_lib.cluster)
    check_case(case, reads, emul_lib.cluster(case.params, case.lens, case.sigs, reads))


@pytest.mark.parametrize("n_reads", ge.TILE_SIZES)
def test_emulator_tiles(n_reads):
    case = ge.tiles(n_reads)
    reads = ge.build(case, emul_lib.cluster)
    assert len(reads["chrom"]) == n_reads
    check_case(case, reads, emul_lib.cluster(case.params, case.lens, case.sigs, reads))


def test_emulator_rejects_rows_ending_before_they_start():
    """Pins the emulator's mirror of k_reads_pass's input check (the library's own check is in the GPU test)."""
    case = ge.window_bounds()
    reads = ge.build(case, emul_lib.cluster)
    emul_lib.cluster(case.params, case.lens, case.sigs, reads)
    for col, v in (("end", reads["start"][0] - 1), ("start", -1)):
        bad = {k: x.copy() for k, x in reads.items()}
        bad[col][0] = v
        with pytest.raises(RuntimeError):
            emul_lib.cluster(case.params, case.lens, case.sigs, bad)


TRA = {c.name: c for c in ge.tra_cases()}


def _contig_recs(aln, c):
    sel = aln["chrom"] == c
    return [(int(a), int(b), int(r), bool(q)) for a, b, r, q in zip(aln["start"][sel], aln["end"][sel], aln["read_id"][sel], aln["is_primary"][sel])]


def test_tra_layouts_hit_their_warp_steps():
    """The record that returns sits at the lane and 32-record step each spot is named for, counted from the first record of
    the max_span lower bound; the round spots return on the record they are named for."""
    case = TRA["tra_steps"]
    aln = ge.build_tra(case, oracle_lib.cluster)
    cands, _, names = oracle_lib.cluster(case.params, case.lens, case.sigs, ge.EMPTY_READS)
    for name, (c, lane, step) in case.lanes.items():
        recs = _contig_recs(aln, c)
        i, s, e = ge._tra_window(cands, c, case.params, case.lens)
        lo = sum(r[0] < s - max(b - a for a, b, _, _ in recs) for r in recs)
        acc = [0, 0, -1]
        assert ge.py_count_coverage(recs, s, e, set(ge.supporters(cands, names, i).tolist()), 20, case.params.gt_round, acc, 1, 0) == 1
        assert ((acc[2] - lo) % 32, (acc[2] - lo) // 32) == (lane, step) == (ge.TRA_UP_LANES[name] % 32, ge.TRA_UP_LANES[name] // 32)
        assert recs[acc[2] + 1][0] < e, name   # spanning records follow the one that returns
    recs = _contig_recs(aln, 8)
    _, s, e = ge._tra_window(cands, 8, case.params, case.lens)
    span = max(b - a for a, b, _, _ in recs)
    assert sorted(a for a, _, _, _ in recs)[1] == s - span   # a record exactly at the lower bound, one below it
    _, s, e = ge._tra_window(cands, 5, case.params, case.lens)
    assert s == 0 and int(cands["pos"][ge._tra_window(cands, 5, case.params, case.lens)[0]]) < case.params.bias_tra
    i, s, e = ge._tra_window(cands, 7, case.params, case.lens)
    assert e == case.lens[7] < int(cands["pos"][i]) + case.params.bias_tra
    i = ge._tra_window(cands, 4, case.params, case.lens)[0]
    assert int(cands["aux"][i]) >> 2 == 4   # intra-contig pair
    case = TRA["tra_rounds"]
    aln = ge.build_tra(case, oracle_lib.cluster)
    cands, _, names = oracle_lib.cluster(case.params, case.lens, case.sigs, ge.EMPTY_READS)
    for c, (round_rec_primary, ret_k, ratio) in {0: (False, 20, 5 / 21), 1: (True, 19, 0.2), 2: (True, 19, 1.0)}.items():
        recs = _contig_recs(aln, c)
        _, s, e = ge._tra_window(cands, c, case.params, case.lens)
        assert recs[19][3] == round_rec_primary   # the 20th fetched record: every record here is fetched
        acc = [0, 0, -1]
        ge.py_count_coverage(recs, s, e, set(), 20, case.params.gt_round, acc, 1, 0)
        prim = sum(r[3] for r in recs[:ret_k + 1])
        assert acc[2] == ret_k and prim / (ret_k + 1) == ratio, c
    assert acc[0] == 20   # spot 2: up_bound and the round on the same record


@pytest.mark.parametrize("name", sorted(TRA))
def test_tra_emulator_matches_python_loop_and_oracle(name):
    """core.h's scalar tra_count_coverage (run by the emulator) against the plain loop and the oracle, and the planted DR."""
    case = TRA[name]
    aln = ge.build_tra(case, emul_lib.cluster)
    got = emul_lib.cluster(case.params, case.lens, case.sigs, ge.EMPTY_READS, aln=aln)
    ref = oracle_lib.cluster(case.params, case.lens, case.sigs, ge.EMPTY_READS, aln=aln)
    d = compare_records.diff_records(ref, got)
    assert not d, "\n".join(d[:5])
    sel, want, by = ge.tra_genos(got[0], got[2], aln, case.params, case.lens, oracle_lib.cal_gl)
    d = ge.diff_genos(want, got[1][sel])
    assert not d, "\n".join(d)
    assert by == case.planted
