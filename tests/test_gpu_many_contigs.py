"""Draft assemblies with more than 32767 contigs: every SV type, with --genotype and the all-alignments table, equal to the
oracle at contig counts on both sides of the point where the TRA key (chr1, chr2*4+type, pos1) needs more than 64 bits
(2*ceil(log2 n) + 33 > 64, i.e. from 32769 contigs on) and is replaced by the dense rank of the (chr1, chr2*4+type) pair.
Also the chained-sorts fallback for long runs of equal primary keys and CUDA-graph replay at those contig counts."""
import numpy as np
import pytest

from cutesv_b200 import _abi, synth
from oracle import compare_records, oracle_lib

SIZES = [32767, 32768, 32769, 40000, 100000, 1 << 20]


def _aln(reads):
    order = np.lexsort((np.arange(len(reads["chrom"])), reads["start"], reads["chrom"]))
    return {k: v[order] for k, v in reads.items()}


def _tra_on_high_ids(cands):
    tra = cands["svtype"] == _abi.CSV_TRA
    return int((tra & ((cands["chrom"] >= 32768) | ((cands["aux"] >> 2) >= 32768))).sum())


def _big_run(case, n_copies=2300):
    """n_copies TRA signatures with one (chr1, chr2, type, pos1) from distinct reads: a run of equal primary keys longer
    than the ranking kernel takes (RUN_MAX = 2048), so the type reruns through the chained sorts."""
    act = case["active"]
    tra = {k: (v.copy() if v is not None else None) for k, v in case["sigs"]["TRA"].items()}
    rid = np.unique(case["reads"]["read_id"])[:n_copies]
    m = len(rid)
    add = dict(chrom=np.full(m, act[-1], np.int32), a=np.full(m, 150000, np.int32), b=(200000 + np.arange(m) % 7).astype(np.int32),
               read_id=rid.astype(np.int32), c=np.full(m, int(act[len(act) // 2]) * 4 + 1, np.int32))
    sigs = dict(case["sigs"])
    sigs["TRA"] = {k: np.concatenate([tra[k], add[k]]) for k in tra}
    return sigs, m


def _check(engine, case, sigs):
    p = _abi.default_params(**case["params"])
    aln = _aln(case["reads"])
    engine.set_params(p)
    engine.set_contigs(case["lens"])
    engine.upload_alignments(aln)
    try:
        got = engine.cluster(sigs, case["reads"])
        ref = oracle_lib.cluster(p, case["lens"], sigs, case["reads"], n_threads=8, aln=aln)
    finally:
        engine.upload_alignments(None)
    d = compare_records.diff_records(ref, got)
    assert not d, "\n".join(d[:5])
    return got


def _profiled(case, sigs):
    """The same comparison on a fresh, profiled ctx: its kernel table then names exactly the kernels this call launched
    (including a rerun after ST_BIG_RUN)."""
    from cutesv_b200.engine import Engine
    eng = Engine(0)
    try:
        eng.set_profiling(True)
        got = _check(eng, case, sigs)
        return got, set(eng.kernel_times())
    finally:
        eng.close()


COMPACT_KERNELS = {"k_tra_pair_flags", "k_tra_compact_key"}


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_draft_assembly_matches_oracle(engine, n):
    case = synth.draft_assembly(n)
    got = _check(engine, case, case["sigs"])
    cands, genos = got[0], got[1]
    assert set(np.unique(cands["svtype"]).tolist()) == set(range(_abi.CSV_NTYPES))
    tra = cands["svtype"] == _abi.CSV_TRA
    assert (genos["status"][tra] != 1).all()   # genotyped on the device from the all-alignments table
    if n > 32768:
        assert _tra_on_high_ids(cands) > 0
    # the packed key up to 32768 contigs (2*ceil(log2 n) + 33 <= 64), the pair-rank key from 32769 on
    _, kt = _profiled(case, case["sigs"])
    if n > 32768:
        assert COMPACT_KERNELS <= kt
    else:
        assert not COMPACT_KERNELS & kt


@pytest.mark.gpu
def test_long_run_of_equal_tra_keys_on_many_contigs(engine):
    case = synth.draft_assembly(100000, seed=9)
    sigs, m = _big_run(case)
    assert m > 2048
    got, kt = _profiled(case, sigs)
    tra = got[0]["svtype"] == _abi.CSV_TRA
    assert got[0]["support"][tra].max() >= 2048
    # the compact key fed the chained-sorts fallback: k_gather_keys is launched only there
    assert COMPACT_KERNELS <= kt and any("k_gather_keys" in k for k in kt)
    _, kt_plain = _profiled(case, case["sigs"])
    assert not any("k_gather_keys" in k for k in kt_plain)


@pytest.mark.gpu
def test_graph_replay_on_many_contigs(engine):
    case = synth.draft_assembly(1 << 20, seed=13)
    p = _abi.default_params(**case["params"])
    aln = _aln(case["reads"])
    engine.set_params(p)
    engine.set_contigs(case["lens"])
    engine.upload_alignments(aln)
    try:
        engine.upload(case["sigs"], case["reads"])
        ref = oracle_lib.cluster(p, case["lens"], case["sigs"], case["reads"], n_threads=8, aln=aln)
        outs = []
        r0 = engine.graph_replays()
        for _ in range(3):
            engine.cluster_device(0x1F)
            outs.append(engine.fetch())
        assert engine.graph_replays() > r0
    finally:
        engine.upload_alignments(None)
    for got in outs:
        d = compare_records.diff_records(ref, got)
        assert not d, "\n".join(d[:5])
    assert _tra_on_high_ids(outs[-1][0]) > 0


@pytest.mark.gpu
def test_contig_table_of_2_pow_29_is_refused(engine):
    """TRA carries chr2*4+type in int32, so a table of 2^29 contigs or more is refused before anything is read or changed."""
    import ctypes as C
    lens = np.full(1, 1000, np.int64)
    rc = engine.L.csv_set_contigs(engine.h, C.c_int32(1 << 29), lens.ctypes.data_as(C.POINTER(C.c_int64)))
    assert rc == _abi.CSV_E_INVALID
