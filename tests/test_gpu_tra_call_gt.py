"""-m gpu: the standalone TRA genotyper (csv_tra_call_gt -> k_tra_call_gt) behind resolveTRA's call_gt drop-ins.

- call_gt / call_gt_batch equal the reference's stored outputs (tests/golden/tra_call_gt.json.gz), types included;
- fed csv_cluster's own TRA candidates (positions and support segments), it returns csv_cluster's genotypes, from a host
  table and from the installed one (aln=None);
- 10^4 seeded multi-contig queries equal the plain count_coverage loop of tests/genotype_edges.py;
- every error code, after which the last results, the installed alignment table and graph replay are unchanged."""
import ctypes as C

import numpy as np
import pytest

import golden_util
import tra_call_gt_golden as tg
from genotype_edges import py_count_coverage
from tra_call_gt_golden import fake_bam  # noqa: F401 (fixture)
from cutesv_b200 import _abi, runtime
from cutesv_b200._lib import CuteSVError
from cutesv_b200.engine import Engine
from oracle import compare_records

pytestmark = pytest.mark.gpu

FIELDS = ("dr", "dv", "gt", "pl", "gq", "status", "qual")


@pytest.fixture
def gpu_engine(engine):
    prev = runtime._engine
    runtime.set_engine(engine)
    yield engine
    runtime.set_engine(prev)


def test_dropins_match_goldens(gpu_engine, fake_bam):
    tg.check_call_gt(fake_bam)
    tg.check_call_gt_batch(fake_bam)


def bam_order(reads):
    order = np.lexsort((np.arange(len(reads["chrom"])), reads["start"], reads["chrom"]))
    return {k: v[order] for k, v in reads.items()}


def candidate_queries(cands, names):
    """csv_cluster's TRA candidates as queries + support CSR."""
    sel = np.flatnonzero(cands["svtype"] == _abi.CSV_TRA)
    c = cands[sel]
    q = np.zeros(len(sel), _abi.TRA_QUERY_DTYPE)
    q["chr1"], q["pos1"], q["chr2"], q["pos2"] = c["chrom"], c["pos"], c["aux"] >> 2, c["pos2"]
    off = np.zeros(len(sel) + 1, np.int64)
    np.cumsum(c["names_cnt"], out=off[1:])
    ids = np.concatenate([names[o:o + k] for o, k in zip(c["names_off"], c["names_cnt"])]).astype(np.int32)
    return sel, q, off, ids


@pytest.mark.parametrize("name", ["cfg3_s0p004", "adv034", "adv144"])
def test_agrees_with_cluster_genotyper(engine, name):
    case = golden_util.load_case(name)
    p = case["params"]
    aln = bam_order(case["reads"])
    engine.set_params(p)
    engine.set_contigs(case["lens"])
    engine.upload_alignments(aln)
    try:
        cands, genos, names = engine.cluster({"TRA": case["sigs"]["TRA"]}, case["reads"])
        sel, q, off, ids = candidate_queries(cands, names)
        assert len(sel) > 0
        host = engine.tra_call_gt(q, off, ids, p.bias_tra, p.gt_round, aln=aln)
        resident = engine.tra_call_gt(q, off, ids, p.bias_tra, p.gt_round)
        for k in FIELDS:
            assert np.array_equal(host[k], genos[sel][k]), k
            assert np.array_equal(resident[k], host[k]), k
    finally:
        engine.upload_alignments(None)


def random_case(seed, n_q=10_000):
    """Five contigs of decreasing record density (the last has none); pairs across contigs and on one contig, some with
    overlapping windows; positions up to a bias past either end; support lists with duplicates and absent ids."""
    rng = np.random.default_rng(seed)
    lens = np.array([1_000_000, 800_000, 600_000, 400_000, 300_000], np.int64)
    counts = [40_000, 15_000, 4_000, 800, 0]
    cols = {k: [] for k in ("chrom", "start", "end", "read_id", "is_primary")}
    next_id = 0
    for c, n in enumerate(counts):
        st = np.sort(rng.integers(0, lens[c], n))
        en = st + rng.integers(1, 5_000, n)
        prim = rng.random(n) < 0.8
        rid = np.where(prim, np.arange(next_id, next_id + n), rng.integers(0, next_id + n, n))   # one primary per id
        next_id += n
        for k, v in zip(cols, (np.full(n, c), st, en, rid, prim)):
            cols[k].append(v)
    aln = {k: np.concatenate(v).astype(np.uint8 if k == "is_primary" else np.int32) for k, v in cols.items()}
    bias, gt_round = 500, 60
    q = np.zeros(n_q, _abi.TRA_QUERY_DTYPE)
    q["chr1"] = rng.integers(0, len(lens), n_q)
    q["chr2"] = np.where(rng.random(n_q) < 0.3, q["chr1"], rng.integers(0, len(lens), n_q))
    for a, b in (("chr1", "pos1"), ("chr2", "pos2")):
        q[b] = (rng.random(n_q) * (lens[q[a]] + 2 * bias)).astype(np.int64) - bias
    near = (q["chr1"] == q["chr2"]) & (rng.random(n_q) < 0.5)
    q["pos2"][near] = np.clip(q["pos1"][near] + rng.integers(-800, 800, near.sum()), -bias, lens[q["chr1"][near]] + bias)
    sup = [rng.choice(np.append(aln["read_id"][rng.integers(0, len(aln["read_id"]), 30)], [10 ** 8]), rng.integers(0, 25))
           for _ in range(n_q)]
    off = np.zeros(n_q + 1, np.int64)
    np.cumsum([len(x) for x in sup], out=off[1:])
    return lens, aln, q, off, np.concatenate(sup).astype(np.int32), bias, gt_round


def loop_genotypes(lens, aln, q, off, ids, bias, gt_round):
    """(DR or -1, DV) per query by py_count_coverage over each window's records from the first one that can overlap."""
    by = {}
    for c in range(len(lens)):
        m = aln["chrom"] == c
        recs = list(zip(aln["start"][m].tolist(), aln["end"][m].tolist(), aln["read_id"][m].tolist(), (aln["is_primary"][m] != 0).tolist()))
        span = int((aln["end"][m] - aln["start"][m]).max()) if m.any() else 0
        by[c] = (recs, aln["start"][m], span)

    def scan(c, s, e, sup, up, acc, xs, xe):
        recs, starts, span = by[c]
        return py_count_coverage(recs[int(np.searchsorted(starts, s - span)):], s, e, sup, up, gt_round, acc, xs, xe)

    dr = np.zeros(len(q), np.int32)
    for i, x in enumerate(q.tolist()):
        chr1, chr2, pos1, pos2 = x
        sup = set(ids[off[i]:off[i + 1]].tolist())
        n = int(off[i + 1] - off[i])
        up = 20 * n if n <= 2 else 9 * n if n <= 5 else 7 * n if n <= 15 else 5 * n
        acc = [0, 0]
        s, e = max(pos1 - bias, 0), min(pos1 + bias, int(lens[chr1]))
        st = scan(chr1, s, e, sup, up, acc, 1, 0)
        if st == 0:
            s2, e2 = max(pos2 - bias, 0), min(pos2 + bias, int(lens[chr2]))
            scan(chr2, s2, e2, sup, up, acc, *((s, e) if chr2 == chr1 else (1, 0)))
        dr[i] = -1 if st == -1 else acc[1]
    return dr, np.diff(off).astype(np.int32)


def test_random_multi_contig_matches_loop(engine):
    lens, aln, q, off, ids, bias, gt_round = random_case(11)
    engine.set_contigs(lens)
    got = engine.tra_call_gt(q, off, ids, bias, gt_round, aln=aln)
    dr, dv = loop_genotypes(lens, aln, q, off, ids, bias, gt_round)
    noisy = dr < 0
    assert 0.05 < noisy.mean() < 0.95 and (dr > 0).any() and (q["chr1"] == q["chr2"]).any()
    assert np.array_equal(got["status"], np.where(noisy, 2, 0)) and np.array_equal(got["dv"], dv) and np.array_equal(got["dr"], dr)
    assert (got["gt"][noisy] == -1).all()
    want = engine.cal_gl(dr[~noisy], dv[~noisy])
    for k in ("gt", "pl", "gq", "qual"):
        assert np.array_equal(got[k][~noisy], want[k]), k


def raw_call(engine, q, n, aln, off, ids, out, bias=50, gt_round=500):
    r, keep = _abi.make_reads_cols(aln) if aln is not None else (None, ())
    vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)   # noqa: E731
    return engine.L.csv_tra_call_gt(engine.h, vp(q), C.c_int64(n), C.byref(r) if r is not None else None, C.c_int32(bias),
                                    C.c_int32(gt_round), None if off is None else off.ctypes.data_as(C.POINTER(C.c_int64)),
                                    _abi.ptr(ids), vp(out))


def test_errors_leave_ctx_unchanged(engine):
    case = golden_util.load_case("adv034")
    p = case["params"]
    lens = np.asarray(case["lens"], np.int64)
    aln = bam_order(case["reads"])
    fresh = Engine(0)   # no contig table
    try:
        with pytest.raises(CuteSVError) as e:
            fresh.tra_call_gt(np.zeros(1, _abi.TRA_QUERY_DTYPE), [0, 0], [], 50, 500, aln=aln)
        assert e.value.code == _abi.CSV_E_STATE
    finally:
        fresh.close()
    engine.set_params(p)
    engine.set_contigs(lens)
    engine.upload_alignments(None)
    cands, _, names = engine.cluster({"TRA": case["sigs"]["TRA"]}, case["reads"])
    _, q, off, ids = candidate_queries(cands, names)
    with pytest.raises(CuteSVError) as e:   # no installed table
        engine.tra_call_gt(q, off, ids, p.bias_tra, p.gt_round)
    assert e.value.code == _abi.CSV_E_STATE
    engine.upload_alignments(aln)
    engine.upload({"TRA": case["sigs"]["TRA"]}, case["reads"])
    good = engine.tra_call_gt(q, off, ids, p.bias_tra, p.gt_round, aln=aln)   # (the call's scratch exists before the capture)
    for _ in range(3):   # eager, eager, capture
        engine.cluster_device()
    before = [x.copy() for x in engine.fetch()]
    table = engine.fetch_alignments()
    r0 = engine.graph_replays()
    out = np.zeros(len(q), _abi.GENO_DTYPE)
    n = len(q)
    bad_off = off.copy()
    bad_off[1] = bad_off[2] + 1   # decreases at 2
    invalid = [lambda: raw_call(engine, q, -1, aln, off, ids, out), lambda: raw_call(engine, q, 1 << 29, aln, off, ids, out),
               lambda: raw_call(engine, None, n, aln, off, ids, out), lambda: raw_call(engine, q, n, aln, None, ids, out),
               lambda: raw_call(engine, q, n, aln, off, ids, None), lambda: raw_call(engine, q, n, aln, off, None, out),
               lambda: raw_call(engine, q, n, aln, off, ids, out, bias=-1), lambda: raw_call(engine, q, n, aln, off + 1, ids, out),
               lambda: raw_call(engine, q, n, aln, bad_off, ids, out)]
    for k, f in enumerate(invalid):
        assert f() == _abi.CSV_E_INVALID, k
    inputs = []
    for field, v in (("chr1", -1), ("chr2", len(lens)), ("pos1", int(lens[q["chr1"][3]]) + p.bias_tra + 1), ("pos2", -p.bias_tra - 1)):
        bad = q.copy()
        bad[field][3] = v
        inputs.append((bad, aln))
    reversed_tbl = {k: v[::-1].copy() for k, v in aln.items()}
    far_contig = {k: v.copy() for k, v in aln.items()}
    far_contig["chrom"][-1] = len(lens)
    inputs += [(q, reversed_tbl), (q, far_contig)]
    for k, (qq, tbl) in enumerate(inputs):
        with pytest.raises(CuteSVError) as e:
            engine.tra_call_gt(qq, off, ids, p.bias_tra, p.gt_round, aln=tbl)
        assert e.value.code == _abi.CSV_E_INPUT, k
        if k < 4:
            assert "query 3" in str(e.value), str(e.value)
    for a, b in zip(before, engine.fetch()):
        assert np.array_equal(a, b)
    after = engine.fetch_alignments()
    assert after is not None and all(np.array_equal(table[k], after[k]) for k in table)
    for tbl in (aln, None):
        again = engine.tra_call_gt(q, off, ids, p.bias_tra, p.gt_round, aln=tbl)
        for k in FIELDS:
            assert np.array_equal(again[k], good[k]), k
    engine.cluster_device()
    assert engine.graph_replays() == r0 + 1
    d = compare_records.diff_records(before, engine.fetch())
    assert not d, "\n".join(d[:3])
    engine.upload_alignments(None)
