"""-m gpu: the device overlap/cover pass behind the genotype drop-ins (csv_overlap_cover, csv_call_gt).

- overlap_cover / assign_gt / the resolvers' call_gt equal the reference's stored outputs (tests/golden/genotype_dropin.json.gz);
- the device-resident reads table gives the same answers as host columns and leaves csv_cluster's results alone;
- a random multi-contig case (1e5 rows x 1e4 windows) equals a numpy evaluation of the overlap / cover rules;
- on clustering goldens, call_gt's DR and genotype equal the csv_geno csv_cluster computed."""
import numpy as np
import pytest

import genotype_golden as gg
import golden_util
from genotype_edges import windows_of_candidates
from cutesv_b200 import _abi, runtime
from cutesv_b200._lib import CuteSVError
from oracle import compare_records

pytestmark = pytest.mark.gpu


@pytest.fixture
def gpu_engine(engine):
    prev = runtime._engine
    runtime.set_engine(engine)
    yield engine
    runtime.set_engine(prev)


def test_overlap_cover_and_assign_gt_goldens(gpu_engine):
    for case in gg.data()["overlap_cover"]:
        gg.check_overlap_cover(case)
    for case in gg.data()["assign_gt"]:
        gg.check_assign_gt(case)


def test_call_gt_goldens(gpu_engine, tmp_path):
    path = str(tmp_path) + "/"
    idx = gg.write_reads_workdir(path)
    for case in gg.data()["call_gt"]:
        gg.check_call_gt(case, path, idx)


def test_bad_inputs_are_input_errors(engine):
    reads = dict(chrom=np.zeros(2, np.int32), start=np.array([5, 9], np.int32), end=np.array([7, 3], np.int32),
                 read_id=np.zeros(2, np.int32), is_primary=np.ones(2, np.uint8))
    ok = _abi.make_windows([0], [0], [20])
    with pytest.raises(CuteSVError) as e:
        engine.overlap_cover(ok, reads)
    assert e.value.code == _abi.CSV_E_INPUT
    for w in (_abi.make_windows([0], [8], [8]), _abi.make_windows([-1], [0], [4])):
        with pytest.raises(CuteSVError) as e:
            engine.overlap_cover(w, dict(reads, end=np.array([7, 30], np.int32)))
        assert e.value.code == _abi.CSV_E_INPUT


def brute_force(windows, reads):
    """The overlap / cover rules per window with numpy: rows of the window's contig with start < e and end > s overlap, primary
    ones with start <= s and end >= e cover."""
    n = len(windows)
    it, pn = np.zeros(n, np.int64), np.zeros(n, np.int64)
    cov, ovl = [], []
    rs2, re2 = 2 * reads["start"].astype(np.int64), 2 * reads["end"].astype(np.int64)
    by_contig = {}
    for c in np.unique(reads["chrom"]):
        sel = np.flatnonzero(reads["chrom"] == c)
        sel = sel[np.argsort(rs2[sel], kind="stable")]
        by_contig[int(c)] = (sel, rs2[sel], int((re2[sel] - rs2[sel]).max()))
    for i, w in enumerate(windows):
        if int(w["chrom"]) not in by_contig:
            cov.append(np.zeros(0, np.int32)); ovl.append(np.zeros(0, np.int32))
            continue
        sel, starts, span = by_contig[int(w["chrom"])]
        k = sel[np.searchsorted(starts, w["s2"] - span):np.searchsorted(starts, w["e2"], side="left")]
        o = (rs2[k] < w["e2"]) & (re2[k] > w["s2"])
        p = o & (reads["is_primary"][k] != 0)
        c = p & (rs2[k] <= w["s2"]) & (re2[k] >= w["e2"])
        it[i], pn[i] = o.sum(), p.sum()
        cov.append(np.unique(reads["read_id"][k[c]]))
        ovl.append(np.unique(reads["read_id"][k[p]]))
    return it, pn, cov, ovl


def random_case(seed, n_reads=100000, n_win=10000):
    rng = np.random.default_rng(seed)
    lens = np.array([2_000_000, 500_000, 3_000_000, 50_000, 1_000_000])
    dens = np.array([0.45, 0.05, 0.25, 0.2, 0.05])   # contigs 1 and 4 are sparse (short segments: warp path), contig 3 piles up
    ch = rng.choice(len(lens), n_reads, p=dens / dens.sum()).astype(np.int32)
    st = (rng.random(n_reads) * lens[ch]).astype(np.int32)
    ln = np.where(rng.random(n_reads) < 0.03, 0, rng.integers(1, 20000, n_reads)).astype(np.int32)
    reads = dict(chrom=ch, start=st, end=st + ln, read_id=rng.integers(0, n_reads // 3, n_reads).astype(np.int32),
                 is_primary=(rng.random(n_reads) < 0.85).astype(np.uint8))
    wc = rng.integers(0, len(lens) + 1, n_win).astype(np.int32)   # contig 5 has windows but no rows
    centre = (rng.random(n_win) * np.append(lens, 10000)[wc]).astype(np.int64)
    half = rng.choice([200, 1000, 2000, 401, 1001], n_win)        # half-widths in half units: odd -> x.5 bounds
    s2 = np.maximum(2 * centre - half, 0)
    s2[:50] = 0                                                   # windows clamped at 0
    return reads, _abi.make_windows(wc, s2, 2 * centre + half)


def test_random_multi_contig_matches_numpy(engine):
    reads, win = random_case(7)
    got = engine.overlap_cover(win, reads)
    it, pn, cov, ovl = brute_force(win, reads)
    assert np.array_equal(got["iteration"], it) and np.array_equal(got["primary_num"], pn)
    for name, exp in (("cover", cov), ("overlap", ovl)):
        off, ids = got[name + "_off"], got[name + "_ids"]
        assert np.array_equal(np.diff(off), [len(x) for x in exp]), name
        assert np.array_equal(ids, np.concatenate(exp)), name
    assert max(len(x) for x in ovl) > 2048 and min(len(x) for x in ovl) < 64   # both dedup kernels ran
    # call_gt on the same windows: pairs of consecutive windows, supports drawn from the covering ids
    rng = np.random.default_rng(8)
    n = len(win) // 2
    sup = [rng.choice(np.concatenate([cov[2 * i], cov[2 * i + 1], [10 ** 6]]), rng.integers(0, 8)) for i in range(n)]
    off = np.zeros(n + 1, np.int64)
    np.cumsum([len(x) for x in sup], out=off[1:])
    g = engine.call_gt(win, 2, off, np.concatenate(sup).astype(np.int32), reads)
    dr = [len(np.setdiff1d(np.union1d(cov[2 * i], cov[2 * i + 1]), sup[i])) for i in range(n)]
    assert np.array_equal(g["dr"], dr) and np.array_equal(g["dv"], [len(x) for x in sup])
    ref = engine.cal_gl(dr, [len(x) for x in sup])
    for k in ("gt", "pl", "gq", "qual"):
        assert np.array_equal(g[k], ref[k]), k


@pytest.mark.parametrize("name", ["cfg2_s0p002", "cfg3_s0p004"])
def test_call_gt_agrees_with_cluster_genotyper(engine, name):
    case = golden_util.load_case(name)
    p = case["params"]
    engine.set_params(p)
    engine.set_contigs(case["lens"])
    engine.upload(case["sigs"], case["reads"])
    engine.cluster_device()
    cands, genos, names = engine.fetch()
    before = [x.copy() for x in (cands, genos, names)]
    win = windows_of_candidates(cands, p)
    checked = 0
    for per, types in ((1, (_abi.CSV_DEL, _abi.CSV_INS)), (2, (_abi.CSV_DUP, _abi.CSV_INV))):
        sel = np.flatnonzero(np.isin(cands["svtype"], types) & (genos["status"] == 0))
        if not len(sel):
            continue
        off = np.zeros(len(sel) + 1, np.int64)
        np.cumsum(cands["names_cnt"][sel], out=off[1:])
        ids = np.concatenate([names[o:o + k] for o, k in zip(cands["names_off"][sel], cands["names_cnt"][sel])])
        w = win[sel][:, :per].reshape(-1)
        host = engine.call_gt(w, per, off, ids, case["reads"])
        resident = engine.call_gt(w, per, off, ids)             # the table csv_cluster used
        for k in ("dr", "dv", "gt", "pl", "gq", "qual"):
            assert np.array_equal(host[k], genos[sel][k]), (per, k)
            assert np.array_equal(resident[k], host[k]), (per, k)
        oc_host = engine.overlap_cover(w, case["reads"])
        oc_dev = engine.overlap_cover(w)
        for k in oc_host:
            assert np.array_equal(oc_host[k], oc_dev[k]), k
        checked += len(sel)
    assert checked > 0
    # the results of the last csv_cluster are untouched, and a following csv_cluster returns the same records (names_off and
    # `cluster` are layout details that may differ between two csv_cluster calls)
    for a, b in zip(before, engine.fetch()):
        assert np.array_equal(a, b)
    engine.cluster_device()
    d = compare_records.diff_records(before, engine.fetch())
    assert not d, "\n".join(d[:3])
