"""-m gpu: inputs that already live in GPU memory (csv_upload_*_device through Engine with torch CUDA tensors) give byte-identical
records to the host-input path, in the caller's stream order, across graph replays, and reject bad inputs without harm."""
import ctypes as C

import numpy as np
import pytest

import golden_util
from cutesv_b200 import _abi, _lib

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

CASES = ["cfg2_s0p002", "cfg3_s0p004"] + [n for n in golden_util.case_names() if n.startswith("adv")]


@pytest.fixture(scope="module")
def eng():
    from cutesv_b200.engine import Engine
    try:
        e = Engine(0)
    except _lib.CuteSVError as err:
        if err.code == _abi.CSV_E_NODEVICE:
            pytest.skip("no usable sm_90 device: %s" % err)
        raise
    yield e
    e.close()


def to_dev(cols):
    """Column dict -> torch CUDA tensors (int32; uint8 is_primary; int64 contig_off)."""
    if cols is None:
        return None
    out = {}
    for k, v in cols.items():
        if v is None:
            out[k] = None
            continue
        dt = np.uint8 if k == "is_primary" else (np.int64 if k == "contig_off" else np.int32)
        out[k] = torch.from_numpy(np.ascontiguousarray(v, dtype=dt)).to("cuda:0")
    return out


def grouped(case):
    n = len(case["lens"])
    return {k: _abi.group_by_contig(v, n) for k, v in case["sigs"].items()}, _abi.group_by_contig(case["reads"], n)


def setup(eng, case):
    eng.set_params(case["params"])
    eng.set_contigs(case["lens"])


def copy(res):
    return tuple(np.array(x, copy=True) for x in res)


def canonical(res):
    """Records with the names buffer's layout taken out: the buffer is filled through an atomic append cursor, so names_off
    (and the kept-cluster slot in `cluster`) differ from run to run on any input path.  Every other byte is compared, and
    every candidate's supporting read ids as its own slice."""
    cands, genos, names = res
    c = np.array(cands, copy=True)
    slices = np.concatenate([names[o:o + n] for o, n in zip(c["names_off"], c["names_cnt"])] + [np.zeros(0, np.int32)])
    c["names_off"] = 0
    c["cluster"] = 0
    return c.tobytes(), np.asarray(genos).tobytes(), slices.tobytes(), len(names)


def assert_same(exp, got):
    for e, g, what in zip(canonical(exp), canonical(got), ("candidate records", "genotype records", "names", "names count")):
        assert e == g, what


def host_and_device(eng, case, sigs_dev, reads_dev, group=False):
    sigs, reads = grouped(case) if group else (case["sigs"], case["reads"])
    exp = copy(eng.cluster(sigs, reads, grouped=group))
    got = copy(eng.cluster(sigs_dev(sigs), reads_dev(reads), grouped=group))
    return exp, got


@pytest.mark.parametrize("name", CASES)
def test_device_inputs_match_host_inputs(eng, name):
    case = golden_util.load_case(name)
    setup(eng, case)
    exp, got = host_and_device(eng, case, lambda s: {k: to_dev(v) for k, v in s.items()}, to_dev)
    assert_same(exp, got)
    # zero-copy views of the same results
    cands, genos, names = eng.result_tensors()
    assert cands.is_cuda and cands.shape == (len(exp[0]), 16) and genos.shape == (len(exp[0]), 10) and names.dtype == torch.int32
    assert_same(eng.fetch(), (cands.cpu().numpy().view(_abi.CAND_DTYPE)[:, 0], genos.cpu().numpy().view(_abi.GENO_DTYPE)[:, 0],
                              names.cpu().numpy()))


@pytest.mark.parametrize("name", CASES)
def test_grouped_device_inputs_match_grouped_host_inputs(eng, name):
    case = golden_util.load_case(name)
    setup(eng, case)
    exp, got = host_and_device(eng, case, lambda s: {k: to_dev(v) for k, v in s.items()}, to_dev, group=True)
    assert_same(exp, got)


@pytest.mark.parametrize("name", ["cfg2_s0p002", "cfg3_s0p004", "adv034"])
def test_device_signatures_with_host_reads(eng, name):
    case = golden_util.load_case(name)
    setup(eng, case)
    exp, got = host_and_device(eng, case, lambda s: {k: to_dev(v) for k, v in s.items()}, lambda r: r)
    assert_same(exp, got)
    exp, got = host_and_device(eng, case, lambda s: s, to_dev)   # and the reverse
    assert_same(exp, got)


def test_device_alignment_table_matches_host(eng):
    case = golden_util.load_case("cfg3_s0p004")
    setup(eng, case)
    r = case["reads"]
    order = np.lexsort((np.arange(len(r["chrom"])), r["start"], r["chrom"]))
    aln = {k: np.ascontiguousarray(v[order]) for k, v in r.items()}
    eng.upload_alignments(aln)
    exp = copy(eng.cluster(case["sigs"], case["reads"]))
    eng.upload_alignments(to_dev(aln))
    got = copy(eng.cluster(case["sigs"], case["reads"]))
    eng.upload_alignments(None)
    assert_same(exp, got)


def produce(cols, stream):
    """The columns as the result of torch ops on `stream`, behind a ~20 ms spin, so that a copy not ordered after the
    producer would read the buffers before they are written."""
    out = {}
    with torch.cuda.stream(stream):
        torch.cuda._sleep(40_000_000)
        for k, v in cols.items():
            if v is None:
                out[k] = None
                continue
            dt = torch.uint8 if k == "is_primary" else torch.int32
            src = torch.from_numpy(np.ascontiguousarray(v)).pin_memory().to("cuda:0", non_blocking=True).to(torch.int64)
            out[k] = (src * 3 - 2 * src).to(dt)
    return out


def test_producer_stream_order(eng):
    case = golden_util.load_case("cfg3_s0p004")
    setup(eng, case)
    exp = copy(eng.cluster(case["sigs"], case["reads"]))
    s = torch.cuda.Stream()
    sigs = {k: produce(v, s) for k, v in case["sigs"].items()}
    reads = produce(case["reads"], s)
    eng.upload(sigs, reads, stream=s)
    eng.cluster_device()
    assert_same(exp, copy(eng.fetch()))
    # stream=None: torch's current stream, here the producer's
    sigs = {k: produce(v, s) for k, v in case["sigs"].items()}
    reads = produce(case["reads"], s)
    with torch.cuda.stream(s):
        eng.upload(sigs, reads)
    eng.cluster_device()
    assert_same(exp, copy(eng.fetch()))


def test_overwrite_after_upload_in_stream_order(eng):
    case = golden_util.load_case("cfg3_s0p004")
    setup(eng, case)
    exp = copy(eng.cluster(case["sigs"], case["reads"]))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        sigs = {k: to_dev(v) for k, v in case["sigs"].items()}
        reads = to_dev(case["reads"])
    s.synchronize()
    eng.upload(sigs, reads, stream=s)
    with torch.cuda.stream(s):   # the caller reuses its buffers right away
        for cols in list(sigs.values()) + [reads]:
            for v in cols.values():
                if v is not None:
                    v.fill_(-7)
    eng.cluster_device()
    assert_same(exp, copy(eng.fetch()))
    # freed and reallocated by torch's caching allocator in the same stream's order
    s2 = torch.cuda.Stream()
    with torch.cuda.stream(s2):
        sigs = {k: to_dev(v) for k, v in case["sigs"].items()}
        reads = to_dev(case["reads"])
        eng.upload(sigs, reads)
        del sigs, reads
        junk = [torch.full((1 << 20,), -9, dtype=torch.int32, device="cuda:0") for _ in range(8)]
    eng.cluster_device()
    assert_same(exp, copy(eng.fetch()))
    del junk


def test_graph_replay_with_device_inputs(eng):
    case = golden_util.load_case("cfg2_s0p002")
    setup(eng, case)
    mod = {k: dict(v) for k, v in case["sigs"].items()}
    mod["DEL"]["b"] = mod["DEL"]["b"] + 1        # new contents, the same sizes
    exp0 = copy(eng.cluster(case["sigs"], case["reads"]))
    exp1 = copy(eng.cluster(mod, case["reads"]))
    assert exp0[0].tobytes() != exp1[0].tobytes()
    reads = to_dev(case["reads"])
    r0 = eng.graph_replays()
    for _ in range(3):
        eng.upload({k: to_dev(v) for k, v in case["sigs"].items()}, reads)
        eng.cluster_device()
        assert_same(exp0, copy(eng.fetch()))
    r1 = eng.graph_replays()
    assert r1 > r0
    eng.upload({k: to_dev(v) for k, v in mod.items()}, reads)
    eng.cluster_device()
    assert_same(exp1, copy(eng.fetch()))
    assert eng.graph_replays() > r1


def test_host_pointer_to_device_call_is_invalid(eng):
    case = golden_util.load_case("adv034")
    setup(eng, case)
    s, keep = _abi.make_sig_cols(case["sigs"]["DEL"])
    rc = eng.L.csv_upload_sigs_device(eng.h, _abi.CSV_DEL, C.byref(s), None)
    assert rc == _abi.CSV_E_INVALID and b"chrom" in eng.L.csv_last_error()
    r, rkeep = _abi.make_reads_cols(case["reads"])
    assert eng.L.csv_upload_reads_device(eng.h, C.byref(r), None) == _abi.CSV_E_INVALID
    assert eng.L.csv_upload_alignments_device(eng.h, C.byref(r), None) == _abi.CSV_E_INVALID
    # a device struct with one host column: the message names that column
    d = to_dev(case["sigs"]["DEL"])
    ds, _ = _abi.device_cols(d, _abi.SIG_FIELDS, 0)
    ds.b = s.b
    assert eng.L.csv_upload_sigs_device(eng.h, _abi.CSV_DEL, C.byref(ds), None) == _abi.CSV_E_INVALID
    assert b"column b" in eng.L.csv_last_error()
    # the engine still computes correct records
    exp, got = host_and_device(eng, case, lambda x: {k: to_dev(v) for k, v in x.items()}, to_dev)
    assert_same(exp, got)


def test_bad_dtypes_and_lengths_raise_before_the_library(eng):
    case = golden_util.load_case("adv034")
    setup(eng, case)
    d = {k: to_dev(v) for k, v in case["sigs"].items()}
    d["DEL"]["a"] = d["DEL"]["a"].to(torch.int64)
    with pytest.raises(TypeError, match="column a"):
        eng.upload(d, to_dev(case["reads"]))
    d = {k: to_dev(v) for k, v in case["sigs"].items()}
    d["INS"]["b"] = d["INS"]["b"][:-1]
    with pytest.raises(ValueError, match="lengths"):
        eng.upload(d, to_dev(case["reads"]))
    r = to_dev(case["reads"])
    r["is_primary"] = r["is_primary"].to(torch.bool)
    with pytest.raises(TypeError, match="is_primary"):
        eng.upload({k: to_dev(v) for k, v in case["sigs"].items()}, r)
    d = {k: to_dev(v) for k, v in case["sigs"].items()}
    d["DEL"]["a"] = d["DEL"]["a"].cpu().numpy()
    with pytest.raises(ValueError, match="all device or all host"):
        eng.upload(d, to_dev(case["reads"]))


@pytest.mark.parametrize("slot", ["DEL", "reads"])
@pytest.mark.parametrize("bad", ["start", "end", "decrease"])
def test_bad_device_contig_offsets_fail_the_next_cluster(eng, slot, bad):
    case = golden_util.load_case("cfg3_s0p004")
    setup(eng, case)
    sigs_g, reads_g = grouped(case)
    exp = copy(eng.cluster(sigs_g, reads_g, grouped=True))
    sigs_d = {k: to_dev(v) for k, v in sigs_g.items()}
    reads_d = to_dev(reads_g)
    off = (reads_d if slot == "reads" else sigs_d[slot])["contig_off"].clone()
    n = int(off[-1])
    if bad == "start":
        off[0] = 1
    elif bad == "end":
        off[-1] = n + 1000
    else:
        off[3] = n          # everything up to contig 3 claims all rows, contig 3 "starts" after contig 4
        off[4] = 0
    target = reads_d if slot == "reads" else sigs_d[slot]
    good = target["contig_off"]
    target["contig_off"] = off
    eng.upload(sigs_d, reads_d, grouped=True)
    eng.cluster_device()
    with pytest.raises(_lib.CuteSVError) as err:
        eng.counts()
    assert err.value.code == _abi.CSV_E_INPUT and "contig_off" in str(err.value)
    # the same engine on valid inputs
    target["contig_off"] = good
    eng.upload(sigs_d, reads_d, grouped=True)
    eng.cluster_device()
    assert_same(exp, copy(eng.fetch()))
