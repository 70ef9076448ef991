"""-m gpu: SA:Z text reduced on the device (Engine.reduce_sa / csv_reduce_sa_device, csv_set_contig_names).  Against the native
decoder's host reduction of the same tags written into a BAM; packets that carry text against the same packets carrying the
host-reduced columns, through Engine.extract and Engine.scan up to cluster_device's candidates and genotypes; a table of 10^5
contig names; and every rejection, which changes nothing."""
import json
import os
import pickle

import numpy as np
import pytest

import bam_writer
import device_packet_util as dpu
import golden_util
import name_util
import sa_text_util as sat
from cutesv_b200 import _abi, _lib, bamio, cli, synth
from cutesv_b200.engine import Engine
from oracle import gen_cli_golden
from test_gpu_device_scan import _packets, _same_records, _state

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_table_left(engine):
    yield
    engine.extract_reset()
    engine.set_scan_regions([], None, {})
    engine.upload_alignments(None)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", 0))


def _reduce(engine, values):
    text, off = sat.text_arrays(values)
    sa_off, cols = engine.reduce_sa(_cuda(text), _cuda(off))
    return sa_off.cpu().numpy(), {f: v.cpu().numpy() for f, v in cols.items()}


def _assert_equal(got, want):
    assert np.array_equal(got[0], want[0]), np.flatnonzero(got[0] != want[0])[:5]
    for f in _abi.SA_FIELDS:
        assert np.array_equal(got[1][f], want[1][f]), (f, np.flatnonzero(got[1][f] != want[1][f])[:5])


def _bench_style_values(seed, n_reads):
    """The SA tags of a scripts/bench_cli.py-style record set (synth.synth_alignments), in BAM order, with its contigs."""
    reads, names, lens = synth.synth_alignments(seed, n_reads=n_reads, n_contigs=3, with_seq=False)
    order = {n: i for i, n in enumerate(names)}
    reads.sort(key=lambda r: (order[r.reference_name], r.reference_start))
    return [dict(r.get_tags()).get("SA") for r in reads], reads, list(zip(names, (int(x) for x in lens)))


def test_reduce_sa_equals_the_host_reduction(engine, tmp_path):
    bamio.build()
    engine.set_contigs(np.array([ln for _, ln in sorted(sat.CONTIGS)], np.int64), names=sat.NAMES)
    for k, values in enumerate([sat.adversarial_values()] + [sat.random_values(s, 3000) for s in range(3)]):
        path = str(tmp_path / ("a%d.bam" % k))
        sat.write_bam(path, values)
        _assert_equal(_reduce(engine, values), sat.host_reduce(path))
    # a seeded bench_cli-style BAM
    values, reads, contigs = _bench_style_values(5, 20_000)
    path = str(tmp_path / "bench.bam")
    bam_writer.write_bam(path, contigs, reads)
    names = sorted(n for n, _ in contigs)
    engine.set_contigs(np.array([dict(contigs)[n] for n in names], np.int64), names=names)
    rd = bamio.BamReader(path, threads=2, keep_seq=False)
    rd.set_chrom_ids({n: i for i, n in enumerate(names)})
    pk = rd.next_packet(1 << 30)
    rd.close()
    assert len(pk["sa"]["chrom"]) > 5000
    _assert_equal(_reduce(engine, values), (pk["sa_off"], pk["sa"]))
    # no records, and records without any tag
    assert _reduce(engine, [])[0].tolist() == [0]
    off, cols = _reduce(engine, [None] * 70)
    assert off.tolist() == [0] * 71 and all(len(v) == 0 for v in cols.values())


def _golden(tmp_path):
    """cli_dataset1 as a real BAM: (bam, the records' SA values in BAM order, parsed arguments)."""
    bamio.build()
    d = str(tmp_path)
    gold = json.load(open(os.path.join(golden_util.GOLDEN, "cli_dataset1.json")))
    pk_path, fa, out, wd = gen_cli_golden.materialise(d)
    ds = pickle.load(open(pk_path, "rb"))
    order = {n: i for i, (n, _) in enumerate(ds["contigs"])}
    reads = sorted(ds["reads"], key=lambda r: (order[r.reference_name], r.reference_start))
    bam = os.path.join(d, "real.bam")
    bam_writer.write_bam(bam, ds["contigs"], reads, extra_unmapped=2)   # unplaced records never reach a packet
    return bam, [dict(r.get_tags()).get("SA") for r in reads], cli.build_parser().parse_args([bam, fa, out, wd] + gold["flags"])


def _text_packet(dev, values):
    out = {k: v for k, v in dev.items() if k not in ("sa", "sa_off")}
    text, off = sat.text_arrays(values, lead=3)
    out["sa_text"], out["sa_text_off"] = _cuda(text), _cuda(off)
    return out


def _run(engine, bam, values, args, max_split_parts, scan, text):
    p = cli.params_from_args(args)
    p.max_split_parts = max_split_parts
    engine.set_params(p)
    rd = bamio.BamReader(bam, threads=2)
    lens = dict((n, rd.get_reference_length(n)) for n, _ in rd.index_statistics())
    rd.close()
    names = sorted(lens)
    engine.set_contigs(np.array([lens[n] for n in names], np.int64), names=names)
    engine.extract_reset()
    o = 0
    for pk, rnames in _packets(bam, {n: i for i, n in enumerate(names)}, 700):
        dev = name_util.named(dpu.to_device(pk), rnames)
        if text:
            dev = _text_packet(dev, values[o:o + len(rnames)])
        o += len(rnames)
        if scan:
            engine.scan(dev, alignments=True)
        else:
            engine.extract(dev, append=True)
    assert o == len(values)
    state = _state(engine)
    engine.rank_names()
    engine.order_ins_ties()
    aln = engine.fetch_alignments() if scan else None
    engine.cluster_device(0x1F)
    cands, genos, nbuf = engine.fetch()
    return state, aln, (cands.copy(), genos.copy(), nbuf.copy())


@pytest.mark.parametrize("max_split_parts", [7, -1])
@pytest.mark.parametrize("scan", [False, True])
def test_text_packets_equal_column_packets(engine, tmp_path, max_split_parts, scan):
    bam, values, args = _golden(tmp_path)
    assert args.genotype and sum(v is not None for v in values) >= 20
    want = _run(engine, bam, values, args, max_split_parts, scan, False)
    got = _run(engine, bam, values, args, max_split_parts, scan, True)
    assert got[0] == want[0]   # signatures, reads rows and INS sequences
    if scan:
        for k in _abi.READS_FIELDS:
            assert np.array_equal(got[1][k], want[1][k]), k
    assert len(want[2][0]) > 0
    _same_records(got[2], want[2])


def test_many_contig_names(engine):
    n = 100_000
    names = ["ctg%d" % k for k in range(n)]   # not in byte order: the library sorts them
    engine.set_contigs(np.full(n, 10_000, np.int64), names=names)
    pick = list(range(0, n, 997)) + [n - 1, 10, 1]
    values = ["".join("%s,%d,-,3S5M,9,0;" % (names[k], k) for k in pick[:20]), None] + ["%s,1,+,5M,1,0;" % names[k] for k in pick[20:]]
    values += ["ctg100000,1,+,5M,1,0;ctg,1,+,5M,1,0;ctg1x,1,+,5M,1,0;ctg0,1,+,5M,1,0;"]
    off, cols = _reduce(engine, values)
    assert cols["chrom"].tolist() == pick + [-1, -1, -1, 0]
    assert cols["pos0"][:20].tolist() == [k - 1 for k in pick[:20]] and off[:3].tolist() == [0, 20, 20]


def _rejected(code, fn, match=None):
    with pytest.raises(_lib.CuteSVError, match=match) as e:
        fn()
    assert e.value.code == code


def test_contig_name_table_rejections(engine):
    engine.set_contigs(np.array([100, 200, 300], np.int64), names=["a", "b", "c"])
    ok = _reduce(engine, ["b,1,+,5M,1,0;c,1,+,5M,1,0;"])
    for bad in (["a", "b"], ["a", "b", "a"], ["a", "", "c"], ["a", "b\0", "c"]):
        _rejected(_abi.CSV_E_INVALID, lambda: engine.set_contigs(np.array([100, 200, 300], np.int64), names=bad))
    _assert_equal(_reduce(engine, ["b,1,+,5M,1,0;c,1,+,5M,1,0;"]), ok)   # the table is the one set last
    engine.set_contigs(np.array([100, 200, 300], np.int64))   # same count: the names stay
    assert _reduce(engine, ["c,1,+,5M,1,0;"])[1]["chrom"].tolist() == [2]
    engine.set_contigs(np.array([100, 200], np.int64))   # another count drops them
    _rejected(_abi.CSV_E_STATE, lambda: _reduce(engine, ["a,1,+,5M,1,0;"]))
    fresh = Engine(0, contig_lens=[1000])
    try:
        _rejected(_abi.CSV_E_STATE, lambda: _reduce(fresh, ["a,1,+,5M,1,0;"]), "csv_set_contig_names")
    finally:
        fresh.close()


def test_rejections_change_nothing(engine, tmp_path):
    import ctypes as C
    bam, values, args = _golden(tmp_path)
    rd = bamio.BamReader(bam, threads=2)
    lens = dict((n, rd.get_reference_length(n)) for n, _ in rd.index_statistics())
    rd.close()
    names = sorted(lens)
    engine.set_params(cli.params_from_args(args))
    engine.set_contigs(np.array([lens[n] for n in names], np.int64), names=names)
    (p0, n0), (p1, n1) = _packets(bam, {n: i for i, n in enumerate(names)}, 700)[:2]
    engine.extract_reset()
    engine.scan(_text_packet(name_util.named(dpu.to_device(p0), n0), values[:len(n0)]), alignments=True)
    state = _state(engine)
    good = _text_packet(name_util.named(dpu.to_device(p1), n1), values[len(n0):len(n0) + len(n1)])
    # the outputs of a successful reduction stay as they were through every failed call
    sa_off, cols = engine.reduce_sa(good["sa_text"], good["sa_text_off"])
    kept = (sa_off.clone(), {f: v.clone() for f, v in cols.items()})

    def unchanged():
        assert _state(engine) == state
        assert sa_off.equal(kept[0]) and all(cols[f].equal(kept[1][f]) for f in _abi.SA_FIELDS)
    text, off = good["sa_text"], good["sa_text_off"]
    for k, v in ((0, -1), (5, int(off[4]) - 1), (len(off) - 1, len(text) + 1)):
        bad = off.clone()
        bad[k] = v
        _rejected(_abi.CSV_E_INPUT, lambda: engine.reduce_sa(text, bad), "text_off")
        _rejected(_abi.CSV_E_INPUT, lambda: engine.scan(dict(good, sa_text_off=bad), alignments=True), "text_off")
        unchanged()
    for value, col in (("chr1,2147483648,+,5M,1,0;", "sa.pos0"), ("chr1,-2147483648,+,5M,1,0;", "sa.pos0"), ("chr1,1,+,5M,2147483648,0;", "sa.mapq"),
                       ("chr1,1,+,2147483648S,1,0;", "sa.first_clip"), ("chr1,1,+,2000000000M2000000000D,1,0;", "sa.ref_span")):
        t, o = sat.text_arrays(values[len(n0):len(n0) + len(n1) - 1] + [value])
        _rejected(_abi.CSV_E_INPUT, lambda: engine.reduce_sa(_cuda(t), _cuda(o)), col)
        _rejected(_abi.CSV_E_INPUT, lambda: engine.scan(dict(good, sa_text=_cuda(t), sa_text_off=_cuda(o)), alignments=True), col)
        unchanged()
    # host memory
    t, o = sat.text_arrays(["chr1,1,+,5M,1,0;"])
    h = _abi.csv_sa_text(1, len(t), o.ctypes.data_as(C.POINTER(C.c_int64)), t.ctypes.data_as(C.POINTER(C.c_uint8)))
    rc = engine.L.csv_reduce_sa_device(engine.h, C.byref(h), None, C.byref(C.POINTER(C.c_int64)()), C.byref(_abi.csv_sa_cols()))
    assert rc == _abi.CSV_E_INVALID
    unchanged()
    # and the accumulation goes on with the good packet
    engine.scan(good, alignments=True)
    engine.rank_names()
