"""-m gpu: scanned packets (Engine.scan / csv_scan_append_named_device).  Every decoded record of a BAM packet goes to the library,
which applies the reference's record filter and -include_bed test and builds the TRA genotyper's alignment table on the device.
Against the host filter followed by the named device extraction, the CLI's own alignment table and records (native source), and
the reference's VCFs."""
import collections
import json
import os

import numpy as np
import pytest

import bam_writer
import device_packet_util as dpu
import golden_util
import name_util
import vcf_util
from cutesv_b200 import _abi, _lib, bamio, cli, rows, vcf
from oracle import compare_records, gen_cli_golden, gen_cli_golden_draft
from test_gpu_device_extract import _canon, _dev_strings, _to_real_bam

pytestmark = pytest.mark.gpu
INS = _abi.CSV_INS


@pytest.fixture(autouse=True)
def _no_table_left(engine):
    """Later tests on the shared engine see no region table and no alignment table from these."""
    yield
    engine.extract_reset()
    engine.set_scan_regions([], None, {})
    engine.upload_alignments(None)


def _materialise(tmp_path, golden):
    """(bam, reference, output, work dir, argv, golden lines) of a CLI golden, written as a real BAM."""
    bamio.build()
    d = str(tmp_path)
    gold = json.load(open(os.path.join(golden_util.GOLDEN, golden + ".json")))
    extra = []
    if golden == "cli_draft_40k":
        _, fa, out, wd, ds = gen_cli_golden_draft.materialise(d)
        order = {n: i for i, (n, _) in enumerate(ds["contigs"])}
        bam = os.path.join(d, "real.bam")
        bam_writer.write_bam(bam, ds["contigs"], sorted(ds["reads"], key=lambda r: (order[r.reference_name], r.reference_start)), extra_unmapped=1)
        extra = ["-include_bed", gen_cli_golden_draft.write_bed(d, ds)]
    else:
        if golden == "cli_config1":
            pk, fa, out, wd = gen_cli_golden.materialise_config1(d)
        elif golden == "cli_dataset2_ins_ties":
            pk, fa, out, wd = gen_cli_golden.materialise(d, gold["seed"], gold["double_ins"])
        else:
            pk, fa, out, wd = gen_cli_golden.materialise(d)
        bam = _to_real_bam(pk, os.path.join(d, "real.bam"))
        if golden == "cli_dataset1_bed":
            extra = ["-include_bed", gen_cli_golden.write_bed(d)]
    return bam, fa, out, wd, [bam, fa, out, wd] + gold["flags"] + extra, gold["lines"]


def _layout(rd, args):
    """The CLI's task windows, regions and contig ids for this BAM."""
    stats = rd.index_statistics()
    tasks, contig_info = cli.task_windows(stats, rd.get_reference_length, args.threads, args.batches)
    chrom_names = sorted(c[0] for c in contig_info)
    return tasks, cli.load_bed(args.include_bed, tasks), contig_info, chrom_names, {n: i for i, n in enumerate(chrom_names)}


def _packets(bam, chrom_id, size):
    """(decoded packet, record names) of the whole BAM in packets of `size` records."""
    rd = bamio.BamReader(bam, threads=2)
    rd.set_chrom_ids(chrom_id)
    out = []
    while True:
        pk = rd.next_packet(size)
        if pk is None:
            break
        names = rd.names()
        out.append((pk, [names[i] for i in pk["read_id"].tolist()]))
    rd.close()
    return out


def _scan_run(engine, bam, args, size=cli.PACKET_READS):
    """Every record through Engine.scan, ranks and ties on the device, csv_cluster.  Returns (records, alignment table, layout)."""
    rd = bamio.BamReader(bam, threads=2)
    tasks, bed, contig_info, chrom_names, chrom_id = _layout(rd, args)
    rd.close()
    engine.set_params(cli.params_from_args(args))
    engine.set_contigs(np.array([dict(contig_info)[n] for n in chrom_names], dtype=np.int64))
    engine.extract_reset()
    engine.set_scan_regions(tasks, bed, chrom_id)
    for pk, names in _packets(bam, chrom_id, size):
        engine.scan(name_util.named(dpu.to_device(pk), names), alignments=bool(args.genotype))
    engine.rank_names()
    engine.order_ins_ties()
    aln = engine.fetch_alignments()
    engine.cluster_device(0x1F)
    cands, genos, nbuf = engine.fetch()
    return (cands.copy(), genos.copy(), nbuf.copy()), aln, (contig_info, chrom_names)


def _write_vcf(engine, records, layout, args, argv, fa, out):
    cands, genos, nbuf = records
    contig_info, chrom_names = layout
    ids = np.unique(nbuf).astype(np.int32)
    name_of = dict(zip(ids.tolist(), engine.fetch_names(ids)))
    emitted = np.unique(cands["aux"][cands["svtype"] == INS]).astype(np.int64)
    seq_of = dict(zip(emitted.tolist(), engine.fetch_ins_seqs(emitted)))
    got = rows.records_to_rows(cands, genos, nbuf, chrom_names, name_of.__getitem__, seq_of.__getitem__, bool(args.genotype))
    results = {}
    for t in _abi.TYPE_NAMES:
        for (tt, chrom), r in got.items():
            if tt == t:
                results.setdefault(chrom, []).extend(r)
    ref = vcf.IndexedFasta(fa)
    vcf.write_vcf(out, results, ref, contig_info, args.sample, argv, dict(genotype=args.genotype, max_size=args.max_size, min_size=args.min_size,
                                                                          report_readid=args.report_readid, ignore_sequence=args.ignore_sequence))
    ref.close()
    return [l for l in open(out) if not l.startswith("##")]


def _cli_run(engine, argv):
    """cli.main_ctrl (native source) on the engine; returns the records and the alignment table it handed to the library."""
    seen = {}
    fetch, upload = engine.fetch, engine.upload_alignments

    def spy_fetch(out=None):
        r = fetch(out)
        seen.setdefault("records", tuple(x.copy() for x in r))
        return r

    def spy_upload(aln, stream=None):
        seen.setdefault("aln", aln)
        return upload(aln, stream)
    engine.fetch, engine.upload_alignments = spy_fetch, spy_upload
    try:
        cli.main_ctrl(cli.build_parser().parse_args(argv), argv, engine=engine)
    finally:
        del engine.fetch, engine.upload_alignments
    return seen["records"], seen.get("aln")


def _same_records(a, b):
    """Equal records up to layout (compare_records.diff_records).  An INS record's aux is the row of its sequence, and rows are
    handed out by atomics during extraction, so it is left out here; the VCFs compare the sequences."""
    def masked(r):
        c = r[0].copy()
        c["aux"][c["svtype"] == INS] = 0
        return (c,) + tuple(r[1:])
    assert not compare_records.diff_records(masked(b), masked(a))


@pytest.mark.parametrize("golden", ["cli_dataset1", "cli_dataset1_bed", "cli_config1", "cli_draft_40k", "cli_dataset2_ins_ties"])
def test_scan_records_alignments_and_vcf_equal_the_cli(engine, tmp_path, golden):
    bam, fa, out, wd, argv, gold = _materialise(tmp_path, golden)
    cli_records, cli_aln = _cli_run(engine, argv)
    args = cli.build_parser().parse_args(argv)
    records, aln, layout = _scan_run(engine, bam, args)
    assert cli_aln is not None and aln is not None and len(aln["chrom"]) > 0
    for k in _abi.READS_FIELDS:   # same rows, order and ids
        assert np.array_equal(aln[k], np.asarray(cli_aln[k])), (k, len(aln[k]), len(cli_aln[k]), aln[k][:8], np.asarray(cli_aln[k])[:8])
    _same_records(records, cli_records)
    lines = _write_vcf(engine, records, layout, args, argv, fa, str(tmp_path / "scan.vcf"))
    assert len(lines) > 5
    if golden == "cli_dataset2_ins_ties":
        assert vcf_util.normalise_rnames(lines) == vcf_util.normalise_rnames(gold)
    else:
        assert lines == gold


# ---- extraction of one scanned packet equals the host filter + the named device extraction ----

def _host_keep(pk, bed, starts, first_task):
    has_cigar = pk["cigar_off"][1:] > pk["cigar_off"][:-1]
    keep = has_cigar & (pk["flag"] != 256) & (pk["flag"] != 272) & (pk["chrom"] >= 0)
    if bed is not None:
        cli.bed_filter(pk, keep, bed, starts, first_task)
    return np.flatnonzero(keep)


def _state(engine, rec_of=None):
    """The extraction's output as multisets, read ids and piece records mapped through rec_of (a subset packet's index -> scanned
    index); INS rows carry their device-built string and their pieces."""
    ex = engine.fetch_extracted()
    m = (lambda a: np.asarray(a)) if rec_of is None else (lambda a: rec_of[np.asarray(a, dtype=np.int64)])
    for s in ex["sigs"].values():
        s["read_id"] = m(s["read_id"])
    ex["rows"]["read_id"] = m(ex["rows"]["read_id"])
    pieces = ex["pieces"].copy()
    if len(pieces):
        pieces[:, 0] = m(pieces[:, 0])
    seqs = _dev_strings(engine)
    s = ex["sigs"]["INS"]
    ins = collections.Counter((tuple(int(s[k][i]) for k in ("chrom", "a", "b", "read_id", "c")), seqs[i],
                               tuple(map(tuple, pieces[ex["piece_off"][i]:ex["piece_off"][i] + ex["piece_cnt"][i]].tolist())))
                              for i in range(len(s["chrom"])))
    return _canon(ex), ins


@pytest.mark.parametrize("golden", ["cli_dataset1", "cli_dataset1_bed"])
def test_every_packet_equals_host_filter_then_named_extraction(engine, tmp_path, golden):
    bam, fa, out, wd, argv, gold = _materialise(tmp_path, golden)
    args = cli.build_parser().parse_args(argv)
    rd = bamio.BamReader(bam, threads=2)
    tasks, bed, contig_info, chrom_names, chrom_id = _layout(rd, args)
    rd.close()
    engine.set_params(cli.params_from_args(args))
    engine.set_contigs(np.array([dict(contig_info)[n] for n in chrom_names], dtype=np.int64))
    engine.set_scan_regions(tasks, bed, chrom_id)
    starts, first_task = cli.window_starts(tasks, chrom_id)
    packets = _packets(bam, chrom_id, 300)
    assert len(packets) > 2
    n_filtered = 0
    for pk, names in packets:
        # secondaries to drop (256, 272) and one that stays (256 | 1024: the reference tests exact values)
        pk = dict(pk, flag=pk["flag"].copy())
        pk["flag"][::5], pk["flag"][1::7], pk["flag"][2::11] = 256, 272, 256 | 1024
        keep = _host_keep(pk, bed, starts, first_task)
        n_filtered += len(names) - len(keep)
        engine.extract_reset()
        engine.scan(name_util.named(dpu.to_device(pk), names))
        got = _state(engine)
        engine.extract_reset()
        sub = dpu.flat_seq(bamio.subset_packet(pk, keep))
        engine.extract(name_util.named(dpu.to_device(sub), [names[i] for i in keep.tolist()]), append=True)
        assert got == _state(engine, keep)
    assert n_filtered > 0


# ---- packet sizes, filtered names ----

def _straddling_bed(tmp_path, tasks):
    """Regions around every second window border (they straddle it) and one inside each first window."""
    lines = []
    for i, t in enumerate(tasks):
        if i % 2 and t[1] > 0:
            lines.append("%s\t%d\t%d\n" % (t[0], int(t[1]) - 3000, int(t[1]) + 3000))
        elif t[1] == 0:
            lines.append("%s\t%d\t%d\n" % (t[0], 100, 5000))
    p = tmp_path / "straddle.bed"
    p.write_text("".join(lines))
    return str(p)


def test_packet_sizes_give_identical_records(engine, tmp_path):
    bam, fa, out, wd, argv, gold = _materialise(tmp_path, "cli_dataset1")
    argv = argv[:4] + ["-b", "40000"] + argv[4:]   # many windows per contig
    rd = bamio.BamReader(bam, threads=2)
    tasks, _, _, _, _ = _layout(rd, cli.build_parser().parse_args(argv))
    rd.close()
    assert len(tasks) > 4
    args = cli.build_parser().parse_args(argv + ["-include_bed", _straddling_bed(tmp_path, tasks)])
    got = {}
    for size in (50_000, 7, 1):
        records, aln, _ = _scan_run(engine, bam, args, size)
        got[size] = (records, aln)
    cli_records, cli_aln = _cli_run(engine, [bam, fa, str(tmp_path / "cli.vcf"), wd] + argv[4:] + ["-include_bed", args.include_bed])
    for size in (50_000, 7, 1):
        _same_records(got[size][0], cli_records)
        for k in _abi.READS_FIELDS:
            assert np.array_equal(got[size][1][k], np.asarray(cli_aln[k]))
    assert len(cli_records[0]) > 0


def test_reads_seen_only_in_filtered_records_get_ranks_and_alignment_rows(engine, tmp_path):
    bam, fa, out, wd, argv, gold = _materialise(tmp_path, "cli_dataset1_bed")
    args = cli.build_parser().parse_args(argv)
    rd = bamio.BamReader(bam, threads=2)
    tasks, bed, contig_info, chrom_names, chrom_id = _layout(rd, args)
    rd.close()
    starts, first_task = cli.window_starts(tasks, chrom_id)
    (pk, names), = _packets(bam, chrom_id, 10 ** 6)
    keep = np.zeros(len(names), bool)
    keep[_host_keep(pk, bed, starts, first_task)] = True
    ok = (pk["cigar_off"][1:] > pk["cigar_off"][:-1]) & (pk["chrom"] >= 0) & (pk["flag"] != 256) & (pk["flag"] != 272)
    outside = int(np.flatnonzero(ok & ~keep)[0])            # dropped by the BED test alone
    secondary = int(np.flatnonzero(keep)[0])                # made secondary below
    pk = dict(pk, flag=pk["flag"].copy())
    pk["flag"][secondary] = 256
    names = list(names)
    names[outside], names[secondary] = "read_outside_every_region", "read_with_only_a_secondary"
    engine.set_params(cli.params_from_args(args))
    engine.set_contigs(np.array([dict(contig_info)[n] for n in chrom_names], dtype=np.int64))
    engine.extract_reset()
    engine.set_scan_regions(tasks, bed, chrom_id)
    engine.scan(name_util.named(dpu.to_device(pk), names), alignments=True)
    nd = engine.rank_names()
    assert nd == len(set(names))
    rank = engine.name_rank_tensor().cpu().numpy()
    aln = engine.fetch_alignments()
    for rec in (outside, secondary):
        r = int(rank[rec])
        assert engine.fetch_names([r]) == [names[rec]]
        row = np.flatnonzero(aln["read_id"] == r)
        assert len(row) == 1
        assert (aln["chrom"][row[0]], aln["start"][row[0]], aln["end"][row[0]]) == (pk["chrom"][rec], pk["ref_start"][rec], pk["ref_end"][rec])
        assert aln["is_primary"][row[0]] == (0 if rec == secondary else int(pk["flag"][rec] in (0, 16)))
    # neither name reaches an extracted row
    ex = engine.fetch_extracted()
    ids = np.concatenate([s["read_id"] for s in ex["sigs"].values()] + [ex["rows"]["read_id"]])
    assert not np.isin([rank[outside], rank[secondary]], ids).any()


# ---- rejections, stream order ----

def _setup_small(engine, tmp_path):
    bam, fa, out, wd, argv, gold = _materialise(tmp_path, "cli_dataset1_bed")
    args = cli.build_parser().parse_args(argv)
    rd = bamio.BamReader(bam, threads=2)
    tasks, bed, contig_info, chrom_names, chrom_id = _layout(rd, args)
    rd.close()
    engine.set_params(cli.params_from_args(args))
    engine.set_contigs(np.array([dict(contig_info)[n] for n in chrom_names], dtype=np.int64))
    engine.extract_reset()
    engine.set_scan_regions(tasks, bed, chrom_id)
    return _packets(bam, chrom_id, 700), (tasks, bed, chrom_id)


def _snapshot(engine):
    return _state(engine)


def test_rejections_change_nothing(engine, tmp_path):
    packets, layout = _setup_small(engine, tmp_path)
    (p0, n0), (p1, n1) = packets[0], packets[1]
    good1 = name_util.named(dpu.to_device(p1), n1)

    def first():
        engine.extract_reset()
        engine.scan(name_util.named(dpu.to_device(p0), n0), alignments=True)
        return _snapshot(engine)

    state = first()
    bad = dict(good1, cigar_off=good1["cigar_off"].clone())
    bad["cigar_off"][3] = bad["cigar_off"][2] - 1
    bad_names = dict(good1, name_off=good1["name_off"].clone())
    bad_names["name_off"][-1] = len(good1["names"]) + 1
    for b in (bad, bad_names):
        with pytest.raises(_lib.CuteSVError) as e:
            engine.scan(b, alignments=True)
        assert e.value.code == _abi.CSV_E_INPUT
        assert _snapshot(engine) == state
    # other packet kinds, a different alignments choice, a region change while the accumulation is open
    for call in (lambda: engine.extract(good1, append=True), lambda: engine.scan(good1, alignments=False),
                 lambda: engine.set_scan_regions(*layout), lambda: engine.set_scan_regions([], None, {})):
        with pytest.raises(_lib.CuteSVError) as e:
            call()
        assert e.value.code == _abi.CSV_E_STATE
        assert _snapshot(engine) == state
    with pytest.raises(ValueError, match="names"):
        engine.scan(dpu.to_device(p1))
    engine.extract_reset()
    engine.extract(good1, append=True)
    with pytest.raises(_lib.CuteSVError) as e:   # a scanned packet cannot join a named extraction
        engine.scan(name_util.named(dpu.to_device(p0), n0))
    assert e.value.code == _abi.CSV_E_STATE
    # the accumulation is still usable; no append after the ranking
    first()
    engine.scan(good1, alignments=True)
    want = _snapshot(engine)
    engine.rank_names()
    ranked = _snapshot(engine)
    with pytest.raises(_lib.CuteSVError) as e:
        engine.scan(good1, alignments=True)
    assert e.value.code == _abi.CSV_E_STATE
    assert _snapshot(engine) == ranked
    engine.set_scan_regions(*layout)   # allowed again once ranked
    # an alignment stream out of BAM order: rank_names refuses it and the ids stay provisional
    first()
    rs = p1["ref_start"].copy()
    rows_ = np.flatnonzero((p1["cigar_off"][1:] > p1["cigar_off"][:-1]) & (p1["chrom"] >= 0))
    k = int(np.flatnonzero(p1["chrom"][rows_[1:]] == p1["chrom"][rows_[:-1]])[0])
    rs[rows_[k]] = rs[rows_[k + 1]] + 10   # an alignment row starting after its successor on the same contig
    engine.scan(name_util.named(dpu.to_device(dict(p1, ref_start=rs)), n1), alignments=True)
    before = _snapshot(engine)
    with pytest.raises(_lib.CuteSVError, match="BAM order") as e:
        engine.rank_names()
    assert e.value.code == _abi.CSV_E_INPUT
    assert _snapshot(engine) == before and engine.fetch_alignments() is None
    with pytest.raises(_lib.CuteSVError):
        engine.name_rank_tensor()
    # and a correct run on the same engine
    first()
    engine.scan(good1, alignments=True)
    engine.rank_names()
    assert _snapshot(engine) == ranked


def test_stream_order_and_overwrite_after_return(engine, tmp_path):
    import torch
    packets, _ = _setup_small(engine, tmp_path)
    pk, names = packets[0]
    engine.scan(name_util.named(dpu.to_device(pk), names), alignments=True)
    engine.rank_names()
    ref, ref_aln = _snapshot(engine), engine.fetch_alignments()
    staged = name_util.named(dpu.to_device(pk), names)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)   # the packet's final tensors are written late on the side stream
        d = {k: ({kk: vv.clone() for kk, vv in v.items()} if isinstance(v, dict) else v.clone()) for k, v in staged.items()}
    assert not side.query()
    engine.extract_reset()
    engine.scan(d, alignments=True, stream=side)
    with torch.cuda.stream(side):   # overwritten in the side stream's order right after the call returns
        for k, v in d.items():
            for t in (v.values() if isinstance(v, dict) else [v]):
                t.fill_(7)
    engine.rank_names()
    assert _snapshot(engine) == ref
    got = engine.fetch_alignments()
    assert all(np.array_equal(got[k], ref_aln[k]) for k in _abi.READS_FIELDS)
