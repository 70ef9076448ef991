"""-m gpu: extraction from alignment records in GPU memory (csv_extract*_device through Engine.extract with torch CUDA packets), INS
sequences built on the device.  Against the REAL reference's parse_read tuples, the host path on the same records, and the
reference's own VCFs end to end."""
import collections
import ctypes as C
import json
import os

import numpy as np
import pytest

import bam_writer
import device_packet_util as dpu
import golden_util
from cutesv_b200 import _abi, _lib, bamio, cli, packing, rows, synth, vcf
from oracle import compare_extract, gen_cli_golden

pytestmark = pytest.mark.gpu
INS = _abi.CSV_INS


def _packet(seed, n=300, kind="short"):
    reads, names, lens = synth.synth_alignments_long(seed, n) if kind == "long" else synth.synth_alignments(seed, n)
    rnames = sorted(set(r.query_name for r in reads))
    pk = packing.pack_alignments(reads, {nm: i for i, nm in enumerate(names)}, {nm: i for i, nm in enumerate(rnames)})
    return reads, names, lens, rnames, dpu.with_bases(pk, [r.query_sequence for r in reads])


def _host(pk):
    return {k: v for k, v in pk.items() if k not in ("seq_off", "seq4")}


def _dev_strings(engine):
    n = engine._ex_counts[INS]
    return engine.fetch_ins_seqs(np.arange(n))


def _ins_rows_with_seq(ex, seqs):
    s = ex["sigs"]["INS"]
    return collections.Counter(zip(s["chrom"].tolist(), s["a"].tolist(), s["b"].tolist(), s["read_id"].tolist(), s["c"].tolist(), seqs))


def _canon(ex):
    out = {}
    for t, cols in ex["sigs"].items():
        out[t] = collections.Counter(zip(*[cols[k].tolist() for k in ("chrom", "a", "b", "read_id", "c")]))
    r = ex["rows"]
    out["rows"] = collections.Counter(zip(r["chrom"].tolist(), r["start"].tolist(), r["end"].tolist(), r["read_id"].tolist(), r["is_primary"].tolist()))
    return out


@pytest.mark.parametrize("name", ["extract_s0", "extract_s1", "extract_s2", "extract_s3", "extract_s4", "extract_s5", "extract_s6",
                                  "extract_l0", "extract_l1", "extract_l2", "extract_l3", "extract_l4"])
def test_device_packet_matches_reference_golden(engine, name):
    meta = json.load(open(os.path.join(golden_util.GOLDEN, name + ".json")))
    reads, names, lens, rnames, pk = _packet(meta["seed"], meta["n_reads"], meta.get("kind", "short"))
    p = _abi.default_params(**meta["params"])
    engine.set_params(p)
    engine.set_contigs(lens)
    engine.extract(dpu.to_device(pk))
    got = engine.fetch_extracted()
    gc, gr = compare_extract.tuples_from_columns(got, names, rnames, lambda rec: reads[rec].query_sequence, dpu.cigar_of_packet(pk),
                                                 (p.min_siglength, p.merge_ins_threshold))
    seqs = _dev_strings(engine)
    gc = dict(gc, INS=[t[:3] + (s,) + t[4:] for t, s in zip(gc["INS"], seqs)])   # the device-built strings, row by row
    ref_c = {k: [tuple(t) for t in v] for k, v in meta["candidate"].items()}
    assert not compare_extract.diff_extract(ref_c, [tuple(t) for t in meta["rows"]], gc, gr)


@pytest.mark.parametrize("seed", range(12))
def test_device_packet_matches_host_packet(engine, seed):
    reads, names, lens, rnames, pk = _packet(seed)
    rng = np.random.default_rng(seed)
    p = _abi.default_params(min_size=int(rng.choice([30, 50, 10])), max_size=int(rng.choice([-1, 100000, 2000])),
                            min_mapq=int(rng.choice([20, 0, 30])), max_split_parts=int(rng.choice([7, -1, 2, 3])),
                            min_read_len=int(rng.choice([500, 100])), min_siglength=int(rng.choice([10, 30])),
                            merge_del_threshold=int(rng.choice([0, 500])), merge_ins_threshold=int(rng.choice([100, 500, 0])))
    engine.set_params(p)
    engine.set_contigs(lens)
    engine.extract(_host(pk))
    host = engine.fetch_extracted()
    host_seqs = dpu.host_ins_strings(host, lambda rec: reads[rec].query_sequence, dpu.cigar_of_packet(pk), (p.min_siglength, p.merge_ins_threshold))
    engine.extract(dpu.to_device(pk))
    dev = engine.fetch_extracted()
    assert _canon(dev) == _canon(host)
    assert _ins_rows_with_seq(dev, _dev_strings(engine)) == _ins_rows_with_seq(host, host_seqs)
    assert engine.extract_skipped() == 0 or p.max_split_parts == -1


def _slice(pk, lo, hi):
    out = {k: pk[k][lo:hi] for k in _abi.READ_FIELDS}
    c0, c1, s0, s1, b0, b1 = (int(pk[k][i]) for k, i in (("cigar_off", lo), ("cigar_off", hi), ("sa_off", lo), ("sa_off", hi), ("seq_off", lo), ("seq_off", hi)))
    out["cigar_off"], out["sa_off"], out["seq_off"] = pk["cigar_off"][lo:hi + 1] - c0, pk["sa_off"][lo:hi + 1] - s0, pk["seq_off"][lo:hi + 1] - b0
    out["cigar"], out["seq4"] = pk["cigar"][c0:c1], pk["seq4"][b0:b1]
    out["sa"] = {k: v[s0:s1] for k, v in pk["sa"].items()}
    return out


def _setup(engine, seed=3, n=400):
    reads, names, lens, rnames, pk = _packet(seed, n)
    engine.set_params(_abi.default_params(min_support=2, genotype=1, min_mapq=0, min_read_len=100))
    engine.set_contigs(lens)
    return reads, pk


@pytest.mark.parametrize("cuts", [(0, 97, 98, 250, 400), (0, 0, 1, 399, 400)])
def test_append_ragged_device_packets_equal_one_call(engine, cuts):
    reads, pk = _setup(engine)
    engine.extract(dpu.to_device(pk))
    one, one_seqs = engine.fetch_extracted(), _dev_strings(engine)
    engine.extract_reset()
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        engine.extract(dpu.to_device(_slice(pk, lo, hi)), append=True)
    many = engine.fetch_extracted()
    assert _canon(many) == _canon(one)
    assert _ins_rows_with_seq(many, _dev_strings(engine)) == _ins_rows_with_seq(one, one_seqs)
    b, s, ln = engine.ins_seq_tensors()
    b, s, ln = b.cpu().numpy(), s.cpu().numpy(), ln.cpu().numpy()
    assert [b[x:x + y].tobytes().decode() for x, y in zip(s.tolist(), ln.tolist())] == _dev_strings(engine)


def test_mixed_device_and_host_packets(engine):
    reads, pk = _setup(engine)
    engine.extract(_host(pk))
    ref = engine.fetch_extracted()
    engine.extract_reset()
    engine.extract(dpu.to_device(_slice(pk, 0, 150)), append=True)
    engine.extract(_host(_slice(pk, 150, 300)), append=True)
    engine.extract(dpu.to_device(_slice(pk, 300, 400)), append=True)
    assert _canon(engine.fetch_extracted()) == _canon(ref)
    with pytest.raises(_lib.CuteSVError) as e:
        engine.fetch_ins_seqs([0])
    assert e.value.code == _abi.CSV_E_STATE
    with pytest.raises(_lib.CuteSVError) as e:
        engine.ins_seq_tensors()
    assert e.value.code == _abi.CSV_E_STATE


def _records(engine):
    out = {}
    for t, name in enumerate(_abi.TYPE_NAMES):
        ex = engine.fetch_sig_cols(name)
        rec = engine.fetch_records(name)
        out[name] = collections.Counter(zip(*[ex[k].tolist() for k in ("chrom", "a", "b", "read_id")], rec.tolist()))
    r = engine.fetch_read_rows()
    out["reads"] = collections.Counter(zip(r["chrom"].tolist(), r["start"].tolist(), r["read_id"].tolist(), engine.fetch_records("reads").tolist()))
    return out


def test_record_column_matches_host_path(engine):
    reads, pk = _setup(engine, 8)
    engine.set_extract_records(True)
    try:
        engine.extract_reset()
        for lo, hi in ((0, 200), (200, 400)):
            engine.extract(_host(_slice(pk, lo, hi)), append=True)
        host = _records(engine)
        engine.extract_reset()
        for lo, hi in ((0, 200), (200, 400)):
            engine.extract(dpu.to_device(_slice(pk, lo, hi)), append=True)
        assert _records(engine) == host
    finally:
        engine.set_extract_records(False)


def test_remap_and_swap_keep_strings_attached(engine):
    reads, pk = _setup(engine, 2, 300)
    engine.extract(dpu.to_device(pk))
    before = engine.fetch_extracted()
    seqs = _dev_strings(engine)
    n_ids = int(max(max(int(v["read_id"].max()) for v in before["sigs"].values() if len(v["read_id"])), before["rows"]["read_id"].max())) + 1
    engine.remap_read_ids(np.random.default_rng(1).permutation(n_ids).astype(np.int32))
    assert _dev_strings(engine) == seqs
    n = len(seqs)
    assert n >= 3
    engine.swap_ins_rows([(0, 2), (2, 1)])
    perm = [2, 0, 1] + list(range(3, n))
    assert _dev_strings(engine) == [seqs[i] for i in perm]
    assert engine.fetch_ins_seqs([1, 1, 0]) == [seqs[0], seqs[0], seqs[2]]


def test_stream_order_and_overwrite_after_return(engine):
    import torch
    reads, pk = _setup(engine, 11)
    engine.extract(_host(pk))
    ref = engine.fetch_extracted()
    ref_seqs = dpu.host_ins_strings(ref, lambda rec: reads[rec].query_sequence, dpu.cigar_of_packet(pk), (10, 100))
    staged = dpu.to_device(pk)   # on the device first: the side stream below only runs device work, so the host never waits for it
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)   # the packet's final tensors are written late, device to device, on the side stream
        d = {k: ({kk: vv.clone() for kk, vv in v.items()} if isinstance(v, dict) else v.clone()) for k, v in staged.items()}
    assert not side.query()   # the copies are still pending when the call is made
    engine.extract(d, stream=side)
    with torch.cuda.stream(side):   # overwritten in the side stream's order right after the call returns
        for k, v in d.items():
            for t in (v.values() if isinstance(v, dict) else [v]):
                t.fill_(7)
    got = engine.fetch_extracted()
    assert _canon(got) == _canon(ref)
    assert _ins_rows_with_seq(got, _dev_strings(engine)) == _ins_rows_with_seq(ref, ref_seqs)


def test_rejections_leave_the_accumulation_intact(engine):
    import torch
    reads, pk = _setup(engine, 5, 200)
    engine.extract(dpu.to_device(_slice(pk, 0, 100)), append=True)
    engine.extract_reset()
    engine.extract(dpu.to_device(_slice(pk, 0, 100)), append=True)
    state, seqs = _canon(engine.fetch_extracted()), _dev_strings(engine)
    good = dpu.to_device(_slice(pk, 100, 200))
    with pytest.raises(ValueError, match="all device or all host"):   # refused before any C call
        engine.extract(dict(good, flag=_slice(pk, 100, 200)["flag"]), append=True)
    with pytest.raises(TypeError, match="cigar_off"):
        engine.extract(dict(good, cigar_off=good["cigar_off"].to(torch.int32)), append=True)
    # a host pointer handed straight to the C call
    h = _slice(pk, 100, 200)
    keep = [np.ascontiguousarray(h[k], dtype=np.int32) for k in _abi.READ_FIELDS] + [np.ascontiguousarray(h[k], dtype=np.int64) for k in ("cigar_off", "sa_off")]
    rc_ = _abi.csv_read_cols(100, *[k.ctypes.data_as(C.POINTER(C.c_int32)) for k in keep[:7]], *[k.ctypes.data_as(C.POINTER(C.c_int64)) for k in keep[7:]])
    sa_ = _abi.csv_sa_cols(0, *([None] * 7))
    counts, nr = (C.c_int64 * 5)(), C.c_int64(0)
    assert engine.L.csv_extract_append_device(engine.h, C.byref(rc_), None, C.c_int64(0), C.byref(sa_), None, None, counts, C.byref(nr)) == _abi.CSV_E_INVALID
    assert b"not device memory" in engine.L.csv_last_error()
    # offsets the device check refuses, appended and as a fresh call
    bad_dec = dict(good, cigar_off=good["cigar_off"].clone())
    bad_dec["cigar_off"][50] = bad_dec["cigar_off"][49] - 1
    bad_end = dict(good, cigar_off=good["cigar_off"].clone())
    bad_end["cigar_off"][-1] = len(good["cigar"]) + 1
    bad_seq = dict(good, seq_off=good["seq_off"].clone())
    bad_seq["seq_off"][-1] = len(good["seq4"]) + 64
    for bad, col in ((bad_dec, "cigar_off"), (bad_end, "cigar_off"), (bad_seq, "seq_off")):
        for append in (True, False):
            with pytest.raises(_lib.CuteSVError, match=col) as e:
                engine.extract(bad, append=append)
            assert e.value.code == _abi.CSV_E_INPUT
            assert _canon(engine.fetch_extracted()) == state and _dev_strings(engine) == seqs
    engine.extract(good, append=True)
    engine_all = engine.fetch_extracted()
    engine.extract(dpu.to_device(pk))
    assert _canon(engine_all) == _canon(engine.fetch_extracted())


# ---- end to end: BAM -> native decoder -> torch CUDA packets -> device extraction and sequences -> VCF ----

def _to_real_bam(pickled, path):
    import pickle
    ds = pickle.load(open(pickled, "rb"))
    order = {n: i for i, (n, _) in enumerate(ds["contigs"])}
    bam_writer.write_bam(path, ds["contigs"], sorted(ds["reads"], key=lambda r: (order[r.reference_name], r.reference_start)), extra_unmapped=2)
    return path


def _vcf_device(engine, tmp_path, golden, materialise):
    bamio.build()
    gold = json.load(open(os.path.join(golden_util.GOLDEN, golden)))
    pk_path, fa, out, wd = materialise(gold)
    bam = _to_real_bam(pk_path, str(tmp_path / "real.bam"))
    argv = [bam, fa, out, wd] + gold["flags"]
    args = cli.build_parser().parse_args(argv)
    rd = bamio.BamReader(bam, threads=2)
    contig_info = [[n, rd.get_reference_length(n)] for n, _ in rd.index_statistics()]
    chrom_names = sorted(c[0] for c in contig_info)
    chrom_id = {n: i for i, n in enumerate(chrom_names)}
    engine.set_params(cli.params_from_args(args))
    engine.set_contigs(np.array([dict(contig_info)[n] for n in chrom_names], dtype=np.int64))
    engine.extract_reset()
    rd.set_chrom_ids(chrom_id)
    aln = []
    while True:
        pk = rd.next_packet(cli.PACKET_READS)
        if pk is None:
            break
        has_cigar = pk["cigar_off"][1:] > pk["cigar_off"][:-1]
        v = np.flatnonzero(has_cigar)
        aln.append(dict(chrom=pk["chrom"][v], start=pk["ref_start"][v], end=pk["ref_end"][v], read_id=pk["read_id"][v],
                        is_primary=((pk["flag"][v] == 0) | (pk["flag"][v] == 16)).astype(np.uint8)))
        keep = has_cigar & (pk["flag"] != 256) & (pk["flag"] != 272) & (pk["chrom"] >= 0)
        sub = dpu.flat_seq(bamio.subset_packet(pk, np.flatnonzero(keep)))
        engine.extract(dpu.to_device(sub), append=True)
    names, rank = rd.names(), rd.name_ranks()
    rd.close()
    read_names = [names[i] for i in np.argsort(rank[:len(names)], kind="stable")]
    engine.remap_read_ids(rank[:max(len(names), 1)])
    c = engine.fetch_sig_cols("INS", cols=("chrom", "a", "b", "read_id"))
    tie = cli.ins_tie_rows(c["chrom"], c["a"], c["b"], c["read_id"])
    pairs = cli.ins_tie_swaps(c["chrom"], c["a"], c["b"], c["read_id"], dict(zip(tie.tolist(), engine.fetch_ins_seqs(tie))))
    engine.swap_ins_rows(pairs)
    if args.genotype:
        a = {k: np.concatenate([x[k] for x in aln]) for k in aln[0]}
        a["read_id"] = rank[a["read_id"]]
        order = np.argsort(a["chrom"], kind="stable")
        engine.upload_alignments({k: v[order] for k, v in a.items()})
    engine.cluster_device(0x1F)
    cands, genos, nbuf = engine.fetch()
    engine.upload_alignments(None)
    emitted = np.unique(cands["aux"][cands["svtype"] == INS]).astype(np.int64)
    seq_of = dict(zip(emitted.tolist(), engine.fetch_ins_seqs(emitted)))
    got = rows.records_to_rows(cands, genos, nbuf, chrom_names, lambda k: read_names[k], seq_of.__getitem__, bool(args.genotype))
    results = {}
    for t in _abi.TYPE_NAMES:
        for (tt, chrom), r in got.items():
            if tt == t:
                results.setdefault(chrom, []).extend(r)
    ref = vcf.IndexedFasta(fa)
    vcf.write_vcf(out, results, ref, contig_info, args.sample, argv, dict(genotype=args.genotype, max_size=args.max_size, min_size=args.min_size,
                                                                          report_readid=args.report_readid, ignore_sequence=args.ignore_sequence))
    ref.close()
    return [l for l in open(out) if not l.startswith("##")], gold["lines"], len(pairs)


@pytest.mark.parametrize("golden", ["cli_dataset1.json", "cli_config1.json"])
def test_vcf_from_device_packets_equals_reference(engine, tmp_path, golden):
    mat = gen_cli_golden.materialise if golden == "cli_dataset1.json" else gen_cli_golden.materialise_config1
    lines, gold, _ = _vcf_device(engine, tmp_path, golden, lambda g: mat(str(tmp_path)))
    assert len(lines) > 5 and lines == gold


def test_vcf_ins_ties_ordered_by_device_strings(engine, tmp_path):
    import vcf_util
    lines, gold, n_pairs = _vcf_device(engine, tmp_path, "cli_dataset2_ins_ties.json",
                                       lambda g: gen_cli_golden.materialise(str(tmp_path), g["seed"], g["double_ins"]))
    assert n_pairs > 0 and len(lines) > 20
    assert vcf_util.normalise_rnames(lines) == vcf_util.normalise_rnames(gold)
