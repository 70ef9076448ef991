"""-m gpu: read names ranked on the device (named device packets, rank_names, fetch_names, name_rank_tensor) and INS tie groups
ordered by the device-built sequences (order_ins_ties).  Against Python's sorted(), the host-ranked path on the same records, the
host tie swaps, and the reference's own VCFs end to end with no host pass over names, ties or signature columns."""
import json
import os

import numpy as np
import pytest

import device_packet_util as dpu
import golden_util
import name_util
from cutesv_b200 import _abi, _lib, bamio, cli, rows, vcf
from oracle import gen_cli_golden
from test_gpu_device_extract import _canon, _dev_strings, _packet, _setup, _slice, _to_real_bam

pytestmark = pytest.mark.gpu
INS = _abi.CSV_INS


def _record_names(pk, rnames):
    """The read name of every record of a synthetic packet (its read_id is the name's index in rnames)."""
    return [rnames[i] for i in pk["read_id"].tolist()]


def _named_run(engine, pk, names, cuts):
    """Named device packets of the slices [cuts[k], cuts[k + 1]) of pk, appended; returns rank_names()."""
    engine.extract_reset()
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        engine.extract(name_util.named(dpu.to_device(_slice(pk, lo, hi)), names[lo:hi]), append=True)
    return engine.rank_names()


@pytest.mark.parametrize("which", sorted(name_util.name_sets()))
def test_ranks_equal_python_sorted(engine, which):
    reads, pk = _setup(engine, 4, 300)
    n_rec = len(pk["chrom"])
    names = name_util.name_sets(7)[which]
    rng = np.random.default_rng(len(names))
    names = [names[i] for i in rng.permutation(len(names))]
    # the same alignment packet again and again, each time with the next slice of names; an empty packet in between
    all_names = []
    engine.extract_reset()
    for k in range(0, max(len(names), 1), n_rec):
        chunk = names[k:k + n_rec]
        chunk = chunk + [names[(k + j) % len(names)] for j in range(n_rec - len(chunk))]   # duplicates across packets
        engine.extract(name_util.named(dpu.to_device(pk), chunk), append=True)
        all_names += chunk
        if k == 0:
            engine.extract(name_util.named(dpu.to_device(_slice(pk, 5, 5)), []), append=True)
    nd = engine.rank_names()
    assert nd == len(set(all_names))
    assert np.array_equal(engine.name_rank_tensor().cpu().numpy(), name_util.dense_ranks(all_names))
    assert engine.fetch_names(np.arange(nd)) == sorted(set(all_names))
    assert engine.rank_names() == nd   # a second call only reports the count


def test_fetch_names_shuffled_with_repeats(engine):
    reads, pk = _setup(engine, 6, 300)
    names = [n + "_suffix" * (i % 3) for i, n in enumerate(name_util.name_sets(1)["ont_uuid"][:len(pk["chrom"])])]
    nd = _named_run(engine, pk, names, (0, len(names)))
    srt = sorted(set(names))
    want = np.random.default_rng(2).integers(0, nd, 500)
    assert engine.fetch_names(want) == [srt[i] for i in want.tolist()]
    assert engine.fetch_names([]) == []
    with pytest.raises(_lib.CuteSVError) as e:
        engine.fetch_names([nd])
    assert e.value.code == _abi.CSV_E_INVALID


# ---- parity with the host-ranked path ----

def _parity(engine, pk, rnames, cuts):
    engine.extract(dpu.to_device(pk))   # read_id: the host's dense ranks (index in the sorted names)
    host = _canon(engine.fetch_extracted())
    _named_run(engine, pk, _record_names(pk, rnames), cuts)
    assert _canon(engine.fetch_extracted()) == host


@pytest.mark.parametrize("name", ["extract_s0", "extract_s1", "extract_s2", "extract_s3", "extract_s4", "extract_s5", "extract_s6",
                                  "extract_l0", "extract_l1", "extract_l2", "extract_l3", "extract_l4"])
def test_ranked_golden_packets_equal_host_ranked(engine, name):
    meta = json.load(open(os.path.join(golden_util.GOLDEN, name + ".json")))
    reads, names, lens, rnames, pk = _packet(meta["seed"], meta["n_reads"], meta.get("kind", "short"))
    engine.set_params(_abi.default_params(**meta["params"]))
    engine.set_contigs(lens)
    _parity(engine, pk, rnames, (0, len(pk["chrom"])))


@pytest.mark.parametrize("seed", range(12))
def test_ranked_seeded_packets_equal_host_ranked(engine, seed):
    reads, names, lens, rnames, pk = _packet(seed)
    rng = np.random.default_rng(seed)
    p = _abi.default_params(min_size=int(rng.choice([30, 50, 10])), max_size=int(rng.choice([-1, 100000, 2000])),
                            min_mapq=int(rng.choice([20, 0, 30])), max_split_parts=int(rng.choice([7, -1, 2, 3])),
                            min_read_len=int(rng.choice([500, 100])), min_siglength=int(rng.choice([10, 30])),
                            merge_del_threshold=int(rng.choice([0, 500])), merge_ins_threshold=int(rng.choice([100, 500, 0])))
    engine.set_params(p)
    engine.set_contigs(lens)
    n = len(pk["chrom"])
    _parity(engine, pk, rnames, (0, n // 3, n // 3, n))


# ---- rejections change nothing ----

def test_rejections_leave_the_accumulation_intact(engine):
    import torch
    reads, names, lens, rnames, pk = _packet(5, 200)
    engine.set_params(_abi.default_params(min_support=2, genotype=1, min_mapq=0, min_read_len=100))
    engine.set_contigs(lens)
    nm = _record_names(pk, rnames)
    n = len(pk["chrom"])
    h = n // 2
    engine.extract(dpu.to_device(pk))
    want = _canon(engine.fetch_extracted())

    def first_half():
        engine.extract_reset()
        engine.extract(name_util.named(dpu.to_device(_slice(pk, 0, h)), nm[:h]), append=True)
        return _canon(engine.fetch_extracted()), _dev_strings(engine)

    state = first_half()
    good = name_util.named(dpu.to_device(_slice(pk, h, n)), nm[h:])
    bad_off = dict(good, name_off=good["name_off"].clone())
    bad_off["name_off"][3] = bad_off["name_off"][2] - 1
    bad_end = dict(good, name_off=good["name_off"].clone())
    bad_end["name_off"][-1] = len(good["names"]) + 1
    long_name = name_util.named(dpu.to_device(_slice(pk, h, n)), ["x" * 255] + nm[h + 1:])
    for bad, match in ((bad_off, "name_off"), (bad_end, "name_off"), (long_name, "254")):
        with pytest.raises(_lib.CuteSVError, match=match) as e:
            engine.extract(bad, append=True)
        assert e.value.code == _abi.CSV_E_INPUT
        assert (_canon(engine.fetch_extracted()), _dev_strings(engine)) == state
    # a named accumulation takes no unnamed packet, device or host, and the reverse
    for unnamed in (dpu.to_device(_slice(pk, h, n)), {k: v for k, v in _slice(pk, h, n).items() if k not in ("seq_off", "seq4")}):
        with pytest.raises(_lib.CuteSVError) as e:
            engine.extract(unnamed, append=True)
        assert e.value.code == _abi.CSV_E_STATE
        assert (_canon(engine.fetch_extracted()), _dev_strings(engine)) == state
    engine.extract_reset()
    engine.extract(dpu.to_device(_slice(pk, 0, h)), append=True)
    with pytest.raises(_lib.CuteSVError) as e:
        engine.extract(good, append=True)
    assert e.value.code == _abi.CSV_E_STATE
    # read_id together with names never reaches the library
    with pytest.raises(ValueError, match="read_id"):
        engine.extract(dict(good, read_id=torch.zeros(n - h, dtype=torch.int32, device="cuda")), append=True)
    # no append after the ranking
    state = first_half()
    engine.extract(good, append=True)
    engine.rank_names()
    ranked = _canon(engine.fetch_extracted())
    assert ranked == want
    with pytest.raises(_lib.CuteSVError) as e:
        engine.extract(good, append=True)
    assert e.value.code == _abi.CSV_E_STATE
    assert _canon(engine.fetch_extracted()) == ranked
    # ranking and fetching before the ranking
    first_half()
    for call in (engine.name_rank_tensor, lambda: engine.fetch_names([0]), engine.order_ins_ties):
        with pytest.raises(_lib.CuteSVError) as e:
            call()
        assert e.value.code == _abi.CSV_E_STATE
    # order_ins_ties without a sequence arena (named packets without bases)
    engine.extract_reset()
    engine.extract(name_util.named(dpu.to_device({k: v for k, v in pk.items() if k not in ("seq_off", "seq4")}), nm), append=True)
    engine.rank_names()
    with pytest.raises(_lib.CuteSVError) as e:
        engine.order_ins_ties()
    assert e.value.code == _abi.CSV_E_STATE
    assert _canon(engine.fetch_extracted()) == want
    # and a correct run on the same engine
    state = first_half()
    engine.extract(good, append=True)
    engine.rank_names()
    assert _canon(engine.fetch_extracted()) == want


def test_stream_order_and_overwrite_after_return(engine):
    import torch
    reads, names, lens, rnames, pk = _packet(11, 400)
    engine.set_params(_abi.default_params(min_support=2, genotype=1, min_mapq=0, min_read_len=100))
    engine.set_contigs(lens)
    engine.extract(dpu.to_device(pk))
    ref = _canon(engine.fetch_extracted())
    staged = name_util.named(dpu.to_device(pk), _record_names(pk, rnames))
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)   # the packet's final tensors, names included, are written late on the side stream
        d = {k: ({kk: vv.clone() for kk, vv in v.items()} if isinstance(v, dict) else v.clone()) for k, v in staged.items()}
    assert not side.query()
    engine.extract(d, stream=side)
    with torch.cuda.stream(side):   # overwritten in the side stream's order right after the call returns
        for k, v in d.items():
            for t in (v.values() if isinstance(v, dict) else [v]):
                t.fill_(7)
    engine.rank_names()
    assert _canon(engine.fetch_extracted()) == ref


# ---- INS ties ----

def _ins_state(engine):
    ex = engine.fetch_extracted()
    s = ex["sigs"]["INS"]
    return [s[k].tolist() for k in ("chrom", "a", "b", "read_id", "c")] + [ex["piece_off"].tolist(), ex["piece_cnt"].tolist(), _dev_strings(engine)]


def _host_tie_expectation(engine):
    """The INS state after the host route (cli.ins_tie_swaps on the device strings, applied as csv_swap_ins_rows applies them),
    computed from a snapshot of this accumulation: extraction hands out rows with atomics, so two extractions may differ in row
    order and the comparison has to be made on one.  Returns (state, rows whose content moves)."""
    before = _ins_state(engine)
    chrom, a, b, rid = (np.array(before[k], dtype=np.int32) for k in range(4))
    pairs = cli.ins_tie_swaps(chrom, a, b, rid, before[7])
    perm = np.arange(len(chrom))
    for i, j in pairs:
        perm[i], perm[j] = perm[j], perm[i]
    return [[col[k] for k in perm.tolist()] for col in before], int((perm != np.arange(len(perm))).sum())


@pytest.mark.parametrize("seed", range(4))
def test_order_ins_ties_equals_host_swaps_on_planted_ties(engine, seed):
    reads, names, lens, rnames, pk = _packet(20 + seed, 400)
    engine.set_params(_abi.default_params(min_support=2, min_mapq=0, min_read_len=100))
    engine.set_contigs(lens)
    nm = _record_names(pk, rnames)
    # the same records again with other bases: every INS row gets a twin tying on (contig, int(pos), len, read) whose string differs
    other = dict(pk, seq4=np.random.default_rng(seed).integers(0, 256, len(pk["seq4"])).astype(np.uint8))
    engine.extract_reset()
    engine.extract(name_util.named(dpu.to_device(pk), nm), append=True)
    engine.extract(name_util.named(dpu.to_device(other), nm), append=True)
    engine.rank_names()
    want, n_moved = _host_tie_expectation(engine)
    moved = engine.order_ins_ties()
    assert n_moved > 0 and moved == n_moved
    assert _ins_state(engine) == want
    assert engine.order_ins_ties() == 0   # ordered already


def test_order_ins_ties_after_remap_read_ids(engine):
    reads, names, lens, rnames, pk = _packet(31, 400)
    engine.set_params(_abi.default_params(min_support=2, min_mapq=0, min_read_len=100))
    engine.set_contigs(lens)
    other = dict(pk, seq4=np.random.default_rng(9).integers(0, 256, len(pk["seq4"])).astype(np.uint8))
    engine.extract_reset()
    engine.extract(dpu.to_device(pk), append=True)
    engine.extract(dpu.to_device(other), append=True)
    want, n_moved = _host_tie_expectation(engine)   # read_id: the host's ranks already
    assert engine.order_ins_ties() == n_moved > 0
    assert _ins_state(engine) == want


# ---- end to end: BAM -> native decoder -> named torch CUDA packets -> device ranks and ties -> VCF ----

def _vcf_device_named(engine, tmp_path, golden, materialise):
    import torch
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
    aln, aln_names = [], []
    rec_of_name = {}   # a record of the accumulation per read name: the provisional id of alignment rows outside it
    n_rec = 0
    while True:
        pk = rd.next_packet(cli.PACKET_READS)
        if pk is None:
            break
        names = rd.names()   # the decoder's table so far; the library only ever sees the bytes
        has_cigar = pk["cigar_off"][1:] > pk["cigar_off"][:-1]
        v = np.flatnonzero(has_cigar)
        aln.append(dict(chrom=pk["chrom"][v], start=pk["ref_start"][v], end=pk["ref_end"][v],
                        is_primary=((pk["flag"][v] == 0) | (pk["flag"][v] == 16)).astype(np.uint8)))
        aln_names += [names[i] for i in pk["read_id"][v].tolist()]
        keep = np.flatnonzero(has_cigar & (pk["flag"] != 256) & (pk["flag"] != 272) & (pk["chrom"] >= 0))
        sub = dpu.flat_seq(bamio.subset_packet(pk, keep))
        rec_names = [names[i] for i in sub["read_id"].tolist()]
        for j, nm in enumerate(rec_names):
            rec_of_name.setdefault(nm, n_rec + j)
        n_rec += len(rec_names)
        engine.extract(name_util.named(dpu.to_device(sub), rec_names), append=True)
    rd.close()
    engine.rank_names()
    n_moved = engine.order_ins_ties()
    if args.genotype:
        a = {k: np.concatenate([x[k] for x in aln]) for k in aln[0]}
        prov = np.array([rec_of_name[nm] for nm in aln_names], dtype=np.int64)
        order = np.argsort(a["chrom"], kind="stable")
        dev = torch.device("cuda", engine.device)
        cols = {k: torch.from_numpy(np.ascontiguousarray(v[order])).to(dev) for k, v in a.items()}
        cols["read_id"] = engine.name_rank_tensor()[torch.from_numpy(prov[order]).to(dev)].contiguous()   # one gather on the device
        engine.upload_alignments(cols)
    engine.cluster_device(0x1F)
    cands, genos, nbuf = engine.fetch()
    engine.upload_alignments(None)
    ids = np.unique(nbuf).astype(np.int32)
    name_of = dict(zip(ids.tolist(), engine.fetch_names(ids)))   # RNAMES: the emitted reads only
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
    return [l for l in open(out) if not l.startswith("##")], gold["lines"], n_moved


@pytest.mark.parametrize("golden", ["cli_dataset1.json", "cli_config1.json"])
def test_vcf_from_named_device_packets_equals_reference(engine, tmp_path, golden):
    mat = gen_cli_golden.materialise if golden == "cli_dataset1.json" else gen_cli_golden.materialise_config1
    lines, gold, _ = _vcf_device_named(engine, tmp_path, golden, lambda g: mat(str(tmp_path)))
    assert len(lines) > 5 and lines == gold


def test_vcf_ins_ties_ordered_on_the_device(engine, tmp_path):
    import vcf_util
    lines, gold, n_moved = _vcf_device_named(engine, tmp_path, "cli_dataset2_ins_ties.json",
                                             lambda g: gen_cli_golden.materialise(str(tmp_path), g["seed"], g["double_ins"]))
    assert n_moved > 0 and len(lines) > 20
    assert vcf_util.normalise_rnames(lines) == vcf_util.normalise_rnames(gold)
