"""The CLI on a draft-assembly BAM with about 40 000 scaffolds in its header (reads on a few dozen of them, some with
string-order ids above 32767, split reads making TRA between them, --genotype, -include_bed): the VCF body equals what the
reference's own main_ctrl wrote (tests/golden/cli_draft_40k.json, made by oracle/gen_cli_golden_draft.py), with a BAI or
with only a CSI index.  CPU variant: kernels replaced by the pipeline emulator; -m gpu variant: the CUDA path."""
import json
import os

import pytest

import bam_writer
import golden_util
from csi_writer import write_csi
from cutesv_b200 import bamio, cli
from oracle import gen_cli_golden_draft

FIRST_COMPACT_ID = 32768   # contig ids from here on do not fit the packed TRA key of a <= 32768-contig table


def _run(engine, tmp_path, index):
    bamio.build()
    gold = json.load(open(os.path.join(golden_util.GOLDEN, "cli_draft_40k.json")))
    pk, fa, out, wd, ds = gen_cli_golden_draft.materialise(str(tmp_path))
    order = {n: i for i, (n, _) in enumerate(ds["contigs"])}
    reads = sorted(ds["reads"], key=lambda r: (order[r.reference_name], r.reference_start))
    bam = str(tmp_path / "draft_real.bam")
    bam_writer.write_bam(bam, ds["contigs"], reads, extra_unmapped=1)
    if index == "csi":
        rd = bamio.BamReader(bam)
        stats = rd.index_statistics()
        rd.close()
        os.remove(bam + ".bai")
        write_csi(bam + ".csi", stats, depth=7)
    argv = [bam, fa, out, wd] + gold["flags"] + ["-include_bed", gen_cli_golden_draft.write_bed(str(tmp_path), ds)]
    cli.main_ctrl(cli.build_parser().parse_args(argv), argv, engine=engine)
    lines = [l for l in open(out) if not l.startswith("##")]
    return lines, gold["lines"], ds


def _check(lines, gold, ds):
    assert lines == gold
    rank = {n: i for i, n in enumerate(sorted(n for n, _ in ds["contigs"]))}
    assert len(rank) >= 40000
    bnd = [l.split("\t") for l in lines[1:] if "SVTYPE=BND" in l]
    assert any(rank[f[0]] >= FIRST_COMPACT_ID for f in bnd)


@pytest.mark.parametrize("index", ["bai", "csi"])
def test_cli_draft_assembly_cpu(tmp_path, index):
    from emul_engine import EmulEngine
    _check(*_run(EmulEngine(), tmp_path, index))


@pytest.mark.gpu
@pytest.mark.parametrize("index", ["bai", "csi"])
def test_cli_draft_assembly_gpu(engine, tmp_path, index):
    _check(*_run(engine, tmp_path, index))


@pytest.mark.gpu
def test_cli_draft_assembly_gpu_takes_the_compact_tra_key(engine, tmp_path):
    """40 000 contigs are past the packed TRA key: the run goes through the pair-rank kernels (a fresh ctx, profiled, so
    that its kernel table holds this run only)."""
    from cutesv_b200.engine import Engine
    eng = Engine(0)
    try:
        eng.set_profiling(True)
        _check(*_run(eng, tmp_path, "bai"))
        kt = eng.kernel_times()
    finally:
        eng.close()
    assert {"k_tra_pair_flags", "k_tra_compact_key"} <= set(kt)
