"""CSI indexes (`samtools index -c`, the index of BAMs with contigs longer than 2^29 bp): the native decoder reads the
per-contig mapped counts from <bam>.csi or <stem>.csi when there is no .bai, with the same result as from the BAI, and the
CLI writes the same VCF.  A malformed CSI raises IOError."""
import json
import os
import pickle
import struct

import pytest

import bam_writer
import golden_util
from csi_writer import bgzf, write_csi
from cutesv_b200 import bamio, cli
from oracle import gen_cli_golden


def _bam(tmp_path):
    bamio.build()
    pk, fa, out, wd = gen_cli_golden.materialise(str(tmp_path))
    ds = pickle.load(open(pk, "rb"))
    order = {n: i for i, (n, _) in enumerate(ds["contigs"])}
    reads = sorted(ds["reads"], key=lambda r: (order[r.reference_name], r.reference_start))
    bam = str(tmp_path / "real.bam")
    bam_writer.write_bam(bam, ds["contigs"], reads, extra_unmapped=2)
    return bam, fa, out, wd


@pytest.mark.parametrize("depth,name", [(5, "{bam}.csi"), (7, "{stem}.csi"), (9, "{bam}.csi")])
def test_csi_gives_the_bai_statistics(tmp_path, depth, name):
    bam, _, _, _ = _bam(tmp_path)
    rd = bamio.BamReader(bam)
    want = rd.index_statistics()
    assert sum(m for _, m in want) > 100
    os.remove(bam + ".bai")
    write_csi(name.format(bam=bam, stem=os.path.splitext(bam)[0]), want, depth=depth, aux=b"\0" * (3 * depth))
    assert rd.index_statistics() == want
    rd.close()


def test_cli_with_only_a_csi_writes_the_reference_vcf(tmp_path):
    from emul_engine import EmulEngine
    bam, fa, out, wd = _bam(tmp_path)
    rd = bamio.BamReader(bam)
    stats = rd.index_statistics()
    rd.close()
    os.remove(bam + ".bai")
    write_csi(bam + ".csi", stats, depth=6)
    gold = json.load(open(os.path.join(golden_util.GOLDEN, "cli_dataset1.json")))
    argv = [bam, fa, out, wd] + gold["flags"]
    cli.main_ctrl(cli.build_parser().parse_args(argv), argv, engine=EmulEngine())
    assert [l for l in open(out) if not l.startswith("##")] == gold["lines"]


@pytest.mark.parametrize("cut", ["half", "header", "body"])
def test_malformed_csi_raises(tmp_path, cut):
    bam, _, _, _ = _bam(tmp_path)
    rd = bamio.BamReader(bam)
    stats = rd.index_statistics()
    os.remove(bam + ".bai")
    csi = bam + ".csi"
    if cut == "half":   # cut inside a compressed block
        write_csi(csi, stats)
        data = open(csi, "rb").read()
        open(csi, "wb").write(data[:len(data) // 2])
    else:               # well-formed BGZF, index content cut short
        body = b"CSI\1" + struct.pack("<iii", 14, 5, 0)
        if cut == "body":
            body += struct.pack("<ii", len(stats), 2) + struct.pack("<IQi", 0, 0, 1)
        open(csi, "wb").write(bgzf(body))
    with pytest.raises(IOError) as e:
        rd.index_statistics()
    assert "CSI" in str(e.value)
    rd.close()
