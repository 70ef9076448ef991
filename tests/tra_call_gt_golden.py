"""Runs resolveTRA's call_gt drop-ins (cuteSV_resolveTRA.call_gt / call_gt_batch) on the cases of
tests/golden/tra_call_gt.json.gz (what the reference's call_gt returned on the same fake BAM, oracle/gen_tra_call_gt_golden.py)
with whatever engine runtime.get_engine() returns, and compares values and their Python types."""
import gzip
import json
import os
import pickle
import sys

import pytest

from cutesv_b200.synth import SynthRead

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "tra_call_gt.json.gz")
_DATA = None


def data():
    global _DATA
    if _DATA is None:
        with gzip.open(GOLDEN, "rt") as f:
            _DATA = json.load(f)
    return _DATA


def write_bam(path, contigs, records):
    """contigs [[name, length]], records [[contig, start, end, flag, name]] -> a pickle tests/fake_pysam reads as a BAM."""
    reads = []
    for chrom, start, end, flag, name in records:
        r = SynthRead()
        r.reference_name, r.reference_start, r.reference_end, r.flag, r.query_name = chrom, start, end, flag, name
        r.mapq, r.query_length, r.query_sequence, r.cigartuples, r.cigar, r.tags = 60, 0, "", [], [], []
        reads.append(r)
    with open(path, "wb") as f:
        pickle.dump(dict(contigs=[tuple(c) for c in contigs], reads=reads), f)


@pytest.fixture
def fake_bam(tmp_path, monkeypatch):
    """The golden's BAM as a fake-pysam pickle, with tests/fake_pysam importable as pysam."""
    monkeypatch.syspath_prepend(os.path.join(HERE, "fake_pysam"))
    sys.modules.pop("pysam", None)
    path = str(tmp_path / "tra.bam")
    write_bam(path, data()["contigs"], data()["records"])
    yield path
    sys.modules.pop("pysam", None)


def args(case):
    return case["pos_1"], case["pos_2"], case["chr_1"], case["chr_2"], case["read_id_list"]


def same(got, case):
    return list(got) == case["result"] and [type(v).__name__ for v in got] == case["types"]


def check_call_gt(bam):
    from cutesv_b200 import cuteSV_resolveTRA
    for case in data()["cases"]:
        got = cuteSV_resolveTRA.call_gt(bam, *args(case), case["bias"], case["gt_round"])
        assert same(got, case), (case["name"], got, case["result"])


def check_call_gt_batch(bam):
    """One call_gt_batch per (bias, gt_round) group of cases."""
    from cutesv_b200 import cuteSV_resolveTRA
    groups = {}
    for case in data()["cases"]:
        groups.setdefault((case["bias"], case["gt_round"]), []).append(case)
    for (bias, gt_round), cases in sorted(groups.items()):
        got = cuteSV_resolveTRA.call_gt_batch(bam, [args(c) for c in cases], bias, gt_round)
        assert len(got) == len(cases)
        for g, case in zip(got, cases):
            assert same(g, case), (case["name"], g, case["result"])
