"""Runs the genotype drop-ins (cuteSV_genotype.overlap_cover / assign_gt, the resolvers' call_gt) on the cases of
tests/golden/genotype_dropin.json.gz (what the reference computed, oracle/gen_genotype_golden.py) with whatever engine
runtime.get_engine() returns, and compares."""
import gzip
import json
import os

import pytest

from cutesv_b200 import cuteSV_genotype, cuteSV_resolveDUP, cuteSV_resolveINDEL, cuteSV_resolveINV, workdir

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "genotype_dropin.json.gz")
_DATA = None


def data():
    global _DATA
    if _DATA is None:
        with gzip.open(GOLDEN, "rt") as f:
            _DATA = json.load(f)
    return _DATA


def dict_rows(d4):
    it, pn, cov, ovl = d4
    assert list(it) == list(pn) == list(cov) == list(ovl)
    return [[k, it[k], pn[k], sorted(cov[k]), sorted(ovl[k])] for k in cov]


def check_overlap_cover(case):
    svs = [tuple(w) for w in case["svs"]]
    if "key_error" in case:
        with pytest.raises(KeyError) as e:
            cuteSV_genotype.overlap_cover(svs, case["reads"])
        assert e.value.args[0] == case["key_error"]
        return
    assert dict_rows(cuteSV_genotype.overlap_cover(svs, case["reads"])) == case["result"]


def check_assign_gt(case):
    src = next(c for c in data()["overlap_cover"] if c["name"] == case["case"])
    it, pn, cov, _ = cuteSV_genotype.overlap_cover([tuple(w) for w in src["svs"]], src["reads"])
    rid = {k: v for k, v in case["read_id"]}
    got = cuteSV_genotype.assign_gt(it, pn, cov, rid)
    assert [[a, b, gt, gl, gq, str(q)] for a, b, gt, gl, gq, q in got] == case["result"]


def write_reads_workdir(path):
    reads = data()["call_gt_reads"]
    return workdir.write_workdir(path, {"reads": [tuple(r) + (c,) for c, rows in sorted(reads.items()) for r in rows]})


def run_call_gt(case, path, idx):
    cand = [list(x) for x in case["candidates"]]
    if case["module"] == "INDEL":
        return cuteSV_resolveINDEL.call_gt(path, case["chr"], cand, case["bias"], case["svtype"], idx)
    m = cuteSV_resolveDUP if case["module"] == "DUP" else cuteSV_resolveINV
    return m.call_gt(path, case["chr"], cand, case["bias"], idx)


def check_call_gt(case, path, idx):
    if "key_error" in case:
        with pytest.raises(KeyError) as e:
            run_call_gt(case, path, idx)
        assert e.value.args[0] == case["key_error"]
        return
    assert run_call_gt(case, path, idx) == case["result"]
