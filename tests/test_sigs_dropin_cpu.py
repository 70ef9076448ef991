"""CPU checks of the signature-phase drop-ins (cutesv_b200.cuteSV_signatures) against the reference's own single_pipe /
process_process_sigs_type output (tests/golden/sigs_dropin.json.gz, oracle/gen_sigs_dropin_golden.py).

The device calls are replaced by their host statements: csv_extract by the emulator of kernel (a) (tests/emul, the same
extract_core.h rules, rows in record order), csv_sort_sigs by a numpy stable lexsort + adjacent de-duplication.  So the
host half -- window filtering, tuple building, INS strings, INS tie finishing, per-contig pickles and index, .sigs text --
is checked here; tests/test_gpu_sigs_dropin.py runs the same against the CUDA library."""
import os
import pickle
import sys

import numpy as np
import pytest

import emul_lib
import sigs_dropin_data as D
from cutesv_b200 import cuteSV_signatures as S, workdir


class HostEngine(object):
    """Engine stand-in: csv_extract through the emulator, csv_sort_sigs through D.np_sort_sigs."""

    def set_params(self, p):
        self.p = p

    def set_contigs(self, lens):
        self.n_contigs = len(lens)

    def set_extract_records(self, on):
        pass

    def extract(self, pk):
        self.ex = emul_lib.extract(self.p, pk)

    def fetch_extracted(self):
        return self.ex

    def fetch_records(self, t):
        n = len(self.ex["rows"]["chrom"]) if t == "reads" else len(self.ex["sigs"][t]["chrom"])
        return np.zeros(n, np.int32)   # the emulator emits record by record: already in order

    def upload(self, sigs, reads):
        self.up = (sigs, reads)

    def sort_sigs(self, svtype):
        sigs, reads = self.up
        return D.np_sort_sigs(svtype, reads if svtype == "reads" else sigs[svtype], self.n_contigs)


@pytest.fixture(scope="module")
def golden():
    return D.load()


@pytest.fixture
def host_engine(monkeypatch):
    emul_lib.build()
    e = HostEngine()
    monkeypatch.setattr(S.runtime, "get_engine", lambda: e)
    return e


def _tuples(lst):
    return [tuple(x) for x in lst]


def test_golden_self_consistent(golden):
    """Per case: the rebuilt lists are the concatenated pid lists sorted with the reference's key and de-duplicated; the
    index keys are the contigs in that order; reads_count counts the reads rows per contig; the .sigs text has one line per
    rebuilt row."""
    assert [c["name"] for c in golden["cases"]] == [c["name"] for c in D.CASES]
    for g in golden["cases"]:
        assert len(g["windows"]) == len(g["tasks"]) == len(g["task_pid"])
        for t in D.TYPES:
            cat = []
            for pid in D.PIDS:
                for w, p in zip(g["windows"], g["task_pid"]):
                    if p == pid:
                        cat.extend(_tuples(w[t]))
            want = sorted(cat, key=workdir.sort_key(t))
            if t != "reads":
                want = S.remove_duplicates_sorted(want)
            got = [x for _, v in g["rebuilt"][t] for x in _tuples(v)]
            assert got == want, (g["name"], t)
            assert g["index_keys"][t] == [c for c, _ in g["rebuilt"][t]]
            if t == "reads":
                assert g["reads_count"][t] == {c: len(v) for c, v in g["rebuilt"][t]}
            assert g["sigs_text"][t].count("\n") == len(got)


def test_sigs_text_and_ins_ties_from_columns(golden, host_engine, tmp_path):
    """process_process_sigs_type on the reference-written pid pickles with the host sort: the rebuilt lists, index keys,
    reads_count and .sigs text equal the reference's (INS tie groups finished by sequence on the host)."""
    n_ties = 0
    for g in golden["cases"]:
        d = str(tmp_path / g["name"]) + "/"
        D.write_pid_pickles(d, g)
        for t in D.TYPES:
            sv, index, rc = S.process_process_sigs_type((t, d, list(D.PIDS), True))
            assert sv == t and list(index) == g["index_keys"][t]
            assert rc == (g["reads_count"][t] if t == "reads" else {})
            with open("%s/%s.sigs" % (d, t)) as f:
                assert f.read() == g["sigs_text"][t], (g["name"], t)
            for chrom, rows in g["rebuilt"][t]:
                assert workdir.load_slice(d, t, chrom, {t: index}) == _tuples(rows)
        ins = [x for _, v in g["rebuilt"]["INS"] for x in v]
        n_ties += sum(1 for a, b in zip(ins, ins[1:]) if a[-1] == b[-1] and int(a[0]) == int(b[0]) and a[1:3] == b[1:3])
    assert n_ties > 0


def test_finish_ins_ties_orders_and_dedups():
    rows = [(10, 5, "r", "TT", "INS", "c"), (10.5, 5, "r", "AA", "INS", "c"), (10, 5, "r", "TT", "INS", "c"), (10, 5, "r", "AA", "INS", "c"),
            (11, 5, "r", "GG", "INS", "c")]
    out, pos = S.finish_ins_ties(rows, [0, 1, 1, 1, 0])
    assert out == [(10.5, 5, "r", "AA", "INS", "c"), (10, 5, "r", "AA", "INS", "c"), (10, 5, "r", "TT", "INS", "c"), (11, 5, "r", "GG", "INS", "c")]
    assert pos.tolist() == [0, 1, 2, 4]


def test_written_offsets_load(golden, host_engine, tmp_path):
    """Every index offset of the written <TYPE>.pickle is a pickle boundary that workdir.load_slice reads as that contig's list."""
    g = golden["cases"][0]
    d = str(tmp_path) + "/"
    D.write_pid_pickles(d, g)
    idx = {}
    for t in D.TYPES:
        sv, index, rc = S.process_process_sigs_type((t, d, list(D.PIDS), False))
        idx[t] = index
        assert not os.path.exists("%s/%s.sigs" % (d, t))
    for t in D.TYPES:
        with open("%s%s.pickle" % (d, t), "rb") as f:
            blob = f.read()
        offs = sorted(idx[t].values())
        for a, b in zip(offs, offs[1:] + [len(blob)]):
            assert len(pickle.dumps(pickle.loads(blob[a:b]))) <= b - a
        for chrom in idx[t]:
            rows = workdir.load_slice(d, t, chrom, idx)
            assert rows and all(r[-1] == chrom for r in rows)


def test_single_pipe_host_half_on_emulator(golden, host_engine, tmp_path, monkeypatch):
    """single_pipe through the emulator of kernel (a): the pid pickles equal the reference's lists window by window, in order."""
    monkeypatch.syspath_prepend(os.path.join(os.path.dirname(os.path.abspath(__file__)), "fake_pysam"))   # stands in for pysam
    monkeypatch.delitem(sys.modules, "pysam", raising=False)
    for case, g in zip(D.CASES, golden["cases"]):
        ds, tasks, bed = D.dataset(case)
        assert tasks == g["tasks"]
        d = str(tmp_path / case["name"]) + "/"
        os.makedirs(d + "signatures")
        D.write_fake_bam(d + "in.bam", ds)
        S.init_reading_process(d + "in.bam", None)
        proc = type("P", (), {})()
        monkeypatch.setattr(S, "current_process", lambda: proc)
        for i, task in enumerate(tasks):
            proc.pid = g["task_pid"][i]
            S.single_pipe(*D.task_args(case, d, task, None if bed is None else [tuple(r) for r in bed[i]]))
            for t in D.TYPES:
                got = D.read_pid_dumps("%ssignatures/%s%s.pickle" % (d, proc.pid, t))[-1]
                assert got == _tuples(g["windows"][i][t]), (case["name"], i, t)
        S.cleanup()
