"""CPU: resolveTRA's call_gt drop-ins (cuteSV_resolveTRA.call_gt / call_gt_batch) run end to end on the test-only emulator
tests/emul/emul_tra_call_gt.cpp, which compiles the kernel's per-query rules (core.h tra_call_gt over the scalar
count_coverage) for the host, and reproduce every stored reference output of tests/golden/tra_call_gt.json.gz."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import tra_call_gt_golden as tg
from tra_call_gt_golden import fake_bam  # noqa: F401 (fixture)
from cutesv_b200 import _abi, runtime


class EmulTraEngine(object):
    """The part of Engine the TRA call_gt drop-ins call, on the emulator."""

    def __init__(self, so):
        self.L = C.CDLL(so)
        self.lens = np.zeros(0, np.int64)

    def set_contigs(self, lens, names=None):
        self.lens = np.ascontiguousarray(lens, dtype=np.int64)

    def tra_call_gt(self, queries, support_off, support_ids, bias, gt_round, aln=None):
        q = np.ascontiguousarray(queries, dtype=_abi.TRA_QUERY_DTYPE)
        so = np.ascontiguousarray(support_off, dtype=np.int64)
        si = np.ascontiguousarray(support_ids, dtype=np.int32)
        r, keep = _abi.make_reads_cols(aln)
        out = np.zeros(max(len(q), 1), dtype=_abi.GENO_DTYPE)
        rc = self.L.emul_tra_call_gt(q.ctypes.data_as(C.c_void_p), C.c_int64(len(q)), C.byref(r), C.c_int32(len(self.lens)),
                                     self.lens.ctypes.data_as(C.c_void_p), C.c_int32(bias), C.c_int32(gt_round),
                                     so.ctypes.data_as(C.c_void_p), _abi.ptr(si), out.ctypes.data_as(C.c_void_p))
        assert rc == 0, rc
        return out[:len(q)]


@pytest.fixture(scope="module")
def emul_so(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "emul_tra_call_gt.cpp")
    so = str(tmp_path_factory.mktemp("emul") / "libemul_tra_call_gt.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    return so


@pytest.fixture
def emul_engine(emul_so):
    prev = runtime._engine
    runtime.set_engine(EmulTraEngine(emul_so))
    yield
    runtime.set_engine(prev)


def test_call_gt_golden(emul_engine, fake_bam):
    tg.check_call_gt(fake_bam)


def test_call_gt_batch_golden(emul_engine, fake_bam):
    tg.check_call_gt_batch(fake_bam)


def test_reversed_window_raises_value_error(emul_engine, fake_bam):
    """A window past the contig end by more than the bias (start > end after clamping) is pysam's ValueError, for either
    breakpoint and in a batch."""
    from cutesv_b200 import cuteSV_resolveTRA
    lens = dict(tg.data()["contigs"])
    L = lens["chr2"]
    for pos_1, pos_2 in ((L + 51, 10_000), (10_000, L + 51), (-51, 10_000)):
        with pytest.raises(ValueError):
            cuteSV_resolveTRA.call_gt(fake_bam, pos_1, pos_2, "chr2", "chr2", ["r00001"], 50, 500)
        with pytest.raises(ValueError):
            cuteSV_resolveTRA.call_gt_batch(fake_bam, [(10_000, 10_000, "chr2", "chr2", []), (pos_1, pos_2, "chr2", "chr2", [])], 50, 500)
    # start == end is a valid window: pos exactly bias past the end, or bias before 0
    assert cuteSV_resolveTRA.call_gt(fake_bam, L + 50, -50, "chr2", "chr2", ["r00001"], 50, 500)[0] == 1
