"""CPU: the genotype drop-ins (overlap_cover, assign_gt and the call_gt of resolveINDEL / resolveDUP / resolveINV) run
end to end on the test-only emulator tests/emul/emul_genotype.cpp, which compiles the kernels' per-pair and per-segment
logic (core.h gc_*) for the host, and reproduce every stored reference output of tests/golden/genotype_dropin.json.gz."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import genotype_golden as gg
from cutesv_b200 import _abi, cuteSV_genotype, runtime


class EmulGenotypeEngine(object):
    """The part of Engine the genotype drop-ins call, on the emulator."""

    def __init__(self, so):
        self.L = C.CDLL(so)

    def overlap_cover(self, windows, reads=None, overlap=True):
        w = np.ascontiguousarray(windows, dtype=_abi.WINDOW_DTYPE)
        n = len(w)
        r, keep = _abi.make_reads_cols(reads)
        cap = max(len(reads["chrom"]) * max(n, 1), 1)
        it, pn = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
        co, oo = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)
        ci, oi = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
        rc = self.L.emul_overlap_cover(w.ctypes.data_as(C.c_void_p), C.c_int64(n), C.byref(r), _abi.ptr(it), _abi.ptr(pn),
                                       co.ctypes.data_as(C.c_void_p), _abi.ptr(ci), oo.ctypes.data_as(C.c_void_p), _abi.ptr(oi), C.c_int64(cap))
        assert rc == 0, rc
        return dict(iteration=it[:n], primary_num=pn[:n], cover_off=co, cover_ids=ci[:co[-1]], overlap_off=oo, overlap_ids=oi[:oo[-1]])

    def call_gt(self, windows, windows_per_cand, support_off, support_ids, reads=None):
        w = np.ascontiguousarray(windows, dtype=_abi.WINDOW_DTYPE)
        so = np.ascontiguousarray(support_off, dtype=np.int64)
        si = np.ascontiguousarray(support_ids, dtype=np.int32)
        n = len(so) - 1
        r, keep = _abi.make_reads_cols(reads)
        out = np.zeros(max(n, 1), dtype=_abi.GENO_DTYPE)
        rc = self.L.emul_call_gt(w.ctypes.data_as(C.c_void_p), C.c_int64(n), C.c_int32(windows_per_cand), C.byref(r),
                                 so.ctypes.data_as(C.c_void_p), _abi.ptr(si), out.ctypes.data_as(C.c_void_p))
        assert rc == 0, rc
        return out[:n]

    def cal_gl(self, c0, c1):
        c0 = np.ascontiguousarray(c0, dtype=np.int32)
        c1 = np.ascontiguousarray(c1, dtype=np.int32)
        out = np.zeros(len(c0), dtype=_abi.GENO_DTYPE)
        self.L.emul_cal_gl(_abi.ptr(c0), _abi.ptr(c1), C.c_int64(len(c0)), out.ctypes.data_as(C.c_void_p))
        return out


@pytest.fixture(scope="module")
def emul_so(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "emul_genotype.cpp")
    so = str(tmp_path_factory.mktemp("emul") / "libemul_genotype.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, src])
    return so


@pytest.fixture
def emul_engine(emul_so):
    prev = runtime._engine
    runtime.set_engine(EmulGenotypeEngine(emul_so))
    yield
    runtime.set_engine(prev)


@pytest.mark.parametrize("i", range(len(gg.data()["overlap_cover"])))
def test_overlap_cover_golden(emul_engine, i):
    gg.check_overlap_cover(gg.data()["overlap_cover"][i])


@pytest.mark.parametrize("i", range(len(gg.data()["assign_gt"])))
def test_assign_gt_golden(emul_engine, i):
    gg.check_assign_gt(gg.data()["assign_gt"][i])


def test_call_gt_golden(emul_engine, tmp_path):
    path = str(tmp_path) + "/"
    idx = gg.write_reads_workdir(path)
    for case in gg.data()["call_gt"]:
        gg.check_call_gt(case, path, idx)


def test_half_units_compare_like_the_bounds():
    v = [0, 3, 2.5, 100.3, 7.0, -1.5, -0.2]
    h = cuteSV_genotype.half_units(v)
    for x, x2 in zip(v, h.tolist()):
        for r in range(-4, 110):
            assert (r <= x) == (2 * r <= x2) and (r < x) == (2 * r < x2) and (r >= x) == (2 * r >= x2), (x, r)


def test_cal_cipos_and_threshold_ref_count():
    assert cuteSV_genotype.cal_CIPOS(10.0, 4) == "-9,9"
    assert cuteSV_genotype.cal_CIPOS(0.0, 7) == "-0,0"
    assert [cuteSV_genotype.threshold_ref_count(n) for n in (0, 2, 3, 5, 6, 15, 16, 40)] == [0, 40, 27, 45, 42, 105, 80, 200]
