"""CPU: SA:Z text to SA rows.  The statement of sa_core.h (the strip walk of k_sa_count / k_sa_fill and the per-entry parse),
compiled for the host (tests/emul/emul_sa.cpp), against the native BAM decoder's host reduction (bamio.BamReader) of the same tags
written into a BAM; its int32 rejections; and _abi.device_packet's SA text keys."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import sa_text_util as sat
from cutesv_b200 import _abi, bamio
from test_device_inputs_cpu import FakeDev
from test_device_names_cpu import named_packet

SA_BAD_OFF, SA_BAD_POS, SA_BAD_MAPQ, SA_BAD_CIGAR = 1, 2, 4, 8


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    bamio.build()
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "emul_sa.cpp")
    so = str(tmp_path_factory.mktemp("emul") / "libemul_sa.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-fPIC", "-shared", "-o", so, src])
    L = C.CDLL(so)
    L.emul_sa_reduce.restype = C.c_uint32
    return L


def _p(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


def emul_reduce(L, text, off, names=sat.NAMES):
    nb, noff, nid = sat.name_table(names)
    n = len(off) - 1
    cap = max(len(text) // 5 + 1, 1)
    sa_off = np.zeros(n + 1, np.int64)
    cols = np.zeros((7, cap), np.int32)
    nr = C.c_int64(0)
    bad = L.emul_sa_reduce(_p(nb, C.c_uint8), _p(noff, C.c_int64), _p(nid, C.c_int32), C.c_int64(len(nid)), _p(text, C.c_uint8),
                           _p(off, C.c_int64), C.c_int64(len(text)), C.c_int64(n), _p(sa_off, C.c_int64), _p(cols, C.c_int32), C.c_int64(cap),
                           C.byref(nr))
    assert nr.value <= cap
    return bad, sa_off, {f: cols[k, :nr.value] for k, f in enumerate(_abi.SA_FIELDS)}


def _check_equal(L, values, tmp_path):
    path = str(tmp_path / "sa.bam")
    sat.write_bam(path, values)
    want_off, want = sat.host_reduce(path)
    text, off = sat.text_arrays(values)
    bad, got_off, got = emul_reduce(L, text, off)
    assert bad == 0
    assert np.array_equal(got_off, want_off), np.flatnonzero(got_off != want_off)[:5]
    for f in _abi.SA_FIELDS:
        assert np.array_equal(got[f], want[f]), (f, np.flatnonzero(got[f] != want[f])[:5])
    return want_off, want


def test_adversarial_values_equal_the_host_reduction(emul, tmp_path):
    values = sat.adversarial_values()
    off, sa = _check_equal(emul, values, tmp_path)
    counts = np.diff(off)
    assert counts[values.index("chr2,1,+,5M,1,0;" * 1000)] == 1000
    assert counts[values.index("chr2,5,-,10M,3,1")] == 0 and counts[values.index(";;")] == 0
    assert counts[values.index("chr1,100,+,50M;")] == 0 and counts[values.index("chr1,100,+,50M,7;")] == 1
    assert (sa["chrom"] == -1).any() and (sa["chrom"] == sat.CHROM_ID["chr10"]).any()
    assert (sa["pos0"] < 0).any() and (sa["mapq"] == 255).any() and (sa["ref_span"] == 2147483647).any()


@pytest.mark.parametrize("seed", range(6))
def test_seeded_values_equal_the_host_reduction(emul, tmp_path, seed):
    _check_equal(emul, sat.random_values(seed, 400), tmp_path)


@pytest.mark.parametrize("value,bit", [
    ("chr1,2147483648,+,5M,1,0;", SA_BAD_POS), ("chr1,-2147483647,+,5M,1,0;chr1,-2147483648,+,5M,1,0;", SA_BAD_POS),
    ("chr1,99999999999999999999999,+,5M,1,0;", SA_BAD_POS), ("chr1,1,+,5M,2147483648,0;", SA_BAD_MAPQ),
    ("chr1,1,+,5M,-2147483649,0;", SA_BAD_MAPQ), ("chr1,1,+,2147483648M,1,0;", SA_BAD_CIGAR),
    ("chr1,1,+,2147483648I,1,0;", SA_BAD_CIGAR), ("chr1,1,+,2000000000M2000000000D,1,0;", SA_BAD_CIGAR),
    ("chr1,1,+,99999999999999999999999999S,1,0;", SA_BAD_CIGAR),
])
def test_numbers_outside_int32_are_rejected(emul, value, bit):
    text, off = sat.text_arrays(["chr1,1,+,5M,1,0;", value])
    assert emul_reduce(emul, text, off)[0] == bit
    # the same number in an entry that is dropped (unterminated, after a NUL, too few fields) is no error
    for v in (value[:-1], "\0" + value, value.rsplit(",", 2)[0] + ";"):
        text, off = sat.text_arrays([v])
        assert emul_reduce(emul, text, off)[0] == 0, v


def test_bad_offsets_are_rejected(emul):
    text, off = sat.text_arrays(["chr1,1,+,5M,1,0;"] * 3)
    for k, v in ((0, -1), (2, off[1] - 1), (3, len(text) + 1)):
        o = off.copy()
        o[k] = v
        assert emul_reduce(emul, text, o)[0] == SA_BAD_OFF


def test_name_lookup_on_many_names(emul):
    names = ["ctg%d" % k for k in range(100_000)]
    srt = sorted(names)
    vals = ["%s,%d,+,5M,1,0;" % (nm, k) for k, nm in enumerate(names[::997])] + ["ctg100000,1,+,5M,1,0;ctg,1,+,5M,1,0;ctg99999x,1,+,5M,1,0;"]
    text, off = sat.text_arrays(vals)
    bad, sa_off, sa = emul_reduce(emul, text, off, names)
    assert bad == 0
    assert sa["chrom"].tolist() == [srt.index(nm) for nm in names[::997]] + [-1, -1, -1]


# ---- the packet keys ----

def test_device_packet_takes_sa_text():
    pk = named_packet()
    n = len(pk["chrom"])
    del pk["sa"], pk["sa_off"]
    pk["sa_text"], pk["sa_text_off"] = FakeDev(17, "|u1"), FakeDev(n + 1, "<i8")
    d = _abi.device_packet(pk, 0)
    assert d.sa_text is not None and d.sa_text.n_records == n and d.sa_text.n_bytes == 17
    with pytest.raises(ValueError, match="one or the other"):
        _abi.device_packet(dict(pk, sa_off=FakeDev(n + 1, "<i8")), 0)
    with pytest.raises(ValueError, match="go together"):
        _abi.device_packet(dict(pk, sa_text=None), 0)
    with pytest.raises(ValueError, match="n \\+ 1"):
        _abi.device_packet(dict(pk, sa_text_off=FakeDev(n, "<i8")), 0)
    with pytest.raises(TypeError, match="sa_text"):
        _abi.device_packet(dict(pk, sa_text=FakeDev(17, "<i4")), 0)
    assert _abi.device_packet(named_packet(), 0).sa_text is None
    host = {f: np.zeros(3, np.int32) for f in _abi.READ_FIELDS}
    host.update(cigar_off=np.zeros(4, np.int64), cigar=np.zeros(0, np.uint32), sa_text=np.zeros(0, np.uint8), sa_text_off=np.zeros(4, np.int64))
    with pytest.raises(ValueError, match="device packets only"):
        _abi.device_packet(host, 0)
