"""CPU: named device packets and the device's read-name and INS-tie routines.  _abi.device_packet's handling of names / name_off
with stand-in __cuda_array_interface__ objects; the key-word, comparison and tie-group routines of names_core.h compiled for the
host (tests/emul/emul_names.cpp) and composed as the device composes them, against Python's sorted() and cli.ins_tie_swaps."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import name_util
from cutesv_b200 import _abi, cli
from test_device_extract_cpu import addr, fake_packet
from test_device_inputs_cpu import FakeDev

# ---- _abi.device_packet with names ----


def named_packet(n=5, n_bytes=40, **over):
    pk = fake_packet(n=n)
    del pk["read_id"]
    pk["names"] = FakeDev(n_bytes, "|u1", addr=0x70000)
    pk["name_off"] = FakeDev(n + 1, "<i8", addr=0x80000)
    pk.update(over)
    return pk


def test_named_packet_carries_the_name_columns():
    d = _abi.device_packet(named_packet(), 0)
    reads, cig, n_cig, sa, seq = d   # unpacks like an unnamed packet
    assert reads.n == 5 and addr(reads.read_id) is None and n_cig == 40 and seq is not None
    assert d.names.n_bytes == 40 and addr(d.names.names) == 0x70000 and addr(d.names.name_off) == 0x80000
    assert _abi.device_packet(fake_packet(), 0).names is None
    assert _abi.device_packet(named_packet(names=FakeDev(40, "<u1", addr=0x70000)), 0).names.n_bytes == 40
    assert _abi.device_packet(named_packet(seq_off=None, seq4=None), 0).names is not None   # names without bases


def test_empty_named_packet():
    d = _abi.device_packet(fake_packet(n=0, n_cigar=0, n_sa=0, n_bytes=0) | {"read_id": None, "names": FakeDev(0, "|u1"),
                                                                            "name_off": FakeDev(1, "<i8", addr=0x80000)}, 0)
    assert d[0].n == 0 and d.names.n_bytes == 0 and addr(d.names.names) is None


@pytest.mark.parametrize("over, exc, msg", [
    (dict(read_id=FakeDev(5)), ValueError, "read_id"),
    (dict(names=FakeDev(40, "<i4")), TypeError, "names"),
    (dict(name_off=FakeDev(6, "<i4")), TypeError, "name_off"),
    (dict(name_off=FakeDev(5, "<i8")), ValueError, "name_off"),
    (dict(name_off=FakeDev(7, "<i8")), ValueError, "name_off"),
    (dict(names=FakeDev(40, "|u1", shape=(20, 2))), TypeError, "names"),
    (dict(name_off=FakeDev(6, "<i8", strides=(16,))), TypeError, "name_off"),
    (dict(names=None), ValueError, "go together"),
    (dict(name_off=None), ValueError, "go together"),
    (dict(names=np.zeros(40, np.uint8)), ValueError, "all device or all host"),
    (dict(name_off=np.zeros(6, np.int64)), ValueError, "all device or all host"),
    (dict(names=FakeDev(40, "|u1", device=1)), ValueError, "device 1"),
])
def test_named_packet_rejections(over, exc, msg):
    with pytest.raises(exc, match=msg):
        _abi.device_packet(named_packet(**over), 0)


def test_names_on_a_host_packet_are_refused():
    host = {f: np.zeros(3, np.int32) for f in _abi.READ_FIELDS if f != "read_id"}
    host.update(cigar_off=np.zeros(4, np.int64), sa_off=np.zeros(4, np.int64), cigar=np.zeros(0, np.uint32),
                sa={f: np.zeros(0, np.int32) for f in _abi.SA_FIELDS})
    b, off = name_util.pack_names(["r1", "r2", "r1"])
    with pytest.raises(ValueError, match="device packets only"):
        _abi.device_packet(dict(host, names=b, name_off=off), 0)


# ---- the routines of names_core.h, compiled for the host ----


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "emul_names.cpp")
    so = str(tmp_path_factory.mktemp("emul") / "libemul_names.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-fPIC", "-shared", "-o", so, src])
    L = C.CDLL(so)
    L.emul_name_ranks.restype = C.c_int64
    L.emul_tie_order.restype = C.c_int64
    return L


def emul_ranks(L, names):
    b, off = name_util.pack_names(names)
    rank = np.full(len(names), -1, np.int32)
    nd = L.emul_name_ranks(b.ctypes.data_as(C.c_void_p) if b.size else None, off.ctypes.data_as(C.c_void_p), C.c_int64(len(names)),
                           rank.ctypes.data_as(C.c_void_p))
    return rank, nd


@pytest.mark.parametrize("which", sorted(name_util.name_sets()))
def test_lsd_name_ranks_equal_python_sorted(emul, which):
    names = name_util.name_sets(3)[which]
    rng = np.random.default_rng(len(names))
    names = [names[i] for i in rng.permutation(len(names))]
    rank, nd = emul_ranks(emul, names)
    want = name_util.dense_ranks(names)
    assert nd == len(set(names))
    assert np.array_equal(rank, want)


def test_name_words_and_compare_details(emul):
    # a prefix sorts first even when the longer name continues with NUL bytes; zero padding alone would tie them
    names = ["ab", "ab\x00", "ab\x00\x00\x00\x00\x00\x00\x00", "ab\x00\x00\x00\x00\x00\x00", "a", "", "\x00"]
    rank, nd = emul_ranks(emul, names)
    assert nd == 7 and np.array_equal(rank, name_util.dense_ranks(names))
    assert emul_ranks(emul, [])[1] == 0


def tie_columns(seed, n=3000):
    """INS columns with many ties on (contig, int(pos), len, read): few positions, lengths and reads; strings from a tiny alphabet
    so that equal strings occur inside groups too."""
    rng = np.random.default_rng(seed)
    chrom = rng.integers(0, 2, n).astype(np.int32)
    a = (rng.integers(0, 40, n) * 2 + rng.integers(0, 2, n)).astype(np.int32)
    b = rng.integers(30, 33, n).astype(np.int32)
    rid = rng.integers(0, 6, n).astype(np.int32)
    seqs = ["".join("ACGT"[j] for j in rng.integers(0, 2, int(rng.integers(1, 12)))) for _ in range(n)]
    return chrom, a, b, rid, seqs


def emul_tie_perm(L, chrom, a, b, rid, seqs):
    """content[row] after the device's tie ordering: the original row whose content lands on `row`."""
    n = len(chrom)
    order, same = cli._tie_runs(chrom, a, b, rid)
    tie = np.zeros(n, np.uint8)
    tie[1:] = same
    perm = np.ascontiguousarray(order, dtype=np.uint32)
    bts, off = name_util.pack_names(seqs)
    start = np.ascontiguousarray(off[:-1])
    ln = np.diff(off).astype(np.int32)
    content = np.arange(n, dtype=np.int32)
    moved = L.emul_tie_order(perm.ctypes.data_as(C.c_void_p), tie.ctypes.data_as(C.c_void_p), C.c_int64(n), bts.ctypes.data_as(C.c_void_p),
                             start.ctypes.data_as(C.c_void_p), ln.ctypes.data_as(C.c_void_p), content.ctypes.data_as(C.c_void_p))
    return content, moved


def host_swap_perm(chrom, a, b, rid, seqs):
    content = np.arange(len(chrom), dtype=np.int32)
    for i, j in cli.ins_tie_swaps(chrom, a, b, rid, seqs):
        content[i], content[j] = content[j], content[i]
    return content


@pytest.mark.parametrize("seed", range(8))
def test_tie_group_order_equals_host_swaps(emul, seed):
    chrom, a, b, rid, seqs = tie_columns(seed, 300 + 700 * seed)
    got, moved = emul_tie_perm(emul, chrom, a, b, rid, seqs)
    want = host_swap_perm(chrom, a, b, rid, seqs)
    assert np.array_equal(got, want)
    assert moved == int((want != np.arange(len(want))).sum()) and moved > 0


def test_tie_groups_larger_than_a_warp(emul):
    n = 200   # one read, one position, one length: a single group of 200 rows
    rng = np.random.default_rng(5)
    chrom, a, b, rid = (np.zeros(n, np.int32) for _ in range(4))
    seqs = ["".join("ACGT"[j] for j in rng.integers(0, 4, 6)) for _ in range(n)]
    got, moved = emul_tie_perm(emul, chrom, a, b, rid, seqs)
    assert np.array_equal(got, host_swap_perm(chrom, a, b, rid, seqs))
    assert [seqs[i] for i in got] == sorted(seqs)
