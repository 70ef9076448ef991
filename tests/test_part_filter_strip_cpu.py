"""CPU: the density filter's per-strip rule (core.h pf_strip_flags / pf_strip_offsets, the code k_part_filter runs) on the
test-only emulator tests/emul/emul_part_filter.cpp, against a numpy evaluation of the rule: bucket b of a partition is
kept when it holds a signature and the buckets [b - rb, b + rb], read through the neighbours' halo past the partition's
ends, hold >= need signatures; kept buckets get exclusive offsets in bucket order."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

PAD = 64   # BKT_PAD: the largest rb and the halo length


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "emul_part_filter.cpp")
    so = str(tmp_path_factory.mktemp("emul") / "libemul_part_filter.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, src])
    L = C.CDLL(so)
    L.emul_part_filter.restype = C.c_uint32
    return L


def _u32(x):
    return np.ascontiguousarray(x, dtype=np.uint32)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _reference(hist, rb, need, hl, hr):
    ext = np.concatenate([hl[:rb][::-1], hist, hr[:rb]]).astype(np.int64)
    pre = np.concatenate([[0], np.cumsum(ext)])
    b = np.arange(len(hist))
    win = pre[b + 2 * rb + 1] - pre[b]
    keep = (hist > 0) & (win >= need)
    kept = np.where(keep, hist, 0).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(kept)])[:-1]
    return keep, off, int(kept.sum())


def _run(lib, hist, rb, need, hl, hr):
    per = len(hist) // 256
    hist, hl, hr = _u32(hist), _u32(hl), _u32(hr)
    keep = np.zeros(len(hist), np.uint8)
    off = np.zeros(len(hist), np.uint32)
    total = lib.emul_part_filter(_ptr(hist), C.c_int(per), C.c_int(rb), C.c_uint32(need), _ptr(hl), _ptr(hr), _ptr(keep), _ptr(off))
    k_ref, o_ref, t_ref = _reference(hist, rb, need, hl, hr)
    assert total == t_ref
    np.testing.assert_array_equal(keep.astype(bool), k_ref)
    np.testing.assert_array_equal(off[k_ref], o_ref[k_ref])


def _halo(rng, rb, density):
    """Halo counts for j < rb and junk beyond, which the rule must never read."""
    h = rng.poisson(density, PAD).astype(np.uint32)
    h[rb:] = 1000003
    return h


@pytest.mark.parametrize("per", [1, 2, 4, 8, 16, 32, 64])
def test_random_histograms(lib, per):
    """Sparse and dense random histograms for every strip length (W = 16 .. 22), rb from 1 to 64."""
    rng = np.random.default_rng(per)
    for rb in list(range(1, 9)) + [15, 16, 17, 31, 32, 33, 63, 64]:
        for density in (0.01, 0.3, 2.0):
            hist = rng.poisson(density, 256 * per)
            need = int(rng.integers(3, 12))
            _run(lib, hist, rb, need, _halo(rng, rb, density), _halo(rng, rb, density))


@pytest.mark.parametrize("per", [1, 2, 64])
def test_windows_across_strips_and_partition_ends(lib, per):
    """Lone signatures that only the window reaching several strips, or the halo past either end, brings to `need`."""
    rng = np.random.default_rng(100 + per)
    bp = 256 * per
    for rb in (1, 2, 63, 64):
        for trial in range(6):
            hist = np.zeros(bp, np.int64)
            hl, hr = np.zeros(PAD, np.int64), np.zeros(PAD, np.int64)
            hl[rb:] = hr[rb:] = 1000003
            # a pair of buckets exactly rb apart, anywhere, including across strip boundaries
            for _ in range(8):
                b = int(rng.integers(0, bp))
                hist[b] += 1
                if b + rb < bp:
                    hist[b + rb] += 2
            # singletons at both ends completed by the halo only, at its farthest reach
            hist[0] += 1
            hist[bp - 1] += 1
            hl[rb - 1] += 2
            hr[rb - 1] += 2
            if trial % 2:   # halo exactly one short on one side
                hl[rb - 1] -= 1
            _run(lib, hist, rb, 3, hl, hr)


def test_big_buckets_and_extremes(lib):
    """Buckets of more than 64 survivors (the counting-sort path), need = 1 and need above every window, empty input."""
    rng = np.random.default_rng(7)
    for per in (1, 8, 64):
        bp = 256 * per
        hist = rng.poisson(0.05, bp)
        hist[rng.integers(0, bp, 20)] += rng.integers(65, 7000, 20)
        for rb, need in ((1, 1), (4, 10), (64, 5), (64, 1 << 30)):
            _run(lib, hist, rb, need, _halo(rng, rb, 0.5), _halo(rng, rb, 0.5))
        _run(lib, np.zeros(bp, np.int64), 64, 3, np.zeros(PAD), np.zeros(PAD))
