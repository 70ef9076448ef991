"""CPU: the density filter's strip pass with 512 strips per partition, the layout of the 512-thread k_part_filter, on the
test-only emulator tests/emul/emul_part_strip_nt.cpp, against a numpy evaluation of the rule.  Strips hold 32 buckets
at W = 22 and 16 at W = 21, one at W = 17; at W = 16 (256 buckets) the threads at or past 256 own an empty strip.  Radii
longer than the strip leave no strip interior."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_part_filter_strip_cpu import PAD, _halo, _ptr, _reference, _u32

NT = 512


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "emul_part_strip_nt.cpp")
    so = str(tmp_path_factory.mktemp("emul") / "libemul_part_strip_nt.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, src])
    L = C.CDLL(so)
    L.emul_part_strip_nt.restype = C.c_uint32
    return L


def _n_interior(bp, rb):
    per = max(1, bp // NT)
    return sum(1 for t in range(min(NT, bp)) if rb <= per and t * per - rb >= 0 and t * per + per - 1 + rb < bp)


def _run(lib, hist, rb, need, hl, hr):
    """The emulator against the rule; returns the number of interior strips."""
    bp = len(hist)
    hist, hl, hr = _u32(hist), _u32(hl), _u32(hr)
    keep = np.zeros(bp, np.uint8)
    off = np.zeros(bp, np.uint32)
    n_int = C.c_int(-1)
    total = lib.emul_part_strip_nt(_ptr(hist), C.c_int(bp), C.c_int(NT), C.c_int(rb), C.c_uint32(need), _ptr(hl), _ptr(hr),
                                   _ptr(keep), _ptr(off), C.byref(n_int))
    msg = "bp %d rb %d" % (bp, rb)
    k_ref, o_ref, t_ref = _reference(hist, rb, need, hl, hr)
    assert total == t_ref, msg
    np.testing.assert_array_equal(keep.astype(bool), k_ref, err_msg=msg)
    np.testing.assert_array_equal(off[k_ref], o_ref[k_ref], err_msg=msg)
    assert n_int.value == _n_interior(bp, rb), msg
    return n_int.value


@pytest.mark.parametrize("bp", [256, 512, 1024, 2048, 4096, 8192, 16384])
def test_random_histograms_512(lib, bp):
    """Sparse and dense random histograms for every partition width (W = 16 .. 22), rb from 1 to 64; at bp = 256 half
    the strips are empty."""
    rng = np.random.default_rng(bp)
    for rb in list(range(1, 9)) + [15, 16, 17, 31, 32, 33, 63, 64]:
        for density in (0.01, 0.3, 2.0):
            hist = rng.poisson(density, bp)
            need = int(rng.integers(3, 12))
            _run(lib, hist, rb, need, _halo(rng, rb, density), _halo(rng, rb, density))


@pytest.mark.parametrize("bp", [256, 512, 16384])
def test_partition_ends_and_big_buckets_512(lib, bp):
    """Singletons at both ends completed by the halo only, buckets of more than 64 signatures, need = 1 and need above
    every window, an empty partition."""
    rng = np.random.default_rng(300 + bp)
    for rb in (1, 2, 33, 64):
        hist = np.zeros(bp, np.int64)
        hl, hr = np.zeros(PAD, np.int64), np.zeros(PAD, np.int64)
        hl[rb:] = hr[rb:] = 1000003
        hist[0] += 1
        hist[bp - 1] += 1
        hl[rb - 1] += 2
        hr[rb - 1] += 1   # one short on the right
        _run(lib, hist, rb, 3, hl, hr)
    hist = rng.poisson(0.05, bp)
    hist[rng.integers(0, bp, 20)] += rng.integers(65, 7000, 20)
    for rb, need in ((1, 1), (4, 10), (64, 5), (64, 1 << 30)):
        _run(lib, hist, rb, need, _halo(rng, rb, 0.5), _halo(rng, rb, 0.5))
    _run(lib, np.zeros(bp, np.int64), 64, 3, np.zeros(PAD), np.zeros(PAD))


@pytest.mark.parametrize("per", [1, 2, 3, 7, 16, 17, 31, 32])
def test_every_radius_512(lib, per):
    """Every rb from 1 to 64 over 512 strips: the interior path for rb <= per, the generic one for every strip when rb is
    longer than the strip (per = 1, 2, 16: W = 17, 18, 21; per = 32: W = 22)."""
    rng = np.random.default_rng(4000 + per)
    interior = 0
    for rb in range(1, PAD + 1):
        density = float(rng.choice([0.05, 0.4, 2.0]))
        hist = rng.poisson(density, NT * per)
        need = int(rng.integers(2, 4 + int(density * (2 * rb + 1))))
        n = _run(lib, hist, rb, need, _halo(rng, rb, density), _halo(rng, rb, density))
        if rb > per:
            assert n == 0
        interior += n
    assert interior > 0


@pytest.mark.parametrize("per", [1, 16, 32])
def test_windows_at_the_interior_edge_512(lib, per):
    """Signatures that only a window reaching exactly rb buckets into the neighbouring strip brings to `need`, in the
    strips next to the partition's ends and the middle strips 255 and 256, with rb at and around the strip length."""
    rng = np.random.default_rng(5000 + per)
    bp = NT * per
    for rb in sorted({1, max(1, per - 1), per, min(PAD, per + 1), min(PAD, 2 * per)}):
        for trial in range(4):
            hist = np.zeros(bp, np.int64)
            hl, hr = np.zeros(PAD, np.int64), np.zeros(PAD, np.int64)
            hl[rb:] = hr[rb:] = 1000003
            for t in (0, 1, 2, 255, 256, 509, 510, 511):
                for b in (t * per, t * per + per - 1):
                    hist[b] += 1
                    lo, hi = b - rb, b + rb
                    if trial % 2 == 0 and lo >= 0:
                        hist[lo] += 2
                    elif hi < bp:
                        hist[hi] += 2
            hist[rng.integers(0, bp, 16)] += 1
            hl[rb - 1] += 1
            hr[rb - 1] += 2
            _run(lib, hist, rb, 3, hl, hr)
