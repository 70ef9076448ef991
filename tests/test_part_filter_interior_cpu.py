"""CPU: the density filter's strip pass for every strip length from 1 to 64 and every radius rb from 1 to 64, on the
test-only emulator tests/emul/emul_part_strip.cpp, against a numpy evaluation of the rule.  Interior strips (every
window inside the partition, rb <= strip length) take core.h's straight-line path, the others the generic one with the
halo; rb > strip length and the strips next to the partition's ends always take the generic one."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_part_filter_strip_cpu import PAD, _halo, _ptr, _reference, _u32


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "emul_part_strip.cpp")
    so = str(tmp_path_factory.mktemp("emul") / "libemul_part_strip.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, src])
    L = C.CDLL(so)
    L.emul_part_strip.restype = C.c_uint32
    return L


def _n_interior(per, rb):
    return sum(1 for t in range(256) if rb <= per and t * per - rb >= 0 and t * per + per - 1 + rb < 256 * per)


def _run(lib, hist, rb, need, hl, hr):
    per = len(hist) // 256
    hist, hl, hr = _u32(hist), _u32(hl), _u32(hr)
    keep = np.zeros(len(hist), np.uint8)
    off = np.zeros(len(hist), np.uint32)
    n_int = C.c_int(-1)
    total = lib.emul_part_strip(_ptr(hist), C.c_int(per), C.c_int(rb), C.c_uint32(need), _ptr(hl), _ptr(hr), _ptr(keep), _ptr(off),
                                C.byref(n_int))
    k_ref, o_ref, t_ref = _reference(hist, rb, need, hl, hr)
    assert total == t_ref, (per, rb)
    np.testing.assert_array_equal(keep.astype(bool), k_ref, err_msg="per %d rb %d" % (per, rb))
    np.testing.assert_array_equal(off[k_ref], o_ref[k_ref], err_msg="per %d rb %d" % (per, rb))
    assert n_int.value == _n_interior(per, rb)
    return n_int.value


@pytest.mark.parametrize("per", range(1, 65))
def test_every_strip_length_and_radius(lib, per):
    """Random histograms dense enough that windows straddle `need`, rb from 1 to 64: the interior path runs for rb <= per
    (strips 1 .. 254 when rb divides into one strip), the generic one for every other strip."""
    rng = np.random.default_rng(1000 + per)
    interior = 0
    for rb in range(1, PAD + 1):
        density = float(rng.choice([0.05, 0.4, 2.0]))
        hist = rng.poisson(density, 256 * per)
        need = int(rng.integers(2, 4 + int(density * (2 * rb + 1))))
        interior += _run(lib, hist, rb, need, _halo(rng, rb, density), _halo(rng, rb, density))
    assert interior > 0


@pytest.mark.parametrize("per", [1, 3, 7, 16, 33, 64])
def test_windows_at_the_interior_edge(lib, per):
    """Signatures that only a window reaching exactly rb buckets into the neighbouring strip brings to `need`, with rb at
    and around the strip length, in the strips next to the partition's ends (generic) and inside (interior)."""
    rng = np.random.default_rng(2000 + per)
    bp = 256 * per
    for rb in sorted({1, max(1, per - 1), per, min(PAD, per + 1), min(PAD, 2 * per)}):
        for trial in range(4):
            hist = np.zeros(bp, np.int64)
            hl, hr = np.zeros(PAD, np.int64), np.zeros(PAD, np.int64)
            hl[rb:] = hr[rb:] = 1000003
            for t in (0, 1, 2, 127, 253, 254, 255):   # the ends' strips and their neighbours
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
