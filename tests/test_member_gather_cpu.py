"""CPU: k_select_heads' record-mode bit tests (core.h chain_head / chain_member / chain_size_class, the code the kernel
runs) on the test-only emulator tests/emul/emul_member_gather.cpp, against a numpy chain split.  A tile of 2048 sorted
elements reads its link mask with a halo of ceil(need / 32) + 1 words before it and max(ceil(need / 32), 3) + 1 after
it: element i of the tile is a member of a kept cluster when its chain run holds >= need elements, wherever the run's head
lies, and a head's size class is its member count up to 32, 33 up to REST_SPLIT = 64 members and 34 beyond.  The mask
sits between junk words (all links set), so a routine that reads past the halo changes the result."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

TILE = 2048
SPLIT = 64        # REST_SPLIT
JUNK = 80         # junk words on either side of the mask (> the largest halo)
NEEDS = (2, 3, 10, 31, 32, 33, 64, 65, 2016)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "emul_member_gather.cpp")
    so = str(tmp_path_factory.mktemp("emul") / "libemul_member_gather.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, src])
    L = C.CDLL(so)
    L.emul_member_gather.restype = None
    return L


def _halos(need):
    w = (need + 31) // 32
    return w + 1, max(w, (SPLIT + 32) // 32) + 1


def _links(n_total, runs):
    """Link bits of n_total sorted elements (bit i: element i is chained to element i - 1): every element a cluster of
    one except the planted runs (start, length), which must not touch each other."""
    link = np.zeros(n_total, bool)
    for s, m in runs:
        assert s >= 0 and s + m <= n_total and not link[s] and not link[s + 1:s + m].any()
        assert s + m == n_total or not link[s + m]
        link[s + 1:s + m] = True
    return link


def _reference(link, n, need):
    """member, head and size class of elements [0, n) from the chain split."""
    lk = link[:n].copy()
    lk[0] = False
    run = np.cumsum(~lk) - 1
    size = np.bincount(run)
    m = size[run]
    member = m >= need
    head = ~lk & member
    cls = np.where(head, np.where(m <= 32, m, np.where(m <= SPLIT, 33, 34)), 0)
    return member, head, cls


def _check(lib, link, n, need):
    """Every tile of [0, n) through the emulator, its mask read from link as the kernel reads it."""
    back, fwd = _halos(need)
    member, head, cls = _reference(link, n, need)
    tiles = (n + TILE - 1) // TILE
    bits_all = np.zeros(len(link) + 64 * (back + fwd + 64), bool)
    bits_all[1:n] = link[1:n]   # element 0 and elements >= n are never linked
    for k in range(tiles):
        lo = k * TILE - 32 * back
        idx = np.arange(lo, k * TILE + TILE + 32 * fwd)
        bits = np.where((idx > 0) & (idx < n), bits_all[np.clip(idx, 0, None)], False)
        words = np.packbits(bits.astype(np.uint8), bitorder="little").view("<u4")
        buf = np.concatenate([np.full(JUNK, 0xFFFFFFFF, np.uint32), words, np.full(JUNK, 0xFFFFFFFF, np.uint32)])
        buf = np.ascontiguousarray(buf, dtype=np.uint32)
        got_m = np.zeros(TILE, np.uint8)
        got_h = np.zeros(TILE, np.uint8)
        got_c = np.zeros(TILE, np.uint8)
        nv = min(TILE, n - k * TILE)
        lib.emul_member_gather(C.c_void_p(buf.ctypes.data + 4 * JUNK), C.c_int(back), C.c_int(TILE), C.c_int(nv), C.c_int(need),
                               C.c_int(SPLIT), got_m.ctypes.data_as(C.c_void_p), got_h.ctypes.data_as(C.c_void_p),
                               got_c.ctypes.data_as(C.c_void_p))
        sl = slice(k * TILE, k * TILE + nv)
        np.testing.assert_array_equal(got_m[:nv].astype(bool), member[sl], err_msg="member, tile %d" % k)
        np.testing.assert_array_equal(got_h[:nv].astype(bool), head[sl], err_msg="head, tile %d" % k)
        np.testing.assert_array_equal(got_c[:nv], cls[sl], err_msg="size class, tile %d" % k)
        assert not got_m[nv:].any() and not got_h[nv:].any()
    return int(member.sum()), int(head.sum())


@pytest.mark.parametrize("need", NEEDS)
def test_runs_around_need(lib, need):
    """Runs of need - 1, need and need + 1 elements inside tiles, across an edge by one element on either side, and from
    more than need elements before a tile."""
    gap = need + 8
    runs = []
    s = 5
    for m in (need - 1, need, need + 1):
        if m >= 1:
            runs.append((s, m))
            s += m + gap
    step = TILE * (2 + (2 * need + 40) // TILE)   # a tile edge that clears every run so far
    e = step + TILE * (s // TILE)
    for m in (need - 1, need, need + 1):   # the last element in the next tile, then the first element in the previous one
        if m >= 2:
            runs.append((e - m + 1, m))
            e += step
            runs.append((e - 1, m))
            e += step
    for m in (need, need + 1, 2 * need + 40):   # starts need + 3 elements before a tile
        runs.append((e - need - 3, m))
        e += step
    n = e + TILE + 77
    link = _links(n, runs)
    members, heads = _check(lib, link, n, need)
    kept = [m for _, m in runs if m >= need]
    assert heads == len(kept) and members == sum(kept)


@pytest.mark.parametrize("need", (2, 10, 32, 33))
def test_size_class_edges(lib, need):
    """Heads of 31 .. 33, 63 .. 65 and 127 .. 129 members, inside a tile and with their runs crossing the next tile's edge,
    including a head on a tile's last position."""
    runs = []
    s = 3
    for m in (31, 32, 33, 63, 64, 65, 127, 128, 129):
        runs.append((s, m))
        s += m + 40
    e = 2 * TILE
    for m in (31, 32, 33, 63, 64, 65, 127, 128, 129):
        runs.append((e - 1, m))
        e += TILE
        runs.append((e - m // 2, m))
        e += TILE
    n = e + 500
    link = _links(n, runs)
    _check(lib, link, n, need)


@pytest.mark.parametrize("need", (10, 33, 2016))
def test_runs_over_several_tiles(lib, need):
    """Runs that span three tiles, end on a tile's last element or start on a tile's first one, and a domain that ends
    inside a tile and inside a run."""
    runs = [(TILE - 5, 2 * TILE + 10), (4 * TILE - need, need), (5 * TILE, need), (7 * TILE - 1, 2)]
    n = 9 * TILE + 100
    runs.append((n - need // 2 - 1, need // 2 + 1))   # a run the domain's end cuts: kept only when need is small
    link = _links(n, runs)
    _check(lib, link, n, need)


@pytest.mark.parametrize("seed", range(4))
def test_random_runs(lib, seed):
    """Random run lengths (geometric, a few long runs), random need, a domain of a partial last tile."""
    rng = np.random.default_rng(seed)
    need = int(rng.choice((2, 5, 10, 20, 40, 100)))
    lens = np.concatenate([rng.geometric(0.08, 3000), rng.integers(100, 3000, 6)])
    rng.shuffle(lens)
    n = int(lens.sum())
    link = np.ones(n, bool)
    link[np.concatenate([[0], np.cumsum(lens)[:-1]])] = False
    n_dom = n - int(rng.integers(1, 1500))
    _check(lib, link, n_dom, need)
