"""-m gpu: the library's device-wide primitives (cutesv_b200/csrc/devprims.cuh) on their own, against int64 numpy references.
k_scan_excl<4> and <8> (exclusive cumsum, carry, total, device count), k_select (flatnonzero, overflow, device count) and the
decoupled look-back itself through a probe kernel (tile t publishes a given value and reads back its exclusive prefix): at
tile edges, with grids smaller than the tile count, misaligned arrays, prefixes and tile totals past 2^30 and 2^31 up to
2^32 - 1, and with status buffers reused over generations or filled with words of other generations."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "gpu_prims"))
import prims_lib  # noqa: E402

pytestmark = pytest.mark.gpu
M32 = 1 << 32
SEL_TILE = 2048


@pytest.fixture(scope="module")
def torch_dev():
    import torch
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0) < (9, 0):
        pytest.skip("no usable sm_90 device")
    return torch


_gen = [4096]


def fresh_gen():
    """A generation no earlier launch of this module used (all within [1, 2^31))."""
    _gen[0] += 1
    return _gen[0]


@pytest.fixture(scope="module")
def sync(torch_dev):
    """One status buffer for the whole module: every launch leaves its words behind for the next generations."""
    return prims_lib.Sync(1 << 14)


def _to_dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.int64) % M32, dtype=np.uint32).view(np.int32)).cuda()


def _u32(t):
    return t.cpu().numpy().view(np.uint32).astype(np.int64)


def _excl(v, carry=0):
    v = np.asarray(v, dtype=np.int64)
    out = np.zeros(len(v), dtype=np.int64)
    if len(v):
        np.cumsum(v[:-1], out=out[1:])
    return (out + carry) % M32


def _scan(torch, sync, items, vals, grid=None, pad=5, offset=0, carry=None, n_dev=None, n_host=None, gen=None):
    """Runs k_scan_excl<items> over `vals` placed at `offset` in a buffer with `pad` sentinel words after them.  Returns
    (the n scanned outputs, the untouched-words check, total_out or None)."""
    vals = np.asarray(vals, dtype=np.int64)
    n = len(vals)
    sentinel = 0x5A5A5A5A
    buf = np.full(offset + n + pad, sentinel, dtype=np.int64)
    buf[offset:offset + n] = vals
    d = _to_dev(torch, buf)
    arr = d[offset:]
    n_host = n if n_host is None else n_host
    n_eff = n_host if n_dev is None else min(n_dev, n_host)
    tiles = max(1, -(-n_eff // (256 * items)))
    cin = _to_dev(torch, [carry]) if carry is not None else None
    tot = _to_dev(torch, [sentinel])
    ndv = _to_dev(torch, [n_dev]) if n_dev is not None else None
    prims_lib.scan_excl(items, arr, n_host, sync, fresh_gen() if gen is None else gen, grid or tiles, n_dev=ndv, carry_in=cin, total_out=tot)
    got = _u32(d)
    untouched = np.array_equal(got[:offset], buf[:offset]) and np.array_equal(got[offset + n_eff:], buf[offset + n_eff:])
    return got[offset:offset + n_eff], untouched, int(_u32(tot)[0])


def _check_scan(torch, sync, items, vals, carry=0, **kw):
    got, untouched, total = _scan(torch, sync, items, vals, carry=carry, **kw)
    v = np.asarray(vals, dtype=np.int64)[:len(got)]
    assert untouched, "words outside [0, n) changed"
    ref = _excl(v, carry)
    bad = np.flatnonzero(got != ref)
    assert len(bad) == 0, "first wrong prefix at %d of %d: %d, expected %d" % (bad[0], len(ref), got[bad[0]], ref[bad[0]])
    assert total == (carry + int(v.sum())) % M32


# ---- k_scan_excl: sizes at tile edges, grids that loop over tickets, the scalar path beside the vector one ----

@pytest.mark.parametrize("items", [4, 8])
@pytest.mark.parametrize("tiles,extra", [(0, 1), (0, 3), (0, 4), (0, 5), (1, -1), (1, 0), (1, 1), (2, -1), (2, 1)])
@pytest.mark.parametrize("grid", [None, 1])
def test_scan_sizes_at_tile_edges(torch_dev, sync, items, tiles, extra, grid):
    """n = tiles * T + extra for the tile T = 256 * items: 1, 3, 4, 5, T - 1, T, T + 1, 2T - 1, 2T + 1."""
    n = tiles * 256 * items + extra
    vals = np.random.default_rng(n * 7 + items).integers(0, 1 << 16, n)
    _check_scan(torch_dev, sync, items, vals, grid=grid)


@pytest.mark.parametrize("items", [4, 8])
@pytest.mark.parametrize("grid", [3, 64])
def test_scan_many_tiles_small_grid(torch_dev, sync, items, grid):
    n = 300 * 256 * items + 17
    vals = np.random.default_rng(grid + items).integers(0, 1 << 12, n)
    _check_scan(torch_dev, sync, items, vals, grid=grid)


@pytest.mark.parametrize("items", [4, 8])
@pytest.mark.parametrize("offset", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [4095, 5001, 3 * 2048 + 2])
def test_scan_misaligned_and_ragged(torch_dev, sync, items, offset, n):
    """arr 4..12 B off 16 B alignment (every thread on the scalar path) or aligned with a ragged end (the 128-bit path with
    a scalar last thread)."""
    vals = np.random.default_rng(offset * 31 + n).integers(0, 1 << 20, n)
    _check_scan(torch_dev, sync, items, vals, offset=offset, grid=5)


@pytest.mark.parametrize("items", [4, 8])
@pytest.mark.parametrize("n_dev", [0, 1, 1023, 2049, 5000, 5001, 9000])
def test_scan_device_count(torch_dev, sync, items, n_dev):
    """n from a device counter, clamped to n_host: the words past it stay as they were, total_out covers n only."""
    vals = np.random.default_rng(n_dev).integers(0, 1 << 24, 5000)
    _check_scan(torch_dev, sync, items, vals, carry=11, n_dev=n_dev, n_host=5000)


@pytest.mark.parametrize("items", [4, 8])
@pytest.mark.parametrize("carry", [0, 1, 123456789, (1 << 31) + 5, M32 - 1])
@pytest.mark.parametrize("n", [0, 1, 2500])
def test_scan_carry_and_total(torch_dev, sync, items, carry, n):
    """carry_in is added to every output and to total_out (modulo 2^32); n = 0 writes total_out = carry and nothing else."""
    vals = np.random.default_rng(n + carry % 1000).integers(0, 1 << 16, n)
    _check_scan(torch_dev, sync, items, vals, carry=carry)


def _large(kind, items):
    T = 256 * items
    rng = np.random.default_rng(LARGE.index(kind) * 10 + items)
    if kind == "prefix_past_2^30_2^31":        # many tiles, each far below 2^30, prefixes walk past 2^30 and 2^31
        n = 40 * T
        return rng.integers(0, (3 << 30) // n * 2, n)
    if kind == "total_2^32-1":
        n = 7 * T + 3
        v = rng.integers(0, M32 // n, n)
        v[-1] = 0
        v[-1] = M32 - 1 - v.sum()
        assert 0 <= v[-1] < M32
        return v
    if kind == "tile_total_2^30":            # tile 0's total is exactly 2^30
        v = rng.integers(0, 1 << 10, 4 * T)
        v[:T] = 0
        v[:T] = (1 << 30) // T
        return v
    if kind == "tile_total_past_2^30":       # tile 1's own total in [2^30, 2^31)
        v = rng.integers(0, 1 << 10, 5 * T)
        v[T:2 * T] = rng.integers((1 << 30) // T, (1 << 31) // T, T)
        return v
    if kind == "tile_total_past_2^31":       # tile 0's own total in [2^31, 2^32), later tiles small
        v = rng.integers(0, 1 << 10, 6 * T)
        v[:T] = rng.integers((1 << 31) // T + 1, (3 << 30) // T, T)
        return v
    if kind == "single_values_past_2^31":    # elements of 2^31 and more, the total still below 2^32
        v = rng.integers(0, 1 << 10, 3 * T + 1)
        v[T + 7] = (1 << 31) + 12345
        v[2 * T - 1] = (1 << 30) + 99
        return v
    raise KeyError(kind)


LARGE = ["prefix_past_2^30_2^31", "total_2^32-1", "tile_total_2^30", "tile_total_past_2^30", "tile_total_past_2^31",
         "single_values_past_2^31"]


@pytest.mark.parametrize("items", [4, 8])
@pytest.mark.parametrize("kind", LARGE)
@pytest.mark.parametrize("grid", [None, 2])
def test_scan_large_prefixes(torch_dev, sync, items, kind, grid):
    vals = _large(kind, items)
    assert vals.sum() < M32
    _check_scan(torch_dev, sync, items, vals, grid=grid)


# ---- the look-back alone: per-tile values, tile counts 1 .. ~3000 ----

def _probe_vals(kind, n):
    rng = np.random.default_rng(n)
    v = np.zeros(n, dtype=np.int64)
    if kind == "2^30_first":
        v[:] = 1
        v[0] = 1 << 30
    elif kind == "2^31-1_first":
        v[:] = 1
        v[0] = (1 << 31) - 1
    elif kind == "2^31_then_2^31-1":
        v[:3] = [1 << 31, (1 << 31) - 1, 1][:n]
    elif kind == "2^32-1_first":
        v[0] = M32 - 1
    elif kind == "large_random":             # every tile's value up to ~2^32 / n, total below 2^32
        v[:] = rng.integers(0, M32 // n, n)
    elif kind == "2^30_every_tile":          # inclusive prefixes of 2^30, 2^31, 3 * 2^30: every flag pattern of the old words
        v[:min(n, 3)] = 1 << 30
        v[3:] = rng.integers(0, 1 << 8, max(n - 3, 0))
    else:
        raise KeyError(kind)
    return v


@pytest.mark.parametrize("kind", ["2^30_first", "2^31-1_first", "2^31_then_2^31-1", "2^32-1_first", "large_random", "2^30_every_tile"])
@pytest.mark.parametrize("n", [1, 2, 3, 33, 65, 1000, 3000])
@pytest.mark.parametrize("grid", ["all", 4])
def test_lookback_probe(torch_dev, sync, kind, n, grid):
    torch = torch_dev
    v = _probe_vals(kind, n)   # prefixes wrap modulo 2^32 like the scans' outputs: [2^31, 2^31 - 1, 1] reaches 2^32 at tile 3
    vals = _to_dev(torch, v)
    excl = _to_dev(torch, np.full(n, 0x5A5A5A5A))
    prims_lib.lookback_probe(vals, excl, sync, fresh_gen(), n if grid == "all" else grid)
    got, ref = _u32(excl), _excl(v)
    bad = np.flatnonzero(got != ref)
    assert len(bad) == 0, "tile %d: %d, expected %d" % (bad[0], got[bad[0]], ref[bad[0]])


# ---- generations: one status buffer reused, or filled with other generations' words ----

def test_generations_reuse_one_buffer(torch_dev, sync):
    """Successive launches on one status buffer with tile counts that go down and up again, so that words of older
    generations lie below and above the current tile count; scans and probes take turns."""
    torch = torch_dev
    rng = np.random.default_rng(5)
    for i, tiles in enumerate([40, 3, 25, 1, 60, 2, 60, 59, 7]):
        items = 4 if i % 2 else 8
        n = tiles * 256 * items - (i % 3)
        vals = rng.integers(0, (3 << 30) // n, n)
        _check_scan(torch, sync, items, vals, grid=min(tiles, 1 + i))
        pv = rng.integers(0, M32 // (2 * tiles), tiles)
        pv[0] = (1 << 31) + i
        excl = _to_dev(torch, np.zeros(tiles))
        prims_lib.lookback_probe(_to_dev(torch, pv), excl, sync, fresh_gen(), 1 + i % 4)
        assert np.array_equal(_u32(excl), _excl(pv))


def _foreign_words(n, gen, rng):
    """n status words of other generations whose low halves take every flag pattern, in both the [gen:32][flag:2][value:30]
    and the [gen:31][incl:1][value:32] reading; none reads as generation `gen` in either."""
    others = np.array([gen - 1, gen + 1, gen + 2, 2 * gen, 2 * gen + 1, 2 * gen + 2, gen // 2, 0, 1, (1 << 31) - 1, (1 << 32) - 1], dtype=np.int64)
    hi = others[rng.integers(0, len(others), n)]
    lo = rng.integers(0, M32, n) & ((1 << 30) - 1) | (rng.integers(0, 4, n) << 30)
    w = (hi.astype(np.uint64) << np.uint64(32)) | lo.astype(np.uint64)
    clash = ((w >> np.uint64(32)) == np.uint64(gen)) | ((w >> np.uint64(33)) == np.uint64(gen))
    w[clash] = np.uint64(0)
    return w.view(np.int64)


@pytest.mark.parametrize("gen", [1, 2, 4097, 1 << 30, (1 << 31) - 1])
def test_prefilled_foreign_generations(torch_dev, gen):
    """A status buffer full of other generations' words (every flag pattern in their low halves), the generation at the
    ends of the range the library issues: scan, select and probe stay exact."""
    torch = torch_dev
    rng = np.random.default_rng(gen)
    s = prims_lib.Sync(4096)
    fill = torch.from_numpy(_foreign_words(4096, gen, rng)).cuda()
    s.status.copy_(fill)
    vals = rng.integers(0, M32 // 3000, 3000)
    vals[0] = (1 << 31) + 1
    excl = _to_dev(torch, np.zeros(3000))
    prims_lib.lookback_probe(_to_dev(torch, vals), excl, s, gen, 7)
    assert np.array_equal(_u32(excl), _excl(vals))
    s.status.copy_(fill)
    sv = _large("tile_total_past_2^31", 4)
    _check_scan(torch, s, 4, sv, grid=3, gen=gen)
    s.status.copy_(fill)
    flags = (rng.random(50 * SEL_TILE + 3) < 0.4).astype(np.uint8)
    _check_select(torch, s, flags, cap=len(flags), grid=5, gen=gen)


# ---- k_select ----

def _check_select(torch, sync, flags, cap, grid, n_dev=None, gen=None):
    flags = np.asarray(flags, dtype=np.uint8)
    n = len(flags) if n_dev is None else n_dev
    ref = np.flatnonzero(flags[:n])
    f = torch.from_numpy(np.concatenate([flags, np.ones(3, np.uint8)])).cuda()   # flagged words past n must not count
    sentinel = 0x5A5A5A5A
    out = torch.full((cap,), sentinel, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    st = _to_dev(torch, [0x100])
    ndv = _to_dev(torch, [n_dev]) if n_dev is not None else None
    prims_lib.select(f, len(flags), out, cnt, st, 0x4, sync, fresh_gen() if gen is None else gen, grid, n_dev=ndv)
    got = _u32(out)
    assert int(_u32(cnt)[0]) == len(ref)
    k = min(cap, len(ref))
    assert np.array_equal(got[:k], ref[:k])
    assert np.all(got[k:] == sentinel)
    assert int(_u32(st)[0]) == (0x104 if len(ref) > cap else 0x100)


@pytest.mark.parametrize("density", [0.0, 1.0, 0.3, 0.002])
@pytest.mark.parametrize("n", [1, 7, SEL_TILE - 1, SEL_TILE, SEL_TILE + 1, 2 * SEL_TILE + 1, 300 * SEL_TILE + 5])
@pytest.mark.parametrize("grid", ["all", 3])
def test_select_densities(torch_dev, sync, density, n, grid):
    flags = (np.random.default_rng(n).random(n) < density).astype(np.uint8)
    _check_select(torch_dev, sync, flags, cap=n, grid=-(-n // SEL_TILE) if grid == "all" else grid)


@pytest.mark.parametrize("cap", [0, 1, 100, 4095])
def test_select_overflow(torch_dev, sync, cap):
    """out_cap below the count: the overflow bit is set, the count stays exact, the first out_cap indices are right and
    nothing is written past out_cap."""
    flags = (np.random.default_rng(cap).random(5 * SEL_TILE + 11) < 0.5).astype(np.uint8)
    _check_select(torch_dev, sync, flags, cap=cap, grid=4)


@pytest.mark.parametrize("n_dev", [0, 1, SEL_TILE, 3 * SEL_TILE - 1, 9000])
def test_select_device_count(torch_dev, sync, n_dev):
    flags = (np.random.default_rng(n_dev).random(9000) < 0.6).astype(np.uint8)
    _check_select(torch_dev, sync, flags, cap=9000, grid=6, n_dev=n_dev)
