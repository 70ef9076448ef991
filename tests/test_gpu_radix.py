"""-m gpu: the library's radix sort (cutesv_b200/csrc/radix.cuh: k_rs_hist, k_rs_hist_scan, k_rs_onesweep<K, IOTA>) on its own,
driven the way radix_sort() in cutesv_b200.cu drives it, against numpy's stable argsort of the masked keys.  uint32 keys
(tiles of T = 4096) and uint64 keys (T = 3072): sizes at the warp, tile and wave edges (a wave W·T is one onesweep tile per
resident CTA, from the occupancy of the compiled kernel), every key width from one pass to eight, the key patterns a stable
onesweep can get wrong (one digit everywhere, real keys equal to the padding value, other digits on the first and last
position of every tile and warp stripe, few distinct values), the iota and the explicit payload, status buffers reused over
generations or filled with other generations' words, a device-side count below the host bound, and one-pass sorts of more
than 2^30 + 2^20 and of 2^31 - 1 rows built and checked on the device."""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "gpu_prims"))
import prims_lib  # noqa: E402

pytestmark = pytest.mark.gpu
GiB = 1 << 30
M32 = 1 << 32
KEYS = {"u32": (4, 32), "u64": (8, 64)}   # key bytes, key bits


@pytest.fixture(scope="module")
def torch_dev():
    import torch
    if not torch.cuda.is_available() or torch.cuda.get_device_capability(0) < (9, 0):
        pytest.skip("no usable sm_90 device")
    yield torch
    torch.cuda.empty_cache()


STATUS_TILES = 8192


@pytest.fixture(scope="module")
def sync(torch_dev):
    """One status buffer for the module (never cleared), as a csv_cluster lane's is over its sorts."""
    return prims_lib.Sync(STATUS_TILES * 256)


_gen = [4096]


def fresh_gen(passes):
    """gen0 of a sort of `passes` passes, none of whose generations an earlier sort of this module used."""
    g = _gen[0] + 1
    _gen[0] += passes + 1
    return g


def _geom(kb):
    T = prims_lib.rs_tile(kb)
    return T, prims_lib.rs_wave(kb)


SIZES = ["1", "31", "32", "33", "255", "256", "257", "T-1", "T", "T+1", "2T-1", "2T+1", "WT-1", "WT", "WT+1", "3WT+17"]


def _size(spec, T, WT):
    """"3WT+17" -> 3 * WT + 17, "T-1" -> T - 1, "257" -> 257."""
    coef, unit, extra = re.fullmatch(r"(\d*)(WT|T)?([+-]\d+)?", spec).groups()
    if unit is None:
        return int(coef)
    return int(coef or 1) * (WT if unit == "WT" else T) + int(extra or 0)


def _mask(bits):
    return np.uint64((1 << bits) - 1)


def _to_dev(torch, a, kb):
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.astype(np.uint32).view(np.int32) if kb == 4 else a.astype(np.uint64).view(np.int64)).cuda()


def _from_dev(t, n):
    a = t[:n].cpu().numpy()
    return a.view(np.uint32).astype(np.uint64) if a.dtype == np.int32 else a.view(np.uint64)


def _payload(rng, n):
    v = rng.integers(0, M32, n, dtype=np.uint64)
    if n:
        v[rng.integers(0, n, 1 + n // 50)] = 0
        v[rng.integers(0, n, 1 + n // 50)] = M32 - 1
    return v


def _sort(torch, sync, keys, bits, kb, payload, gen0=None, n_dev=None, out=None):
    """Sorts the uint64 numpy keys (already below 2^bits) through prims_lib.radix_sort; returns (keys, payload) of the result
    as uint64 numpy arrays of n (or n_dev) rows and the payload sent (None: iota)."""
    n = len(keys)
    passes = max(1, (bits + 7) // 8)
    T = prims_lib.rs_tile(kb)
    assert (n + T - 1) // T <= STATUS_TILES
    kd = _to_dev(torch, keys, kb)
    vd = None if payload is None else _to_dev(torch, payload, 4)
    nd = None if n_dev is None else _to_dev(torch, [n_dev], 4)
    ko, vo = prims_lib.radix_sort(kd, vd, bits, sync, fresh_gen(passes) if gen0 is None else gen0, n_dev=nd, n_host=n, out=out)
    m = n if n_dev is None else n_dev
    return _from_dev(ko, m), _from_dev(vo, m), (ko, vo, kd, vd)


def _check(keys, bits, got_k, got_v, payload, what=""):
    m = len(got_k)
    ref = np.argsort(keys[:m] & _mask(bits), kind="stable")
    want_k = keys[:m][ref]
    want_v = ref.astype(np.uint64) if payload is None else payload[:m][ref]
    bad = np.flatnonzero((got_k != want_k) | (got_v != want_v))
    assert len(bad) == 0, "%s%d of %d rows wrong, first at %d: key %#x payload %d, expected key %#x payload %d" % (
        what, len(bad), m, bad[0], int(got_k[bad[0]]), int(got_v[bad[0]]), int(want_k[bad[0]]), int(want_v[bad[0]]))


def _run(torch, sync, keys, bits, kb, payload_kind, rng, **kw):
    payload = None if payload_kind == "iota" else _payload(rng, len(keys))
    gk, gv, _ = _sort(torch, sync, keys, bits, kb, payload, **kw)
    _check(keys, bits, gk, gv, payload)


def _uniform(rng, n, bits):
    return rng.integers(0, np.iinfo(np.uint64).max, n, dtype=np.uint64, endpoint=True) & _mask(bits)


# ---- sizes at the warp, tile and wave edges ----

@pytest.mark.parametrize("payload", ["iota", "explicit"])
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("K", list(KEYS))
def test_sizes(torch_dev, sync, K, size, payload):
    kb, bits = KEYS[K]
    T, WT = _geom(kb)
    n = _size(size, T, WT)
    rng = np.random.default_rng(n * 3 + kb)
    _run(torch_dev, sync, _uniform(rng, n, bits), bits, kb, payload, rng)


# ---- widths: 1 .. 4 and 5 .. 8 passes, and a last pass that only uses its low bits ----

WIDTHS = [("u32", b) for b in (1, 7, 8, 9, 16, 17, 24, 31, 32)] + [("u64", b) for b in (33, 40, 41, 56, 57, 63, 64)]


@pytest.mark.parametrize("size", ["2T+1", "WT+1"])
@pytest.mark.parametrize("K,bits", WIDTHS)
def test_widths(torch_dev, sync, K, bits, size):
    kb = KEYS[K][0]
    T, WT = _geom(kb)
    n = _size(size, T, WT)
    rng = np.random.default_rng(bits * 7 + n)
    keys = _uniform(rng, n, bits)
    keys[rng.integers(0, n, 5)] = _mask(bits)   # the widest key, so the last pass really sees its top bit
    _run(torch_dev, sync, keys, bits, kb, "iota", rng)


# ---- key patterns ----

def _pattern(kind, rng, n, bits, T, items):
    mx = _mask(bits)
    if kind == "equal":                     # one digit in every pass: every row in one digit run
        return np.full(n, rng.integers(0, 1 << min(bits, 63), dtype=np.uint64) & mx, dtype=np.uint64)
    if kind == "all_max":                   # every key the padding value (all ones)
        return np.full(n, mx, dtype=np.uint64)
    if kind == "zero_max":
        return np.where(rng.random(n) < 0.5, np.uint64(0), mx).astype(np.uint64)
    if kind == "alternating":
        a, b = _uniform(rng, 2, bits)
        return np.where(np.arange(n) % 2 == 0, a, b).astype(np.uint64)
    if kind == "ascending":
        return np.arange(n, dtype=np.uint64) * np.uint64(0x01010101) & mx
    if kind == "descending":
        return (np.uint64(n) - np.arange(n, dtype=np.uint64)) * np.uint64(0x01010101) & mx
    if kind == "few":                       # at most 5 distinct values: long equal runs whose order only the payload shows
        return rng.choice(_uniform(rng, 5, bits), n)
    if kind == "const_digit":               # the middle pass's digit is one value, the other passes vary
        p = (bits + 7) // 8 // 2
        k = _uniform(rng, n, bits) & ~np.uint64(0xFF << (8 * p))
        return (k | np.uint64(0xA5 << (8 * p))) & mx
    if kind == "tile_edges":                # another digit on the first / last row of every tile and every warp stripe
        k = np.full(n, _uniform(rng, 1, bits)[0], dtype=np.uint64)
        stripe = 32 * items
        pos = np.arange(n) % T
        edge = (pos == 0) | (pos == T - 1) | (pos % stripe == 0) | (pos % stripe == stripe - 1)
        k[edge] = _uniform(rng, int(edge.sum()), bits)
        return k
    raise KeyError(kind)


PATTERNS = ["equal", "all_max", "zero_max", "alternating", "ascending", "descending", "few", "const_digit", "tile_edges"]


@pytest.mark.parametrize("payload", ["iota", "explicit"])
@pytest.mark.parametrize("size", ["257", "2T+1", "WT+1"])
@pytest.mark.parametrize("kind", PATTERNS)
@pytest.mark.parametrize("K", list(KEYS))
def test_patterns(torch_dev, sync, K, kind, size, payload):
    kb, bits = KEYS[K]
    T, WT = _geom(kb)
    n = _size(size, T, WT)
    rng = np.random.default_rng(PATTERNS.index(kind) * 1000 + n)
    _run(torch_dev, sync, _pattern(kind, rng, n, bits, T, T // 256), bits, kb, payload, rng)


@pytest.mark.parametrize("payload", ["iota", "explicit"])
@pytest.mark.parametrize("size", ["2T+1", "WT+1"])
@pytest.mark.parametrize("K,bits", [("u32", 8), ("u32", 16), ("u32", 24), ("u32", 32), ("u64", 40), ("u64", 48), ("u64", 56), ("u64", 64)])
def test_one_digit_everywhere(torch_dev, sync, K, bits, size, payload):
    """All keys equal at every pass count from 1 to 8: every row of every tile sits in one digit run, so the rows keep their
    order only if every rank inside a warp does (an even number of passes could undo one pass's reversal)."""
    kb = KEYS[K][0]
    T, WT = _geom(kb)
    n = _size(size, T, WT)
    rng = np.random.default_rng(bits + n)
    _run(torch_dev, sync, _pattern("equal", rng, n, bits, T, T // 256), bits, kb, payload, rng)


@pytest.mark.parametrize("payload", ["iota", "explicit"])
@pytest.mark.parametrize("size", ["1", "T-1", "T+1", "2T-1", "WT-1", "WT+1"])
@pytest.mark.parametrize("kind", ["all_max", "zero_max"])
@pytest.mark.parametrize("K", list(KEYS))
def test_keys_equal_to_padding(torch_dev, sync, K, kind, size, payload):
    """Real all-ones keys beside the last tile's padding keys (all ones too): n mod T = 1 and T - 1, one tile and a wave."""
    kb, bits = KEYS[K]
    T, WT = _geom(kb)
    n = _size(size, T, WT)
    rng = np.random.default_rng(n + kb)
    _run(torch_dev, sync, _pattern(kind, rng, n, bits, T, T // 256), bits, kb, payload, rng)


# ---- look-back state: one status buffer over many sorts, other generations' words, the top of the generation range ----

@pytest.mark.parametrize("K", list(KEYS))
def test_status_reused_over_sizes(torch_dev, sync, K):
    """Sorts of decreasing then increasing n at increasing generations on one status buffer: the words a larger earlier sort
    left lie above the tile count of the next, and a later larger sort walks over a smaller one's."""
    kb, bits = KEYS[K]
    T, WT = _geom(kb)
    rng = np.random.default_rng(kb)
    for i, n in enumerate([2 * WT + 5, WT + 1, 7 * T - 1, T + 1, 33, 2 * T, WT - 1, 3 * WT + 17]):
        _run(torch_dev, sync, _uniform(rng, n, bits if i % 2 else 16), bits if i % 2 else 16, kb, "iota" if i % 3 else "explicit", rng)


def _foreign(n, gens, rng):
    """n status words of the generations `gens`, inclusive or not, with values 0 or 2^32 - 1 (and random ones)."""
    g = np.asarray(gens, dtype=np.uint64)[rng.integers(0, len(gens), n)]
    incl = rng.integers(0, 2, n).astype(np.uint64)
    val = np.where(rng.random(n) < 0.4, np.uint64(0), np.where(rng.random(n) < 0.6, np.uint64(M32 - 1), rng.integers(0, M32, n, dtype=np.uint64)))
    return ((g << np.uint64(33)) | (incl << np.uint64(32)) | val).view(np.int64)


@pytest.mark.parametrize("gen0", [1, 4097, 1 << 30, (1 << 21) * 1024 - 9])
@pytest.mark.parametrize("bits", [8, "full"])
@pytest.mark.parametrize("K", list(KEYS))
def test_status_prefilled_with_other_generations(torch_dev, K, bits, gen0):
    """Every status word written by generation gen0 - 1 or gen0 + passes (the neighbours of the sort's own generations),
    inclusive or not, with values 0 and 2^32 - 1; gen0 up to the top of the range the library issues (its last generation
    2^31 - 2 for eight passes)."""
    torch = torch_dev
    kb, full = KEYS[K]
    bits = full if bits == "full" else bits
    passes = (bits + 7) // 8
    T, WT = _geom(kb)
    n = WT + T // 2
    rng = np.random.default_rng(gen0 + kb)
    s = prims_lib.Sync(((n + T - 1) // T + 8) * 256)
    s.status.copy_(torch.from_numpy(_foreign(s.status.numel(), [gen0 - 1, gen0 + passes], rng)).cuda())
    assert gen0 + passes - 1 < (1 << 31)
    keys = _pattern("few", rng, n, bits, T, T // 256)
    _run(torch, s, keys, bits, kb, "explicit", rng, gen0=gen0)


# ---- a device-side count below the host bound; grids sized for the bound ----

@pytest.mark.parametrize("n_dev", ["0", "1", "T-1", "T", "T+1", "WT-1", "WT+1"])
@pytest.mark.parametrize("K", list(KEYS))
def test_device_count(torch_dev, sync, K, n_dev):
    """n_dev rows sorted, none past them read or written: the grid and the histogram grid are sized for n_host = 2WT + 7."""
    torch = torch_dev
    kb, bits = KEYS[K]
    T, WT = _geom(kb)
    n_host, m = 2 * WT + 7, _size(n_dev, T, WT)
    rng = np.random.default_rng(m + kb)
    keys, payload = _uniform(rng, n_host, bits), _payload(rng, n_host)
    sk, sv = 0x5A5A5A5A5A5A5A5A & ((1 << bits) - 1), 0x5A5A5A5A
    out = (_to_dev(torch, np.full(n_host, sk, np.uint64), kb), _to_dev(torch, np.full(n_host, sv, np.uint64), 4))
    gk, gv, (ko, vo, _, _) = _sort(torch, sync, keys, bits, kb, payload, n_dev=m, out=out)
    _check(keys, bits, gk, gv, payload)
    passes = (bits + 7) // 8   # the result is in the first-pass output buffers after an odd number of passes
    tail_k = np.full(n_host - m, sk, np.uint64) if passes % 2 else keys[m:]
    tail_v = np.full(n_host - m, sv, np.uint64) if passes % 2 else payload[m:]
    assert np.array_equal(_from_dev(ko, n_host)[m:], tail_k) and np.array_equal(_from_dev(vo, n_host)[m:], tail_v), "rows past n_dev changed"


# ---- more than 2^30 rows: one iota pass of uint32 keys, built and checked on the device ----

CHECK_STEP = 1 << 24


@pytest.mark.parametrize("n", [(1 << 30) + (1 << 20) + 3, (1 << 31) - 1])
def test_large_one_pass(torch_dev, n):
    """Digit 1 holds more than 2^30 rows, so its look-back prefixes and digit 255's base pass 2^30; every tile holds one digit-0
    and one digit-255 row at positions that vary from tile to tile (prims.cu k_lg_keys).  n = 2^31 - 1 is the library's row
    limit.  The result is compared with its closed form on the device, 2^24 rows per step."""
    torch = torch_dev
    T = prims_lib.rs_tile(4)
    tiles = (n + T - 1) // T
    need = 3 * 4 * n + tiles * 256 * 8 + (64 << 20)
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("needs %.1f GiB of free device memory, %.1f GiB free" % (need / GiB, free / GiB))
    keys = ko = vo = s = rk = rv = None
    try:
        keys = torch.empty(n, dtype=torch.int32, device="cuda")
        prims_lib.rs_large_keys(keys, n)
        ko = torch.empty(n, dtype=torch.int32, device="cuda")
        vo = torch.empty(n, dtype=torch.int32, device="cuda")
        s = prims_lib.Sync(tiles * 256)
        rk, rv = prims_lib.radix_sort(keys, None, 8, s, fresh_gen(1), out=(ko, vo))
        assert rk.data_ptr() == ko.data_ptr() and rv.data_ptr() == vo.data_ptr()
        n_bad = torch.zeros(1, dtype=torch.int64, device="cuda")
        first = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        for lo in range(0, n, CHECK_STEP):
            prims_lib.rs_large_check(ko, vo, n, lo, min(CHECK_STEP, n - lo), n_bad, first)
        bad, at = int(n_bad.item()), int(first.item())
        assert bad == 0, "%d of %d rows wrong, first at %d: key %#x payload %d" % (
            bad, n, at, int(ko[at].item()) & 0xFFFFFFFF, int(vo[at].item()) & 0xFFFFFFFF)
    finally:
        del keys, ko, vo, s, rk, rv
        torch.cuda.empty_cache()
