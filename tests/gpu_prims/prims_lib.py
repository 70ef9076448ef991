"""ctypes binding of the test-only launchers of the library's device-wide primitives and radix sort (tests/gpu_prims/prims.cu).
Device buffers are torch CUDA tensors; every call runs on torch's current stream and synchronises before it returns."""
import ctypes as C
import os
import subprocess

from cutesv_b200 import build as lib_build

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libcsv_prims.so")
_SRCS = [os.path.join(_HERE, "prims.cu"), os.path.join(_HERE, "../../cutesv_b200/csrc/devprims.cuh"),
         os.path.join(_HERE, "../../cutesv_b200/csrc/radix.cuh")]
_lib = None


def build(force=False):
    """Compiles prims.cu with the library's own nvcc flags (sm_90a) when the .so is missing or older than its sources."""
    if force or not os.path.exists(_SO) or any(os.path.getmtime(_SO) < os.path.getmtime(s) for s in _SRCS):
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call([nvcc] + lib_build.NVCC_FLAGS + ["-o", _SO, _SRCS[0]])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        vp, i64, u32, i32 = C.c_void_p, C.c_int64, C.c_uint32, C.c_int
        L.prims_scan_excl.argtypes = [i32, vp, i64, vp, vp, vp, vp, vp, vp, u32, i32, vp]
        L.prims_select.argtypes = [vp, i64, vp, vp, u32, vp, vp, u32, vp, vp, vp, u32, i32, vp]
        L.prims_lookback_probe.argtypes = [vp, i32, vp, vp, vp, vp, u32, i32, vp]
        L.prims_lb_ordinals.restype = u32
        L.prims_rs_hist.argtypes = [i32, vp, i64, vp, i32, vp, i32, vp]
        L.prims_rs_hist_scan.argtypes = [vp, i32, vp]
        L.prims_rs_onesweep.argtypes = [i32, i32, vp, vp, vp, vp, i64, vp, i32, vp, vp, vp, vp, u32, i32, vp]
        L.prims_rs_tile.argtypes = [i32]
        L.prims_rs_resident.argtypes = [i32]
        L.prims_rs_large_keys.argtypes = [vp, i64, vp]
        L.prims_rs_large_check.argtypes = [vp, vp, i64, i64, i64, vp, vp, vp]
        _lib = L
    return _lib


def lb_ordinals():
    return int(lib().prims_lb_ordinals())


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _run(fn, *args):
    import torch
    rc = fn(*args, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    if rc != 0:
        raise RuntimeError("launch failed: cudaError %d" % rc)
    torch.cuda.synchronize()


class Sync:
    """A TileSync's device words: the ticket (zeroed before every launch), the epoch word and the status buffer, which is
    never cleared, so successive launches with different generations share it as the library's do."""

    def __init__(self, status_words, device=0):
        import torch
        dev = torch.device("cuda", device)
        self.ticket = torch.zeros(1, dtype=torch.int32, device=dev)
        self.epoch = torch.zeros(1, dtype=torch.int32, device=dev)
        self.status = torch.zeros(max(status_words, 1), dtype=torch.int64, device=dev)

    def args(self, gen):
        """Sets the epoch word and returns (ticket, status, epoch, ordinal) for generation `gen`."""
        k = lb_ordinals()
        self.epoch.fill_(gen // k)
        self.ticket.zero_()
        return _p(self.ticket), _p(self.status), _p(self.epoch), C.c_uint32(gen % k)


def scan_excl(items, arr, n_host, sync, gen, grid, n_dev=None, carry_in=None, total_out=None):
    """k_scan_excl<items> in place on the int32 tensor `arr` (read as uint32)."""
    _run(lib().prims_scan_excl, C.c_int(items), _p(arr), C.c_int64(n_host), _p(n_dev), _p(carry_in), _p(total_out), *sync.args(gen),
         C.c_int(grid))


def select(flags, n_host, out, out_count, status_word, overflow_bit, sync, gen, grid, n_dev=None):
    """k_select over a uint8 flag tensor: out[k] = the k-th i with flags[i] != 0."""
    _run(lib().prims_select, _p(flags), C.c_int64(n_host), _p(n_dev), _p(out), C.c_uint32(out.numel()), _p(out_count), _p(status_word),
         C.c_uint32(overflow_bit), *sync.args(gen), C.c_int(grid))


def lookback_probe(vals, excl, sync, gen, grid):
    """Tile t publishes vals[t] and writes its exclusive prefix to excl[t] (both int32 tensors read as uint32)."""
    _run(lib().prims_lookback_probe, _p(vals), C.c_int(vals.numel()), _p(excl), *sync.args(gen), C.c_int(grid))


# ---- radix sort (cutesv_b200/csrc/radix.cuh) ----

RS_MAX_PASSES = 8
RS_THREADS = 256


def _key_bytes(keys):
    import torch
    if keys.dtype not in (torch.int32, torch.int64):
        raise TypeError("keys: int32 (read as uint32) or int64 (read as uint64), not %s" % keys.dtype)
    return keys.element_size()


def rs_tile(key_bytes):
    """Keys per k_rs_onesweep tile: 4096 for uint32 keys, 3072 for uint64 keys."""
    return int(lib().prims_rs_tile(C.c_int(key_bytes)))


def rs_resident(key_bytes):
    """k_rs_onesweep CTAs resident per SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor)."""
    r = int(lib().prims_rs_resident(C.c_int(key_bytes)))
    if r <= 0:
        raise RuntimeError("occupancy query failed: cudaError %d" % -r)
    return r


def rs_wave(key_bytes):
    """Keys of one wave of resident onesweep tiles: resident CTAs per SM x SM count x tile."""
    import torch
    return rs_resident(key_bytes) * torch.cuda.get_device_properties(0).multi_processor_count * rs_tile(key_bytes)


def rs_hist(keys, n_host, passes, hist, grid, n_dev=None):
    _run(lib().prims_rs_hist, C.c_int(_key_bytes(keys)), _p(keys), C.c_int64(n_host), _p(n_dev), C.c_int(passes), _p(hist), C.c_int(grid))


def rs_hist_scan(hist, passes):
    _run(lib().prims_rs_hist_scan, _p(hist), C.c_int(passes))


def rs_onesweep(keys_in, vals_in, keys_out, vals_out, n_host, shift, gbase, sync, gen, grid, n_dev=None):
    """One k_rs_onesweep<K, IOTA> pass, IOTA when vals_in is None."""
    _run(lib().prims_rs_onesweep, C.c_int(_key_bytes(keys_in)), C.c_int(vals_in is None), _p(keys_in), _p(vals_in), _p(keys_out), _p(vals_out),
         C.c_int64(n_host), _p(n_dev), C.c_int(shift), _p(gbase), *sync.args(gen), C.c_int(grid))


def radix_sort(keys, vals, bits, sync, gen0, n_dev=None, n_host=None, out=None):
    """The steps of the library's radix_sort() driver (cutesv_b200/csrc/cutesv_b200.cu), in its order: the histogram of
    RS_MAX_PASSES passes zeroed, k_rs_hist, k_rs_hist_scan, then ceil(bits / 8) onesweep passes that ping-pong between two key
    and two payload buffers, n_tiles CTAs per pass, one zeroed ticket per pass and pass p at generation gen0 + p on the one
    status buffer of `sync`, which is never cleared.  keys: int32 or int64 tensor (read as uint32 / uint64); vals: int32
    payload tensor, or None for the iota first pass the library uses.  n_dev: an int32 device count (<= n_host) the kernels
    read instead of n_host; the grids stay sized for n_host.  out: (keys, vals) buffers for the first pass to write (the
    ping-pong partners), allocated when None.  Returns the (keys, vals) tensors that hold the result."""
    import torch
    kb = _key_bytes(keys)
    n = keys.numel() if n_host is None else n_host
    passes = max(1, (bits + 7) // 8)
    if passes > RS_MAX_PASSES:
        raise ValueError("%d bits" % bits)
    T = rs_tile(kb)
    n_tiles = (n + T - 1) // T
    sms = torch.cuda.get_device_properties(keys.device).multi_processor_count
    hist = torch.zeros(RS_MAX_PASSES * 256, dtype=torch.int32, device=keys.device)
    rs_hist(keys, n, passes, hist, max(1, min((n + RS_THREADS * 16 - 1) // (RS_THREADS * 16), sms * 4)), n_dev=n_dev)
    rs_hist_scan(hist, passes)
    ko, vo = out if out is not None else (torch.empty_like(keys), torch.empty(max(keys.numel(), 1), dtype=torch.int32, device=keys.device))
    ki, vi = keys, vals
    if vi is None and passes > 1:   # the iota pass reads no payload; the second pass writes into this one
        vi = torch.empty_like(vo)
    for p in range(passes):
        rs_onesweep(ki, vals if p == 0 and vals is None else vi, ko, vo, n, 8 * p, hist[p * 256:], sync, gen0 + p, max(n_tiles, 1), n_dev=n_dev)
        ki, ko = ko, ki
        vi, vo = vo, vi
    return ki, vi


def rs_large_keys(keys, n):
    """The keys of the large closed-form sort (prims.cu k_lg_keys) into the int32 tensor `keys`."""
    _run(lib().prims_rs_large_keys, _p(keys), C.c_int64(n))


def rs_large_check(keys, vals, n, lo, cnt, n_bad, first_bad):
    """Adds to the int64 tensor n_bad the positions of [lo, lo + cnt) where the sorted keys / payloads differ from the closed
    form, and lowers first_bad[0] to the first of them."""
    _run(lib().prims_rs_large_check, _p(keys), _p(vals), C.c_int64(n), C.c_int64(lo), C.c_int64(cnt), _p(n_bad), _p(first_bad))
