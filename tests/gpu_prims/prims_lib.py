"""ctypes binding of the test-only launchers of the library's device-wide primitives (tests/gpu_prims/prims.cu).  Device
buffers are torch CUDA tensors; every call runs on torch's current stream and synchronises before it returns."""
import ctypes as C
import os
import subprocess

from cutesv_b200 import build as lib_build

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libcsv_prims.so")
_SRCS = [os.path.join(_HERE, "prims.cu"), os.path.join(_HERE, "../../cutesv_b200/csrc/devprims.cuh")]
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
