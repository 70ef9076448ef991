"""ctypes binding of libcutesv_b200.so (include/cutesv_b200.h).

This is the stub a cuteSV maintainer would add (INTEGRATION.md).  There is no CPU fallback: if the
CUDA library is missing or no H100 is usable the import / csv_create fails loudly.
"""
import ctypes as C
import os

from . import _abi

_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libcutesv_b200.so")
_lib = None

_VP = C.c_void_p
_I32P = C.POINTER(C.c_int32)
_I64P = C.POINTER(C.c_int64)

_SIGNATURES = {
    "csv_last_error": (C.c_char_p, []),
    "csv_version": (C.c_int, []),
    "csv_default_params": (C.c_int, [C.POINTER(_abi.csv_params)]),
    "csv_create": (C.c_int, [C.c_int, _VP, C.POINTER(_VP)]),
    "csv_destroy": (C.c_int, [_VP]),
    "csv_set_params": (C.c_int, [_VP, C.POINTER(_abi.csv_params)]),
    "csv_set_contigs": (C.c_int, [_VP, C.c_int32, _I64P]),
    "csv_host_alloc": (C.c_int, [C.POINTER(_VP), C.c_size_t]),
    "csv_host_free": (C.c_int, [_VP]),
    "csv_host_register": (C.c_int, [_VP, C.c_size_t]),
    "csv_host_unregister": (C.c_int, [_VP]),
    "csv_upload_sigs": (C.c_int, [_VP, C.c_int, C.POINTER(_abi.csv_sig_cols)]),
    "csv_upload_reads": (C.c_int, [_VP, C.POINTER(_abi.csv_reads_cols)]),
    "csv_upload_sigs_grouped": (C.c_int, [_VP, C.c_int, C.POINTER(_abi.csv_sig_cols), _I64P]),
    "csv_upload_reads_grouped": (C.c_int, [_VP, C.POINTER(_abi.csv_reads_cols), _I64P]),
    "csv_upload_alignments": (C.c_int, [_VP, C.POINTER(_abi.csv_reads_cols)]),
    "csv_upload_sigs_device": (C.c_int, [_VP, C.c_int, C.POINTER(_abi.csv_sig_cols), _VP]),
    "csv_upload_reads_device": (C.c_int, [_VP, C.POINTER(_abi.csv_reads_cols), _VP]),
    "csv_upload_sigs_grouped_device": (C.c_int, [_VP, C.c_int, C.POINTER(_abi.csv_sig_cols), _I64P, _VP]),
    "csv_upload_reads_grouped_device": (C.c_int, [_VP, C.POINTER(_abi.csv_reads_cols), _I64P, _VP]),
    "csv_upload_alignments_device": (C.c_int, [_VP, C.POINTER(_abi.csv_reads_cols), _VP]),
    "csv_cluster": (C.c_int, [_VP, C.c_uint32]),
    "csv_result_counts": (C.c_int, [_VP, _I64P, _I64P]),
    "csv_fetch": (C.c_int, [_VP, _VP, _VP, C.c_int64, _I32P, C.c_int64]),
    "csv_result_device_ptrs": (C.c_int, [_VP, C.POINTER(_VP), C.POINTER(_VP), C.POINTER(_VP)]),
    "csv_cluster_host": (C.c_int, [_VP, C.POINTER(_abi.csv_sig_cols), C.POINTER(_abi.csv_reads_cols), C.c_uint32, _VP, _VP,
                                   C.c_int64, _I32P, C.c_int64, _I64P, _I64P]),
    "csv_cluster_host_grouped": (C.c_int, [_VP, C.POINTER(_abi.csv_sig_cols), C.POINTER(_I64P), C.POINTER(_abi.csv_reads_cols), _I64P,
                                           C.c_uint32, _VP, _VP, C.c_int64, _I32P, C.c_int64, _I64P, _I64P]),
    "csv_cal_gl": (C.c_int, [_VP, _I32P, _I32P, C.c_int64, _VP]),
    "csv_overlap_cover": (C.c_int, [_VP, _VP, C.c_int64, C.POINTER(_abi.csv_reads_cols), _I32P, _I32P, _I64P, _I32P, C.c_int64, _I64P, _I32P,
                                    C.c_int64, _I64P, _I64P]),
    "csv_call_gt": (C.c_int, [_VP, _VP, C.c_int64, C.c_int32, C.POINTER(_abi.csv_reads_cols), _I64P, _I32P, _VP]),
    "csv_tra_call_gt": (C.c_int, [_VP, _VP, C.c_int64, C.POINTER(_abi.csv_reads_cols), C.c_int32, C.c_int32, _I64P, _I32P, _VP]),
    "csv_extract": (C.c_int, [_VP, C.POINTER(_abi.csv_read_cols), C.POINTER(C.c_uint32), C.c_int64,
                              C.POINTER(_abi.csv_sa_cols), _I64P, _I64P]),
    "csv_extract_append": (C.c_int, [_VP, C.POINTER(_abi.csv_read_cols), C.POINTER(C.c_uint32), C.c_int64,
                                     C.POINTER(_abi.csv_sa_cols), _I64P, _I64P]),
    "csv_extract_device": (C.c_int, [_VP, C.POINTER(_abi.csv_read_cols), C.POINTER(C.c_uint32), C.c_int64, C.POINTER(_abi.csv_sa_cols),
                                     C.POINTER(_abi.csv_seq_cols), _VP, _I64P, _I64P]),
    "csv_extract_append_device": (C.c_int, [_VP, C.POINTER(_abi.csv_read_cols), C.POINTER(C.c_uint32), C.c_int64, C.POINTER(_abi.csv_sa_cols),
                                            C.POINTER(_abi.csv_seq_cols), _VP, _I64P, _I64P]),
    "csv_extract_named_device": (C.c_int, [_VP, C.POINTER(_abi.csv_read_cols), C.POINTER(C.c_uint32), C.c_int64, C.POINTER(_abi.csv_sa_cols),
                                           C.POINTER(_abi.csv_seq_cols), C.POINTER(_abi.csv_name_cols), _VP, _I64P, _I64P]),
    "csv_extract_append_named_device": (C.c_int, [_VP, C.POINTER(_abi.csv_read_cols), C.POINTER(C.c_uint32), C.c_int64,
                                                  C.POINTER(_abi.csv_sa_cols), C.POINTER(_abi.csv_seq_cols), C.POINTER(_abi.csv_name_cols), _VP,
                                                  _I64P, _I64P]),
    "csv_rank_names": (C.c_int, [_VP, _I64P]),
    "csv_name_ranks_device_ptr": (C.c_int, [_VP, C.POINTER(_VP), _I64P]),
    "csv_fetch_names": (C.c_int, [_VP, _I32P, C.c_int64, C.POINTER(C.c_uint8), C.c_int64, _I64P]),
    "csv_order_ins_ties": (C.c_int, [_VP, _I64P]),
    "csv_fetch_alignments": (C.c_int, [_VP, C.c_int64, _I32P, _I32P, _I32P, _I32P, C.POINTER(C.c_uint8), _I64P]),
    "csv_set_scan_regions": (C.c_int, [_VP, C.c_int32, _I64P, C.POINTER(C.c_double), _I64P, _I64P]),
    "csv_scan_append_named_device": (C.c_int, [_VP, C.POINTER(_abi.csv_read_cols), C.POINTER(C.c_uint32), C.c_int64, C.POINTER(_abi.csv_sa_cols),
                                               C.POINTER(_abi.csv_seq_cols), C.POINTER(_abi.csv_name_cols), C.c_int, _VP, _I64P, _I64P, _I64P]),
    "csv_set_contig_names": (C.c_int, [_VP, C.c_int32, C.POINTER(C.c_uint8), _I64P]),
    "csv_reduce_sa_device": (C.c_int, [_VP, C.POINTER(_abi.csv_sa_text), _VP, C.POINTER(_I64P), C.POINTER(_abi.csv_sa_cols)]),
    "csv_ins_seq_device_ptrs": (C.c_int, [_VP, C.POINTER(_VP), C.POINTER(_VP), C.POINTER(_VP), _I64P]),
    "csv_fetch_ins_seqs": (C.c_int, [_VP, _I64P, C.c_int64, C.POINTER(C.c_uint8), C.c_int64, _I64P]),
    "csv_extract_reset": (C.c_int, [_VP]),
    "csv_extract_skipped": (C.c_int64, [_VP]),
    "csv_remap_read_ids": (C.c_int, [_VP, _I32P, C.c_int64]),
    "csv_swap_ins_rows": (C.c_int, [_VP, _I64P, C.c_int64]),
    "csv_fetch_sigs_range": (C.c_int, [_VP, C.c_int, C.c_int64, C.c_int64, _I32P, _I32P, _I32P, _I32P, _I32P, _I32P, _I32P]),
    "csv_fetch_pieces_range": (C.c_int, [_VP, C.c_int64, C.c_int64, _I32P]),
    "csv_extract_records": (C.c_int, [_VP, C.c_int]),
    "csv_fetch_records": (C.c_int, [_VP, C.c_int, C.c_int64, C.c_int64, _I32P]),
    "csv_sort_sigs": (C.c_int, [_VP, C.c_int, _I64P, C.c_int64, _I64P, _I64P, C.POINTER(C.c_uint8)]),
    "csv_fetch_sigs": (C.c_int, [_VP, C.c_int, C.c_int64, _I32P, _I32P, _I32P, _I32P, _I32P, _I32P, _I32P]),
    "csv_fetch_pieces": (C.c_int, [_VP, C.c_int64, _I32P, _I64P]),
    "csv_fetch_read_rows": (C.c_int, [_VP, C.c_int64, _I32P, _I32P, _I32P, _I32P, C.POINTER(C.c_uint8)]),
    "csv_set_profiling": (C.c_int, [_VP, C.c_int]),
    "csv_set_lanes": (C.c_int, [_VP, C.c_int]),
    "csv_stage_ms": (C.c_int, [_VP, C.POINTER(C.c_float)]),
    "csv_kernel_times": (C.c_int64, [_VP, C.c_char_p, C.c_int64]),
    "csv_launch_count": (C.c_int64, [_VP]),
    "csv_graph_replays": (C.c_int64, [_VP]),
    "csv_set_shard": (C.c_int, [_VP, C.POINTER(C.c_uint8)]),
    "csv_comm_unique_id": (C.c_int, [_VP, C.c_size_t]),
    "csv_comm_init": (C.c_int, [_VP, _VP, C.c_int, C.c_int]),
    "csv_comm_destroy": (C.c_int, [_VP]),
    "csv_allgather": (C.c_int, [_VP]),
    "csv_set_gather": (C.c_int, [_VP, C.c_int]),
    "csv_gather_mode": (C.c_int, [_VP]),
    "csv_gathered_counts": (C.c_int, [_VP, _I64P, _I64P]),
    "csv_fetch_gathered": (C.c_int, [_VP, _VP, _VP, C.c_int64, _I32P, C.c_int64]),
    "csv_gathered_device_ptrs": (C.c_int, [_VP, C.POINTER(_VP), C.POINTER(_VP), C.POINTER(_VP)]),
    "csv_debug_counters": (C.c_int, [_VP, C.POINTER(C.c_uint32)]),
    "csv_sort_probe": (C.c_int, [_VP, C.POINTER(C.c_float), _I64P, C.POINTER(C.c_int32)]),
}
EXPORTS = tuple(sorted(_SIGNATURES))


class CuteSVError(RuntimeError):
    def __init__(self, code, msg):
        RuntimeError.__init__(self, "cutesv_b200 error %d: %s" % (code, msg))
        self.code = code


def so_path():
    return _SO


def lib():
    """Load the CUDA library; raises (never falls back) when it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            raise ImportError("libcutesv_b200.so is not built (run `python -m cutesv_b200.build`); "
                              "cutesv_b200 has no CPU fallback")
        L = C.CDLL(_SO)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise CuteSVError(rc, lib().csv_last_error().decode("utf-8", "replace"))
