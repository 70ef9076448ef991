"""CPU: normalisation of device-resident upload columns (_abi.device_cols) with stand-in __cuda_array_interface__ objects."""
import ctypes as C

import numpy as np
import pytest

from cutesv_b200 import _abi


class FakeDev(object):
    """A device array as far as the interface goes: typestr, shape, strides, address, and torch's `device.index`."""

    class _Dev(object):
        def __init__(self, index):
            self.index = index

    def __init__(self, n, typestr="<i4", addr=0x7F0000000000, strides=None, device=0, shape=None):
        self.__cuda_array_interface__ = {"shape": shape if shape is not None else (n,), "typestr": typestr, "data": (addr, False),
                                         "strides": strides, "version": 3}
        self.device = FakeDev._Dev(device)

    def __len__(self):
        return self.__cuda_array_interface__["shape"][0]


def sig_cols(n, **over):
    cols = {f: FakeDev(n, addr=0x1000 * (k + 1)) for k, f in enumerate(_abi.SIG_FIELDS)}
    cols.update(over)
    return cols


def reads_cols(n, **over):
    cols = {f: FakeDev(n, "|u1" if f == "is_primary" else "<i4", addr=0x1000 * (k + 1)) for k, f in enumerate(_abi.READS_FIELDS)}
    cols.update(over)
    return cols


def addr(p):
    return C.cast(p, C.c_void_p).value


def test_host_columns_take_the_numpy_path():
    assert _abi.device_cols(None, _abi.SIG_FIELDS, 0) is None
    host = {f: np.zeros(4, np.int32) for f in _abi.SIG_FIELDS}
    assert _abi.device_cols(host, _abi.SIG_FIELDS, 0) is None


def test_signature_struct_carries_the_device_addresses():
    s, off = _abi.device_cols(sig_cols(7), _abi.SIG_FIELDS, 0)
    assert off is None and s.n == 7
    assert [addr(getattr(s, f)) for f in _abi.SIG_FIELDS] == [0x1000, 0x2000, 0x3000, 0x4000, 0x5000]
    s, _ = _abi.device_cols(sig_cols(7, c=None), _abi.SIG_FIELDS, 0)   # DEL / DUP without column c
    assert addr(s.c) is None


def test_reads_struct_and_grouped_offsets():
    cols = reads_cols(5)
    del cols["chrom"]
    cols["contig_off"] = FakeDev(4, "<i8", addr=0x9000)
    s, off = _abi.device_cols(cols, _abi.READS_FIELDS, 0, grouped=True, n_contigs=3)
    assert s.n == 5 and addr(s.chrom) is None and addr(off) == 0x9000 and addr(s.is_primary) == 0x5000
    with pytest.raises(ValueError, match="n_contigs"):
        _abi.device_cols(cols, _abi.READS_FIELDS, 0, grouped=True, n_contigs=4)
    del cols["contig_off"]
    with pytest.raises(ValueError, match="contig_off"):
        _abi.device_cols(cols, _abi.READS_FIELDS, 0, grouped=True, n_contigs=3)


def test_empty_device_columns_clear_the_slot():
    s, off = _abi.device_cols(sig_cols(0), _abi.SIG_FIELDS, 0)
    assert s.n == 0 and addr(s.a) is None and off is None


@pytest.mark.parametrize("field,typestr", [("a", "<i8"), ("read_id", "<u4"), ("c", "<f4"), ("chrom", "|u1")])
def test_wrong_signature_dtype_raises_type_error(field, typestr):
    with pytest.raises(TypeError, match=field):
        _abi.device_cols(sig_cols(6, **{field: FakeDev(6, typestr)}), _abi.SIG_FIELDS, 0)


def test_is_primary_must_be_uint8():
    with pytest.raises(TypeError, match="is_primary"):
        _abi.device_cols(reads_cols(6, is_primary=FakeDev(6, "|b1")), _abi.READS_FIELDS, 0)
    with pytest.raises(TypeError, match="start"):
        _abi.device_cols(reads_cols(6, start=FakeDev(6, "|u1")), _abi.READS_FIELDS, 0)


def test_non_contiguous_or_multi_dimensional_columns_raise():
    with pytest.raises(TypeError, match="contiguous"):
        _abi.device_cols(sig_cols(6, b=FakeDev(6, strides=(8,))), _abi.SIG_FIELDS, 0)
    with pytest.raises(TypeError, match="one dimension"):
        _abi.device_cols(sig_cols(6, b=FakeDev(6, shape=(3, 2))), _abi.SIG_FIELDS, 0)
    _abi.device_cols(sig_cols(6, b=FakeDev(6, strides=(4,))), _abi.SIG_FIELDS, 0)   # explicit unit strides are contiguous


def test_mismatched_lengths_raise():
    with pytest.raises(ValueError, match="lengths"):
        _abi.device_cols(sig_cols(6, read_id=FakeDev(5)), _abi.SIG_FIELDS, 0)
    with pytest.raises(ValueError, match="lengths"):
        _abi.device_cols(reads_cols(6, is_primary=FakeDev(7, "|u1")), _abi.READS_FIELDS, 0)


def test_mixing_host_and_device_in_one_upload_raises():
    with pytest.raises(ValueError, match="all device or all host arrays"):
        _abi.device_cols(sig_cols(6, a=np.zeros(6, np.int32)), _abi.SIG_FIELDS, 0)


def test_column_on_another_device_raises():
    with pytest.raises(ValueError, match="device 1"):
        _abi.device_cols(sig_cols(6, a=FakeDev(6, device=1)), _abi.SIG_FIELDS, 0)
    _abi.device_cols(sig_cols(6, a=FakeDev(6, device=1), b=FakeDev(6, device=1), chrom=FakeDev(6, device=1), read_id=FakeDev(6, device=1),
                              c=FakeDev(6, device=1)), _abi.SIG_FIELDS, 1)


def test_missing_required_column_raises():
    cols = sig_cols(6)
    del cols["read_id"]
    with pytest.raises(ValueError, match="read_id"):
        _abi.device_cols(cols, _abi.SIG_FIELDS, 0)
