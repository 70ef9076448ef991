"""-m gpu: the device-built INS sequence arena of one packet at its size limits.  The row offsets come from the look-back scan
of the rows' lengths (1024 rows per tile), so a first tile of 2^30 or 2^31 bytes and a packet just below 4 GiB test the scan's
32-bit prefixes end to end; a packet of 4 GiB or more must be refused with CSV_E_CAPACITY, an append call leaving the
accumulation as it was and a non-append call leaving it empty.

Records lie on one contig, each with CIGAR 100M L·I 100M and a distinct L, so that row k's length names its record.  The
bases are random bytes drawn on the device (BAM's 4-bit layout, first base in the high nibble): a host-built copy of several
GB would only add a transfer.  Every check runs on the device through Engine.ins_seq_tensors(), the bytes in chunks."""
import ctypes as C

import numpy as np
import pytest

import device_packet_util as dpu
from cutesv_b200 import _abi, _lib

pytestmark = pytest.mark.gpu
GiB = 1 << 30
M32 = 1 << 32
INS = _abi.CSV_INS
BASES = np.frombuffer(b"=ACMGRSVTWYHKDBN", dtype=np.uint8).copy()
CHUNK = 1 << 24   # arena bytes compared per step


@pytest.fixture(scope="module")
def eng():
    """An engine of its own, closed at the end of the module so that its multi-GB arena does not outlive these tests."""
    from cutesv_b200._lib import CuteSVError
    from cutesv_b200.engine import Engine
    try:
        e = Engine(0)
    except CuteSVError as err:
        if err.code == _abi.CSV_E_NODEVICE:
            pytest.skip("no usable sm_90 device: %s" % err)
        raise
    e.set_params(_abi.default_params(max_size=-1, min_mapq=0, min_read_len=100))
    e.set_contigs(np.array([10_000_000], dtype=np.int64))
    e.set_extract_records(True)
    yield e
    e.close()
    import torch
    torch.cuda.empty_cache()


def _need(nbytes):
    import torch
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip("needs %.1f GiB of free device memory, %.1f GiB free" % (nbytes / GiB, free / GiB))


def _packet(Ls, seed):
    """Device packet of len(Ls) records, record i with CIGAR 100M Ls[i]I 100M and random bases; also returns the host copies
    of what the checks need (seq_off, L)."""
    import torch
    Ls = np.asarray(Ls, dtype=np.int64)
    n = len(Ls)
    assert len(np.unique(Ls)) == n and Ls.max() < (1 << 28)
    qlen = 200 + Ls
    seq_off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum((qlen + 1) // 2, out=seq_off[1:])
    start = 1000 + 300 * np.arange(n, dtype=np.int64)
    cig = np.stack([np.full(n, 100 << 4), (Ls << 4) | 1, np.full(n, 100 << 4)], axis=1).reshape(-1).astype(np.uint32)
    pk = dict(chrom=np.zeros(n, np.int32), ref_start=start.astype(np.int32), ref_end=(start + 200).astype(np.int32), flag=np.zeros(n, np.int32),
              mapq=np.full(n, 60, np.int32), query_len=qlen.astype(np.int32), read_id=np.arange(n, dtype=np.int32),
              cigar_off=3 * np.arange(n + 1, dtype=np.int64), sa_off=np.zeros(n + 1, np.int64), cigar=cig,
              sa={k: np.zeros(0, np.int32) for k in _abi.SA_FIELDS}, seq_off=seq_off)
    d = dpu.to_device(pk)
    g = torch.Generator(device="cuda").manual_seed(seed)
    d["seq4"] = torch.empty(int(seq_off[-1]), dtype=torch.uint8, device="cuda").random_(0, 256, generator=g)
    return d, dict(seq_off=seq_off, L=Ls)


def _exact(fn, k):
    """fn(cap) is a fetch that fails with CSV_E_CAPACITY when the library holds more than cap rows: True when it holds k."""
    return fn(k) == _abi.CSV_OK and (k == 0 or fn(k - 1) == _abi.CSV_E_CAPACITY)


def _holds(eng, counts, n_rows, n_pieces):
    """The library itself (not the engine's mirrors) holds exactly these signature, reads-row and piece counts."""
    nulls = [None] * 7
    for t in range(_abi.CSV_NTYPES):
        if not _exact(lambda cap: eng.L.csv_fetch_sigs(eng.h, t, C.c_int64(cap), *nulls), counts[t]):
            return False
    if not _exact(lambda cap: eng.L.csv_fetch_read_rows(eng.h, C.c_int64(cap), *[None] * 5), n_rows):
        return False
    npz = C.c_int64(-1)
    _lib.check(eng.L.csv_fetch_pieces(eng.h, C.c_int64(0), None, C.byref(npz)))
    return npz.value == n_pieces


def _check_arena(eng, pk, host, rows=None, rec0=0):
    """Rows [rows) of the arena (all by default) are the packet's records rec0.. : start is the exclusive int64 cumsum of len
    over the whole arena, len[k] the L of row k's record, and the bytes the record's bases L from query position 100."""
    import torch
    b, start, ln = eng.ins_seq_tensors()
    n_all = start.numel()
    r0, r1 = (0, n_all) if rows is None else rows
    ln64 = ln.to(torch.int64)
    expect_start = torch.cumsum(ln64, 0) - ln64
    bad = torch.nonzero(start != expect_start)
    assert bad.numel() == 0, "row %d starts at %d, expected %d" % (int(bad[0]), int(start[bad[0]]), int(expect_start[bad[0]]))
    rec = torch.from_numpy(eng.fetch_records("INS", r0, r1 - r0).astype(np.int64) - rec0).cuda()
    assert int(rec.min()) >= 0 and int(rec.max()) < len(host["L"])
    L = torch.from_numpy(host["L"]).cuda()[rec]
    assert torch.equal(ln64[r0:r1], L)
    assert int(torch.unique(rec).numel()) == r1 - r0   # one row per record
    seq_off, seq4, lut = torch.from_numpy(host["seq_off"]).cuda(), pk["seq4"], torch.from_numpy(BASES).cuda()
    cum = np.concatenate([[0], np.cumsum(host["L"][rec.cpu().numpy()])])
    k = r0
    while k < r1:   # rows [k, e) hold at most CHUNK bytes (or one longer row)
        e = max(k + 1, int(np.searchsorted(cum, cum[k - r0] + CHUNK, side="right")) - 1 + r0)
        e = min(e, r1)
        a, z = int(start[k]), int(start[e - 1]) + int(ln64[e - 1])
        row = torch.repeat_interleave(torch.arange(k, e, device="cuda"), ln64[k:e])
        nib = torch.arange(a, z, device="cuda") - start[row] + 100 + 2 * seq_off[rec[row - r0]]
        byte = seq4[nib >> 1].to(torch.int64)
        want = lut[torch.where((nib & 1) == 1, byte & 15, byte >> 4)]
        got = b[a:z]
        if not torch.equal(got, want):
            i = int(torch.nonzero(got != want)[0])
            raise AssertionError("arena byte %d (row %d) is %r, expected %r" % (a + i, int(row[i]), chr(int(got[i])), chr(int(want[i]))))
        del row, nib, byte, want
        k = e


def _lengths_first_tile_past(n, per_row, extra=64):
    """n distinct lengths of at least per_row each: any 1024 rows sum to 1024 * per_row or more."""
    return per_row + extra + np.arange(n, dtype=np.int64)


def test_first_tile_past_2_30(eng):
    """1040 rows of just over 2^20 bytes: the first scan tile sums past 2^30 (about 1.1 GB of arena in all)."""
    Ls = _lengths_first_tile_past(1040, 1 << 20)
    total = int(Ls.sum())
    _need(total + (total + 400 * len(Ls)) // 2 + 2 * GiB)
    pk, host = _packet(Ls, 1)
    out = eng.extract(pk)
    assert out["counts"]["INS"] == len(Ls)
    _check_arena(eng, pk, host)
    b, _, _ = eng.ins_seq_tensors()
    assert b.numel() == total
    assert total > GiB


def _lengths_total(n, per_row, total):
    """n distinct lengths of at least per_row each that sum to `total`."""
    Ls = per_row + 8 * np.arange(n, dtype=np.int64)
    Ls[-1] = 0
    Ls[-1] = total - Ls.sum()
    assert Ls[-1] > Ls[:-1].max()
    return Ls


def test_first_tile_past_2_31_total_2_32_minus_1(eng):
    """2040 rows of at least 2^21 bytes: the first tile sums past 2^31 and the arena holds exactly 2^32 - 1 bytes, the most one
    packet may add."""
    Ls = _lengths_total(2040, 1 << 21, M32 - 1)
    _need(M32 + M32 // 2 + 3 * GiB)
    pk, host = _packet(Ls, 2)
    out = eng.extract(pk)
    assert out["counts"]["INS"] == len(Ls)
    _check_arena(eng, pk, host)
    b, _, _ = eng.ins_seq_tensors()
    assert b.numel() == M32 - 1
    del pk, b
    eng.extract_reset()


def _small(seed, n=40):
    Ls = 40 + 3 * np.arange(n, dtype=np.int64) + seed
    return _packet(Ls, 100 + seed)


def test_packet_of_4_gib_refused(eng):
    """One packet whose INS strings add up to 2^32 bytes: CSV_E_CAPACITY.  Appended, it leaves the accumulation as it was
    (counts and the strings of the earlier packet) and a later append still works; as a fresh call it leaves it empty."""
    import torch
    _need(M32 // 2 + 2 * GiB)
    s1, h1 = _small(1)
    s2, h2 = _small(2)
    big, _ = _packet(_lengths_total(2040, 1 << 21, M32), 3)
    eng.extract_reset()
    first = eng.extract(s1, append=True)
    counts = [first["counts"][t] for t in _abi.TYPE_NAMES]
    assert counts[INS] == 40
    n_rows, n_pieces = first["n_rows"], first["n_pieces"]
    before = [x.clone() for x in eng.ins_seq_tensors()]
    with pytest.raises(_lib.CuteSVError) as e:
        eng.extract(big, append=True)
    assert e.value.code == _abi.CSV_E_CAPACITY
    assert _holds(eng, counts, n_rows, n_pieces)
    after = eng.ins_seq_tensors()
    assert all(torch.equal(x, y) for x, y in zip(before, after))
    _check_arena(eng, s1, h1)
    second = eng.extract(s2, append=True)
    assert second["counts"]["INS"] == 80 and second["first"]["INS"] == 40
    _check_arena(eng, s1, h1, rows=(0, 40))
    _check_arena(eng, s2, h2, rows=(40, 80), rec0=40)
    with pytest.raises(_lib.CuteSVError) as e:
        eng.extract(big, append=False)
    assert e.value.code == _abi.CSV_E_CAPACITY
    assert _holds(eng, [0] * _abi.CSV_NTYPES, 0, 0)
    with pytest.raises(_lib.CuteSVError) as e:
        eng.ins_seq_tensors()
    assert e.value.code == _abi.CSV_E_STATE
    eng.extract_reset()
