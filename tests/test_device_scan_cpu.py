"""CPU: scanned packets.  The region rule of scan_core.h (scan_in_regions) compiled for the host (tests/emul/emul_scan.cpp) against
the CLI's own numpy rule (cli.bed_filter, what the native source runs for -include_bed) on random windows and regions; the arrays
_abi.scan_regions builds for csv_set_scan_regions; and _abi.scan_packet's argument checks."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from cutesv_b200 import _abi, cli
from test_device_extract_cpu import fake_packet
from test_device_names_cpu import named_packet


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "emul_scan.cpp")
    so = str(tmp_path_factory.mktemp("emul") / "libemul_scan.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-fPIC", "-shared", "-o", so, src])
    return C.CDLL(so)


def _p(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype)) if a is not None and a.size else None


def emul_keep(L, table, chrom, start, end):
    n_contigs, win_off, win_start, reg_off, reg = table
    keep = np.zeros(len(chrom), np.uint8)
    chrom, start, end = (np.ascontiguousarray(x, dtype=np.int32) for x in (chrom, start, end))
    L.emul_scan_keep(C.c_int32(n_contigs), _p(win_off, C.c_int64), _p(win_start, C.c_double), _p(reg_off, C.c_int64), _p(reg, C.c_int64),
                     _p(chrom, C.c_int32), _p(start, C.c_int32), _p(end, C.c_int32), C.c_int64(len(chrom)), _p(keep, C.c_uint8))
    return keep.astype(bool)


def cli_keep(tasks, bed, chrom_id, chrom, start, end):
    pk = {"chrom": np.asarray(chrom, np.int32), "ref_start": np.asarray(start, np.int32), "ref_end": np.asarray(end, np.int32)}
    keep = np.ones(len(chrom), dtype=bool)
    starts, first_task = cli.window_starts(tasks, chrom_id)
    cli.bed_filter(pk, keep, bed, starts, first_task)
    return keep


def random_case(seed, tmp_path):
    """Coverage-balanced windows with fractional bounds (cli.task_windows), BED regions padded by load_bed (negative lo near a
    contig start), many windows without regions, and records placed on window starts, region bounds and contig ends."""
    rng = np.random.default_rng(seed)
    n_ctg = int(rng.integers(1, 6))
    names = ["c%d" % k for k in range(n_ctg)]
    lens = {nm: int(rng.integers(3_000, 200_000)) for nm in names}
    stats = [(nm, int(rng.integers(0, 5_000))) for nm in names]
    tasks, _ = cli.task_windows(stats, lens.__getitem__, int(rng.integers(1, 8)), int(rng.choice([10_000_000, 7_777, 20_001])))
    lines = []
    for nm in names:
        for _ in range(int(rng.integers(0, 12))):
            lo = int(rng.integers(0, lens[nm]))
            lines.append("%s\t%d\t%d\n" % (nm, lo, lo + int(rng.integers(1, 3_000))))
    bed_path = tmp_path / ("r%d.bed" % seed)
    bed_path.write_text("".join(lines))
    bed = cli.load_bed(str(bed_path), tasks)
    chrom_id = {nm: i for i, nm in enumerate(sorted(names))}
    # record starts: random, every window start (rounded both ways, and +-1), every region bound +-1
    pts = [(chrom_id[t[0]], int(np.floor(t[1])) + d) for t in tasks for d in (-1, 0, 1)]
    pts += [(chrom_id[t[0]], int(np.ceil(t[1]))) for t in tasks]
    for t, regs in zip(tasks, bed):
        for lo, hi in regs:
            pts += [(chrom_id[t[0]], v + d) for v in (lo, hi) for d in (-1, 0, 1)]
    pts += [(chrom_id[nm], lens[nm] - int(rng.integers(1, 50))) for nm in names]
    pts += [(int(rng.integers(0, n_ctg)), int(rng.integers(0, 200_000))) for _ in range(2_000)]
    chrom = np.array([c for c, _ in pts], np.int32)
    start = np.maximum(np.array([s for _, s in pts], np.int64), 0).astype(np.int32)
    span = rng.choice([0, 1, 2, 500, 3_000, 20_000], len(pts))
    end = (start + span).astype(np.int32)
    # ends exactly on a region's lo: shift some records so that end == lo
    for t, regs in zip(tasks, bed):
        for lo, hi in regs:
            if lo > 0:
                chrom = np.append(chrom, np.int32(chrom_id[t[0]]))
                start = np.append(start, np.int32(max(lo - 100, 0)))
                end = np.append(end, np.int32(lo))
    return tasks, bed, chrom_id, chrom, start, end


@pytest.mark.parametrize("seed", range(24))
def test_region_rule_equals_the_cli_numpy_rule(emul, tmp_path, seed):
    tasks, bed, chrom_id, chrom, start, end = random_case(seed, tmp_path)
    table = _abi.scan_regions(tasks, bed, chrom_id)
    got = emul_keep(emul, table, chrom, start, end)
    want = cli_keep(tasks, bed, chrom_id, chrom, start, end)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]


def test_fractional_window_bounds_and_edges(emul):
    # one contig, windows [0, 2.5), [2.5, 5), [5, 7.5) ...; regions on the second and last windows only
    tasks = [["c", 0, 2.5], ["c", 2.5, 5.0], ["c", 5.0, 7.5], ["c", 7.5, 10]]
    bed = [[], [(-1000, 3)], [], [(8, 9), (20, 30)]]
    chrom_id = {"c": 0}
    start = np.array([2, 3, 3, 4, 5, 7, 8, 8, 9, 9, 25], np.int32)
    end = np.array([3, 3, 4, 6, 6, 8, 8, 9, 9, 10, 26], np.int32)
    chrom = np.zeros(len(start), np.int32)
    want = cli_keep(tasks, bed, chrom_id, chrom, start, end)
    # start 2 < 2.5: window 0 (no regions); 3 >= 2.5: window 1, region [-1000, 3) needs start < 3; 8 >= 7.5: last window
    assert want.tolist() == [False, False, False, False, False, False, False, True, False, False, True]
    assert np.array_equal(emul_keep(emul, _abi.scan_regions(tasks, bed, chrom_id), chrom, start, end), want)


def test_contig_without_window_and_no_table(emul):
    tasks = [["a", 0, 100]]
    chrom_id = {"a": 0, "b": 1}
    table = _abi.scan_regions(tasks, [[(-1000, 1100)]], chrom_id)
    assert table[0] == 2 and table[1].tolist() == [0, 1, 1]
    got = emul_keep(emul, table, [0, 1, 2], [5, 5, 5], [6, 6, 6])
    assert got.tolist() == [True, False, False]   # contig 1 has no window, 2 is beyond the table
    assert _abi.scan_regions(tasks, None, chrom_id)[0] == 0
    assert emul_keep(emul, (0, None, None, None, None), [0, 1, 7], [5, 5, 5], [6, 6, 6]).all()


def test_scan_regions_arrays():
    tasks = [["b", 0, 10.5], ["a", 0, 4], ["b", 10.5, 21], ["a", 4, 8]]
    bed = [[(1, 2)], [], [(3, 4), (5, 6)], [(-7, 8)]]
    n, win_off, win_start, reg_off, reg = _abi.scan_regions(tasks, bed, {"a": 0, "b": 1})
    assert n == 2 and win_off.tolist() == [0, 2, 4]
    assert win_start.dtype == np.float64 and win_start.tolist() == [0, 4, 0, 10.5]
    assert reg_off.tolist() == [0, 0, 1, 2, 4]
    assert reg.dtype == np.int64 and reg.tolist() == [[-7, 8], [1, 2], [3, 4], [5, 6]]
    with pytest.raises(ValueError, match="region lists"):
        _abi.scan_regions(tasks, bed[:3], {"a": 0, "b": 1})


def test_scan_packet_checks():
    d = _abi.scan_packet(named_packet(), 0)
    assert d.names is not None and d[0].n == 5
    with pytest.raises(ValueError, match="names"):
        _abi.scan_packet(fake_packet(), 0)   # read_id instead of names
    host = {f: np.zeros(3, np.int32) for f in _abi.READ_FIELDS}
    host.update(cigar_off=np.zeros(4, np.int64), sa_off=np.zeros(4, np.int64), cigar=np.zeros(0, np.uint32),
                sa={f: np.zeros(0, np.int32) for f in _abi.SA_FIELDS})
    with pytest.raises(ValueError, match="GPU memory"):
        _abi.scan_packet(host, 0)
    with pytest.raises(ValueError, match="go together"):
        _abi.scan_packet(named_packet(names=None), 0)
    with pytest.raises(ValueError, match="device 1"):
        _abi.scan_packet(named_packet(names=named_packet()["names"].__class__(40, "|u1", device=1)), 0)
