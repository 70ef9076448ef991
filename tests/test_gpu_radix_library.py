"""-m gpu: the library's own radix_sort() driver through its callers, at the radix sort's round, tile and wave edges.
csv_sort_sigs on DEL and TRA columns whose key is exactly 32, 33, 64, 65, 128 or 129 bits (tests/radix_cases.py), against
numpy's lexsort, with the onesweep launches of the profiled call counted; csv_sort_sigs on the reads table at 1, 2, 256 and 257
contigs and at n = T ± 1 and W·T ± 1; csv_rank_names on 8- and 9-byte names around the uint64 tile and wave, against Python's
sorted()."""
import os
import sys

import numpy as np
import pytest

import device_packet_util as dpu
import name_util
import radix_cases as R
import sigs_dropin_data as D
from cutesv_b200 import _abi

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "gpu_prims"))
import prims_lib  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def prof():
    """A context of its own with profiling on: its kernel table names what the last call launched."""
    from cutesv_b200._lib import CuteSVError
    from cutesv_b200.engine import Engine
    try:
        e = Engine(0)
    except CuteSVError as err:
        if err.code == _abi.CSV_E_NODEVICE:
            pytest.skip("no usable sm_90 device: %s" % err)
        raise
    e.set_profiling(True)
    yield e
    e.close()


def _onesweep_launches(eng):
    return sum(n for name, (n, _) in eng.kernel_times().items() if name.startswith("k_rs_onesweep"))


def _sort_and_check(eng, svtype, cols, nc):
    want = D.np_sort_sigs(svtype, cols, nc)
    got = eng.sort_sigs(svtype)
    for k in ("order", "contig_off"):
        assert np.array_equal(got[k], want[k]), k


def _edge_cols(rng, svtype, maxima, n):
    """n rows of few distinct values per field (many exact duplicates and ties), each field's largest value planted."""
    cols = {}
    for f in R.FIELDS[svtype]:
        mx = maxima[f]
        vals = np.unique(np.concatenate([[0, mx, mx // 2], rng.integers(0, mx + 1, 4)]))
        if f == "c":   # chr2 * 4 + type with chr2 a contig
            vals = vals[(vals >> 2) <= maxima["chrom"]]
        cols[f] = rng.choice(vals, n).astype(np.int32)
        cols[f][rng.integers(0, n)] = mx
    cols.setdefault("c", None)
    return cols


@pytest.mark.parametrize("name", list(R.ROUND_EDGES))
def test_sort_sigs_round_edges(prof, name):
    svtype, maxima, total = R.ROUND_EDGES[name]
    nc = R.n_contigs(svtype, maxima)
    n = 20011
    cols = _edge_cols(np.random.default_rng(total), svtype, maxima, n)
    prof.set_contigs(np.full(nc, (1 << 31) - 1, np.int64))
    prof.upload({svtype: cols}, None)
    _sort_and_check(prof, svtype, cols, nc)
    assert _onesweep_launches(prof) == R.onesweep_passes(total)


@pytest.mark.parametrize("size", ["T-1", "T+1", "WT-1", "WT+1"])
@pytest.mark.parametrize("nc", [1, 2, 256, 257])
def test_sort_reads_table_at_tile_and_wave_edges(prof, nc, size):
    """The reads table's key is the contig alone: 1, 1, 8 and 9 bits, one or two uint32 passes."""
    T, WT = prims_lib.rs_tile(4), prims_lib.rs_wave(4)
    n = {"T-1": T - 1, "T+1": T + 1, "WT-1": WT - 1, "WT+1": WT + 1}[size]
    rng = np.random.default_rng(nc * 7 + n)
    chrom = rng.integers(0, nc, n).astype(np.int32)
    chrom[rng.integers(0, n)] = nc - 1
    s = rng.integers(0, 1 << 20, n).astype(np.int32)
    reads = dict(chrom=chrom, start=s, end=s + 5, read_id=rng.integers(0, 50, n).astype(np.int32), is_primary=np.ones(n, np.uint8))
    prof.set_contigs(np.full(nc, 1 << 21, np.int64))
    prof.upload({}, reads)
    _sort_and_check(prof, "reads", reads, nc)
    assert _onesweep_launches(prof) == (2 if nc == 257 else 1)


def _names(rng, n, width):
    """n ASCII names of 8 bytes (width 8), or of 8 and 9 bytes (width 9, half of the 9-byte ones an 8-byte name plus one
    byte); about one in eight repeats an earlier name."""
    alpha = np.frombuffer(b"0123456789abcdef", np.uint8)
    raw = alpha[rng.integers(0, 16, (n, 9))]
    out = [bytes(r[:8]).decode() for r in raw]
    if width == 9:
        for i in np.flatnonzero(rng.random(n) < 0.5).tolist():
            out[i] = (out[i - 1] if i and i % 2 else out[i])[:8] + chr(raw[i, 8])
    for i in np.flatnonzero(rng.random(n) < 0.125).tolist():
        out[i] = out[int(rng.integers(0, n))]
    return out


def _name_packet(n):
    """n records on one contig, CIGAR 100M each, no SA and no bases."""
    start = (1000 + 7 * np.arange(n, dtype=np.int64)) % 5_000_000
    return dict(chrom=np.zeros(n, np.int32), ref_start=start.astype(np.int32), ref_end=(start + 100).astype(np.int32), flag=np.zeros(n, np.int32),
                mapq=np.full(n, 60, np.int32), query_len=np.full(n, 100, np.int32), read_id=np.arange(n, dtype=np.int32),
                cigar_off=np.arange(n + 1, dtype=np.int64), sa_off=np.zeros(n + 1, np.int64), cigar=np.full(n, 100 << 4, np.uint32),
                sa={k: np.zeros(0, np.int32) for k in _abi.SA_FIELDS})


@pytest.mark.parametrize("width", [8, 9])
@pytest.mark.parametrize("size", ["T-1", "T", "T+1", "WT-1", "WT+1"])
def test_rank_names_at_tile_and_wave_edges(engine, size, width):
    """One uint32 length round, then one (8 bytes) or two (9 bytes) uint64 word rounds over T = 3072-key tiles."""
    T, WT = prims_lib.rs_tile(8), prims_lib.rs_wave(8)
    n = {"T-1": T - 1, "T": T, "T+1": T + 1, "WT-1": WT - 1, "WT+1": WT + 1}[size]
    names = _names(np.random.default_rng(n + width), n, width)
    assert max(map(len, names)) == width
    engine.set_params(_abi.default_params(min_mapq=0, min_read_len=100))
    engine.set_contigs(np.array([10_000_000], np.int64))
    engine.extract_reset()
    engine.extract(name_util.named(dpu.to_device(_name_packet(n)), names), append=True)
    nd = engine.rank_names()
    srt = sorted(set(names))
    assert nd == len(srt)
    got = engine.name_rank_tensor().cpu().numpy()
    bad = np.flatnonzero(got != name_util.dense_ranks(names))
    assert len(bad) == 0, "%d of %d ranks wrong, first at record %d (%r)" % (len(bad), n, bad[0], names[bad[0]])
    pick = np.unique(np.concatenate([[0, nd - 1], np.random.default_rng(n).integers(0, nd, 500)]))
    assert engine.fetch_names(pick) == [srt[i] for i in pick.tolist()]
