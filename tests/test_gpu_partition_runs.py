"""-m gpu: the partitioned INS/DEL front end's run table against the oracle.

k_part_scatter groups every round of 8192 rows by partition and writes it back in place; k_part_filter reads a partition
as its list of runs, one per round, most of them short and many empty.  These inputs put the runs at their extremes:
row counts around a round, a round whose rows all fall in one partition (and spill its stage), a partition fed by one
round only, rows in exactly the first and last rb buckets of partitions (the scatter's edge counts), close to the
largest partition count, and rows the scatter's validation must refuse.  Multiples of 2^22 in contig 0 (linear offset
0) are partition edges whatever partition width the library picks."""
import numpy as np
import pytest

from cutesv_b200 import _abi, _lib
from cutesv_b200.engine import Engine
from test_gpu_partition_filter import PARAMS, _cat, _check, _cols
from test_gpu_partition_rounds import SMALL_LENS, _noise

pytestmark = pytest.mark.gpu

ROUND = 8192
EDGE = 1 << 22
RB = 2   # PARAMS: (min_support - 1) * bias = 400 bp -> 2 buckets


def _engine(cfg):
    return Engine(0, params=_abi.default_params(**cfg["params"]), contig_lens=cfg["lens"])


def _put(cfg, name, row, cols):
    """Overwrite rows row .. row + len - 1 of one type with `cols` (the row count stays)."""
    sig = cfg["sigs"][name]
    k = len(cols["chrom"])
    for key, v in cols.items():
        if v is not None:
            sig[key][row:row + k] = v


def _block(rng, n, pos, ins, n_reads=20000):
    return _cols(np.zeros(n), pos, np.where(rng.random(n) < 0.5, 300, 900) + rng.integers(-20, 20, n),
                 rng.integers(0, n_reads, n), ins, rng.integers(0, 2, n) if ins else None)


def test_row_counts_around_a_round():
    """65 536 rows, 8192 k +- 1, 8192 k +- 4 and counts that are not multiples of 4, on one engine."""
    counts = [(65536, 65536 + 3), (ROUND * 9 - 1, ROUND * 9 + 1), (ROUND * 10 - 4, ROUND * 10 + 4), (ROUND * 11 + 2, 70001)]
    eng = None
    try:
        for i, (nd, ni) in enumerate(counts):
            cfg = _noise(40 + i, SMALL_LENS, dict(DEL=nd, INS=ni))
            eng = eng or _engine(cfg)
            assert _check(eng, cfg) > 0
    finally:
        if eng:
            eng.close()


def test_one_round_in_one_partition_spills():
    """Every row of round 2 (DEL) and of round 5 (INS) in one partition: one full run, empty runs of that round for every
    other partition, and far more survivors than the partition's shared-memory stage holds."""
    rng = np.random.default_rng(50)
    cfg = _noise(50, SMALL_LENS, dict(DEL=ROUND * 10 + 5, INS=ROUND * 9 + 3))
    _put(cfg, "DEL", 2 * ROUND, _block(rng, ROUND, 2 * EDGE + rng.integers(0, 1 << 16, ROUND), False))
    _put(cfg, "INS", 5 * ROUND, _block(rng, ROUND, EDGE + rng.integers(0, 1 << 16, ROUND), True))
    eng = _engine(cfg)
    try:
        assert _check(eng, cfg) > 0
    finally:
        eng.close()


def test_partition_fed_by_one_round():
    """A partition whose only rows (five clusters of six) lie in round 4: every other round's run for it is empty."""
    rng = np.random.default_rng(60)
    cfg = _noise(60, SMALL_LENS, dict(DEL=ROUND * 10 + 1, INS=ROUND * 10 + 7))
    lo, hi = 3 * EDGE, 3 * EDGE + (1 << 16)
    for name in ("DEL", "INS"):
        ins = name == "INS"
        sig = cfg["sigs"][name]
        pos = sig["a"].astype(np.int64) >> (1 if ins else 0)
        move = (sig["chrom"] == 0) & (pos >= lo - 2048) & (pos < hi + 2048)   # the partition and its halo left empty
        sig["a"][move] += (2 if ins else 1) * 200_000
        parts = [_cols(np.zeros(6), lo + 9000 * k + 500 + rng.integers(0, 200, 6), 400 + rng.integers(-5, 5, 6),
                       rng.integers(0, 20000, 6), ins, rng.integers(0, 2, 6) if ins else None) for k in range(5)]
        _put(cfg, name, 4 * ROUND + 100, _cat(parts))
    eng = _engine(cfg)
    try:
        assert _check(eng, cfg) > 0
    finally:
        eng.close()


def test_rows_in_the_edge_buckets():
    """Clusters whose members sit in exactly the last rb buckets of a partition and the first rb buckets of the next (and
    one bucket further, outside the halo), so that only the scatter's edge counts bring them to min_support."""
    rng = np.random.default_rng(70)
    cfg = _noise(70, SMALL_LENS, dict(DEL=ROUND * 12 + 3, INS=ROUND * 12 + 1))
    for name in ("DEL", "INS"):
        ins = name == "INS"
        parts = []
        for e in range(1, 5):
            E = e * EDGE
            for offs in ([-RB * 256, -300, -1, 0, 250, RB * 256 - 1],         # both sides' edge buckets
                         [-RB * 256 - 1, -RB * 256, -1, 0, 1, RB * 256 - 1],   # one member just outside the halo
                         [-RB * 256, -200, -2, RB * 256 - 256, RB * 256 - 1],  # five: min_support exactly
                         [-1, 0]):                                              # too few anywhere
                k = len(offs)
                parts.append(_cols(np.zeros(k), E + np.array(offs), 500 + rng.integers(-3, 3, k),
                                   rng.integers(0, 20000, k), ins, rng.integers(0, 2, k) if ins else None))
        _put(cfg, name, 3 * ROUND + 17, _cat(parts))
    eng = _engine(cfg)
    try:
        assert _check(eng, cfg) > 0
    finally:
        eng.close()


def test_close_to_the_largest_partition_count():
    """Three contigs of about 1.4 Gb: a linear span just under 2^32, about 1 000 partitions of 2^22 bp."""
    lens = np.array([1_400_000_000, 1_400_000_000, 1_390_000_000], dtype=np.int64)
    rng = np.random.default_rng(80)
    n_reads = 20000
    reads_chrom = rng.integers(0, 3, n_reads).astype(np.int32)
    r_start = (rng.random(n_reads) * (lens[reads_chrom] - 20000)).astype(np.int64)
    reads = dict(chrom=reads_chrom, start=r_start.astype(np.int32), end=(r_start + 15000).astype(np.int32),
                 read_id=np.arange(n_reads, dtype=np.int32), is_primary=np.ones(n_reads, np.uint8))
    sigs = {}
    for name, n in (("DEL", 70001), ("INS", 69999)):
        ins = name == "INS"
        top = np.minimum(lens, 1_000_000_000) if ins else lens   # INS keeps 2 * pos below 2^31
        n_cl = 6 * 60
        ch = rng.integers(0, 3, n - n_cl)
        pos = (rng.random(n - n_cl) * (top[ch] - 10)).astype(np.int64)
        parts = [_cols(ch, pos, 60 + rng.integers(0, 400, n - n_cl), rng.integers(0, n_reads, n - n_cl), ins,
                       rng.integers(0, 2, n - n_cl) if ins else None)]
        for k in range(60):   # clusters of six across partition edges of every contig
            c = k % 3
            E = int(rng.integers(1, int(top[c]) // EDGE)) * EDGE
            parts.append(_cols(np.full(6, c), E - 150 + rng.integers(0, 300, 6), 400 + rng.integers(-5, 5, 6),
                               rng.integers(0, n_reads, 6), ins, rng.integers(0, 2, 6) if ins else None))
        cols = _cat(parts)
        perm = rng.permutation(n)
        sigs[name] = {k: None if v is None else v[perm] for k, v in cols.items()}
    cfg = dict(lens=lens, sigs=sigs, reads=reads, params=dict(PARAMS))
    pad = 1001
    assert int((lens + pad).sum()) < 1 << 32 and int((lens + pad).sum()) >> 22 >= 990
    eng = _engine(cfg)
    try:
        assert _check(eng, cfg) > 0
    finally:
        eng.close()


@pytest.mark.parametrize("bad", ["contig", "past_contig", "negative"])
def test_scatter_refuses_invalid_rows(bad):
    """One invalid row in an input that takes the filter: csv_cluster fails with CSV_E_INPUT, and the engine clusters a
    valid input correctly afterwards."""
    cfg = _noise(90, SMALL_LENS, dict(DEL=ROUND * 9 + 3, INS=ROUND * 9 + 1))
    good = {k: {c: None if v is None else v.copy() for c, v in s.items()} for k, s in cfg["sigs"].items()}
    name = "INS" if bad == "past_contig" else "DEL"
    sig = cfg["sigs"][name]
    row = 5 * ROUND + 77
    if bad == "contig":
        sig["chrom"][row] = len(SMALL_LENS)
    elif bad == "past_contig":
        sig["a"][row] = 2 * (int(SMALL_LENS[sig["chrom"][row]]) + 1)
    else:
        sig["a"][row] = -5
    eng = _engine(cfg)
    try:
        with pytest.raises(_lib.CuteSVError) as err:
            eng.cluster(cfg["sigs"], cfg["reads"])
        assert err.value.code == _abi.CSV_E_INPUT
        cfg["sigs"] = good
        assert _check(eng, cfg) > 0
    finally:
        eng.close()
