"""-m gpu: the partitioned INS/DEL front end's paged layout against the oracle.

k_part_scatter reserves ordinals of a partition for every round and writes its pairs into that partition's pages of
2048 pairs, drawn from one pool; k_part_filter reads the partition's pages and resets its fill counter and page-table
entries.  These inputs put the pages at their extremes: partitions of a page's size +- 1, reservations that cross page
boundaries, a round that fills eight pages of one partition, empty partitions, the largest pool (every partition with a
partly filled page), close to the largest partition count with many rounds, and one engine that must find a clean table
on every call: repeated calls, calls of different sizes and a call after the scatter refused invalid rows.  Multiples of
2^22 in contig 0 (linear offset 0) are partition starts whatever partition width the library picks, and a partition is
at least 2^16 bp wide."""
import numpy as np
import pytest

from cutesv_b200 import _abi, _lib
from cutesv_b200.engine import Engine
from test_gpu_partition_filter import PARAMS, _cat, _check, _cols

pytestmark = pytest.mark.gpu

PAGE = 2048
ROUND = 16384
EDGE = 1 << 22
PART_MIN = 1 << 16
LENS = np.array([60_000_000, 40_000_003], dtype=np.int64)
N_READS = 20000


def _reads(rng, lens):
    weights = lens / lens.sum()
    chrom = rng.choice(len(lens), N_READS, p=weights).astype(np.int32)
    start = (rng.random(N_READS) * (lens[chrom] - 20000)).astype(np.int64)
    return dict(chrom=chrom, start=start.astype(np.int32), end=(start + 15000).astype(np.int32),
                read_id=np.arange(N_READS, dtype=np.int32), is_primary=np.ones(N_READS, np.uint8))


def _rows(rng, chrom, pos, ins):
    k = len(pos)
    return _cols(np.full(k, chrom), pos, np.where(rng.random(k) < 0.5, 300, 900) + rng.integers(-20, 20, k),
                 rng.integers(0, N_READS, k), ins, rng.integers(0, 2, k) if ins else None)


def _paged(seed, sizes, n, shuffle=True):
    """sizes[j] rows in the first 2^16 bp of partition start (j + 1) * 2^22 of contig 0, the other rows spread over contig
    1 (so every other partition of contig 0 is empty); rows shuffled unless `shuffle` is False."""
    rng = np.random.default_rng(seed)
    sigs = {}
    for name in ("DEL", "INS"):
        ins = name == "INS"
        parts = [_rows(rng, 0, (j + 1) * EDGE + 512 + rng.integers(0, PART_MIN - 1024, k), ins) for j, k in enumerate(sizes)]
        rest = n - sum(sizes)
        parts.append(_rows(rng, 1, (rng.random(rest) * (LENS[1] - 10)).astype(np.int64), ins))
        cols = _cat(parts)
        perm = rng.permutation(n) if shuffle else np.arange(n)
        sigs[name] = {k: None if v is None else v[perm] for k, v in cols.items()}
    return dict(lens=LENS, sigs=sigs, reads=_reads(rng, LENS), params=dict(PARAMS))


def _engine(cfg):
    return Engine(0, params=_abi.default_params(**cfg["params"]), contig_lens=cfg["lens"])


def _run(*cfgs):
    eng = _engine(cfgs[0])
    try:
        for cfg in cfgs:
            assert _check(eng, cfg) > 0
    finally:
        eng.close()


def test_partitions_around_a_page():
    """Partitions of PAGE - 1, PAGE, PAGE + 1, 2 PAGE and 2 PAGE + 1 rows fed by every round, so that reservations of
    about 300 rows cross page boundaries, beside empty partitions."""
    _run(_paged(100, [PAGE - 1, PAGE, PAGE + 1, 2 * PAGE, 2 * PAGE + 1], 7 * ROUND + 5))


def test_one_round_fills_pages_of_one_partition():
    """Round 2 entirely in one partition that every other round also feeds: the round's reservation of 16 384 rows spans
    eight or nine pages and usually starts inside one; the partition spills its shared-memory stage."""
    cfg = _paged(110, [3 * ROUND + 777], 8 * ROUND + 3, shuffle=False)
    rng = np.random.default_rng(111)
    for name in ("DEL", "INS"):   # rows 0 .. 3 ROUND + 776 are the partition's; ROUND of them make round 2
        sig = cfg["sigs"][name]
        n = len(sig["chrom"])
        part = np.arange(3 * ROUND + 777)
        rest = np.concatenate([part[ROUND:], np.arange(len(part), n)])
        order = np.empty(n, np.int64)
        order[2 * ROUND:3 * ROUND] = part[:ROUND]
        order[np.r_[0:2 * ROUND, 3 * ROUND:n]] = rest[rng.permutation(len(rest))]
        for k, v in sig.items():
            if v is not None:
                sig[k] = v[order]
    _run(cfg)


def test_largest_pool():
    """A row every 2^16 bp of the linear coordinate (at least one in every partition, one partly filled page each) and
    every other row in one partition."""
    rng = np.random.default_rng(120)
    p = _abi.default_params(**PARAMS)
    pad = max(p.bias_del, p.bias_ins, p.bias_inv, p.bias_dup, p.bias_tra, p.gt_bias_ins) + 1
    off = np.concatenate([[0], np.cumsum(LENS + pad)])
    lin = np.arange(100, int(off[-1]), PART_MIN)
    ch = np.searchsorted(off, lin, side="right") - 1
    pos = lin - off[ch]
    keep = pos < LENS[ch] - 10
    ch, pos = ch[keep], pos[keep]
    n = 65536 + 3
    sigs = {}
    for name in ("DEL", "INS"):
        ins = name == "INS"
        single = _cols(ch, pos, 400 + rng.integers(-5, 5, len(ch)), rng.integers(0, N_READS, len(ch)), ins,
                       rng.integers(0, 2, len(ch)) if ins else None)
        big = _rows(rng, 0, 2 * EDGE + 512 + rng.integers(0, PART_MIN - 1024, n - len(ch)), ins)
        cols = _cat([single, big])
        perm = rng.permutation(n)
        sigs[name] = {k: None if v is None else v[perm] for k, v in cols.items()}
    _run(dict(lens=LENS, sigs=sigs, reads=_reads(rng, LENS), params=dict(PARAMS)))


def test_close_to_the_largest_partition_count_many_rounds():
    """Three contigs of about 1.4 Gb (about 1 000 partitions of 2^22 bp) and 20 rounds per type, with partitions of a
    page's size +- 1 planted at partition starts."""
    lens = np.array([1_400_000_000, 1_400_000_000, 1_390_000_000], dtype=np.int64)
    rng = np.random.default_rng(130)
    n = 20 * ROUND - 11
    planted = [PAGE - 1, PAGE, PAGE + 1]
    sigs = {}
    for name in ("DEL", "INS"):
        ins = name == "INS"
        top = np.minimum(lens, 1_000_000_000) if ins else lens   # INS keeps 2 * pos below 2^31
        parts = [_rows(rng, 0, (7 + 50 * j) * EDGE + 512 + rng.integers(0, PART_MIN - 1024, k), ins) for j, k in enumerate(planted)]
        m = n - sum(planted)
        ch = rng.integers(0, 3, m)
        pos = (rng.random(m) * (top[ch] - 10)).astype(np.int64)
        stray = (ch == 0) & np.isin(pos // EDGE, [7 + 50 * j for j in range(len(planted))])
        pos[stray] += EDGE   # the planted partitions hold exactly their rows
        parts.append(_cols(ch, pos, 60 + rng.integers(0, 400, m), rng.integers(0, N_READS, m), ins,
                           rng.integers(0, 2, m) if ins else None))
        cols = _cat(parts)
        perm = rng.permutation(n)
        sigs[name] = {k: None if v is None else v[perm] for k, v in cols.items()}
    _run(dict(lens=lens, sigs=sigs, reads=_reads(rng, lens), params=dict(PARAMS)))


def test_one_engine_repeated_and_resized_calls():
    """One engine: the same input three times (eager, graph capture, replay), then smaller, larger and the first again.
    Page-table rows change width with the row count, so any entry a filter left set would corrupt a later call."""
    a = _paged(140, [PAGE + 1, 3 * PAGE - 1], 6 * ROUND + 1)
    b = _paged(141, [PAGE - 1, PAGE], 4 * ROUND + 9)
    c = _paged(142, [5 * PAGE + 3, PAGE, 1], 11 * ROUND + 2)
    _run(a, a, a, b, c, c, a)


@pytest.mark.parametrize("name", ["DEL", "INS"])
def test_call_after_refused_rows(name):
    """An invalid row makes csv_cluster fail with CSV_E_INPUT after the scatter ran; the next call on the engine, with
    partitions around a page, finds a clean table."""
    cfg = _paged(150, [PAGE + 1, PAGE - 1], 6 * ROUND + 7)
    good = {k: {c: None if v is None else v.copy() for c, v in s.items()} for k, s in cfg["sigs"].items()}
    cfg["sigs"][name]["chrom"][3 * ROUND + 5] = len(LENS)
    eng = _engine(cfg)
    try:
        with pytest.raises(_lib.CuteSVError) as err:
            eng.cluster(cfg["sigs"], cfg["reads"])
        assert err.value.code == _abi.CSV_E_INPUT
        cfg["sigs"] = good
        assert _check(eng, cfg) > 0
        assert _check(eng, cfg) > 0
    finally:
        eng.close()
