"""-m gpu: the partitioned density filter at the extremes of its window radius rb (in 256-bp buckets), against the oracle
and the filter rule (test_gpu_partition_filter._check).

rb = 1 (min_support 3, bias 100) keeps a bucket on its direct neighbours alone.  rb = 63 (min_support 5, bias 4000) needs
a sparse genome of about 640 Mb to take the filter; the library then cuts it into partitions of 2^21 bp, whose strips of
32 buckets per thread are shorter than the window, so every window spans several strips.  Clusters are planted across
partition edges (multiples of 2^21 in contig 0, whose linear offset is 0) where only the neighbour's halo completes them."""
import numpy as np
import pytest

import test_gpu_partition_filter as tpf
from cutesv_b200 import _abi
from cutesv_b200.engine import Engine

pytestmark = pytest.mark.gpu

BKT = 256
EDGE = 1 << 21


def _dataset(seed, lens, n_noise, params, plant):
    """Uniform noise over the contigs plus plant(edge) -> [bucket offsets from the edge] per partition edge of contig 0."""
    rng = np.random.default_rng(seed)
    n_reads = 20000
    weights = lens / lens.sum()
    reads_chrom = rng.choice(len(lens), n_reads, p=weights).astype(np.int32)
    r_start = (rng.random(n_reads) * (lens[reads_chrom] - 20000)).astype(np.int64)
    reads = dict(chrom=reads_chrom, start=r_start.astype(np.int32), end=(r_start + 15000).astype(np.int32),
                 read_id=np.arange(n_reads, dtype=np.int32), is_primary=np.ones(n_reads, np.uint8))
    sigs = {}
    for name in ("DEL", "INS"):
        ins = name == "INS"
        ch = rng.choice(len(lens), n_noise, p=weights)
        pos = (rng.random(n_noise) * (lens[ch] - 10)).astype(np.int64)
        parts = [tpf._cols(ch, pos, 60 + rng.integers(0, 400, n_noise), rng.integers(0, n_reads, n_noise), ins,
                           rng.integers(0, 2, n_noise) if ins else None)]
        for e in range(1, int(lens[0] // EDGE)):
            buckets = np.asarray(plant(e), np.int64)
            k = len(buckets)
            p = e * EDGE + buckets * BKT + rng.integers(0, BKT, k)
            parts.append(tpf._cols(np.zeros(k), p, 400 + rng.integers(-5, 5, k), rng.integers(0, n_reads, k), ins,
                                   rng.integers(0, 2, k) if ins else None))
        sigs[name] = tpf._cat(parts)
    return dict(lens=lens, sigs=sigs, reads=reads, params=params)


def _run(cfg):
    eng = Engine(0, params=_abi.default_params(**cfg["params"]), contig_lens=cfg["lens"])
    try:
        for _ in range(3):   # graph capture and replay
            assert tpf._check(eng, cfg) > 0
    finally:
        eng.close()


def test_radius_1():
    """rb = 1: a pair and a single member in adjacent buckets across an edge, a member two buckets away that the window
    must not count, and clusters of three in one bucket on either side of the edge."""
    lens = np.array([20 * EDGE + 12345, 12 * EDGE + 777, 8 * EDGE + 5], dtype=np.int64)
    params = dict(min_support=3, bias_del=100, bias_ins=100, ratio_del=0.3, ratio_ins=0.3, genotype=1)
    plants = [[-1, -1, 0], [-1, 0, 0, 2], [-2, 0, 0], [-1, -1, -1], [0, 0, 0, 1]]
    _run(_dataset(11, lens, 70000, params, lambda e: plants[e % len(plants)]))


def test_radius_63():
    """rb = 63 at 2^21-bp partitions: members up to 63 buckets from each other across an edge (kept only through the
    halo), members 64 buckets apart (not in one window), and pile-ups far inside a partition."""
    lens = np.array([150 * EDGE + 12345, 100 * EDGE + 777, 55 * EDGE + 5], dtype=np.int64)
    params = dict(min_support=5, bias_del=4000, bias_ins=4000, ratio_del=0.3, ratio_ins=0.3, genotype=1)
    plants = [[-40, -40, 20, 20, 23], [-63, -63, 0, 0, 0], [-1, 62, 62, 62, 62], [-32, -32, 32, 32, 32],
              [-64, -64, 0, 0], [-30, -30, -30, 34, 34], [500, 500, 501, 502, 560, 560]]
    _run(_dataset(12, lens, 68000, params, lambda e: plants[e % len(plants)]))
