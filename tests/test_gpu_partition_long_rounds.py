"""-m gpu: k_part_scatter's rounds of 16 384 rows against the oracle.

One 1024-thread CTA scatters a round of ROUND rows: two bulk copies bring the round's whole 4-row groups into shared
memory, the rows of a last partial group are loaded one by one, and the grouped pairs are written back over the same
shared memory.  These inputs sit at the round's edges: row counts around multiples of a round, last rounds shorter than
one 16 B group (no bulk copy at all), clusters whose members straddle a round edge, a round whose rows all fall into one
partition (one run of ROUND pairs, spilling the filter's stage) and a round that feeds every partition.  The genome of
34 Mb makes the library pick partitions of 2^16 bp on a 132-SM H100, so a round spread over it reaches all of them."""
import numpy as np
import pytest

from cutesv_b200 import _abi
from cutesv_b200.engine import Engine
from test_gpu_partition_filter import _cat, _check, _cols
from test_gpu_partition_rounds import SMALL_LENS, _noise
from test_gpu_partition_runs import EDGE, _block, _put

pytestmark = pytest.mark.gpu

ROUND = 16384   # the filter is taken from 65 536 rows on, and up to about 100 000 on this genome: 5 or 6 rounds


def _engine(cfg):
    return Engine(0, params=_abi.default_params(**cfg["params"]), contig_lens=cfg["lens"])


def _check_all(cfgs):
    eng = None
    try:
        for cfg in cfgs:
            eng = eng or _engine(cfg)
            assert _check(eng, cfg) > 0
    finally:
        if eng:
            eng.close()


def test_row_counts_around_a_round():
    """Counts at 16 384 k +- 1 and +- 4, and counts that are not multiples of 4, on one engine."""
    counts = [(ROUND * 5 - 1, ROUND * 5 + 1), (ROUND * 6 - 4, ROUND * 6 + 4), (ROUND * 5 + 6, ROUND * 6 - 3), (ROUND * 5, 70001)]
    _check_all([_noise(100 + i, SMALL_LENS, dict(DEL=nd, INS=ni)) for i, (nd, ni) in enumerate(counts)])


def test_last_round_shorter_than_one_group():
    """A last round of 1, 2 and 3 rows: no whole 4-row group, so the round takes no bulk copy."""
    counts = [(ROUND * 5 + 1, ROUND * 5 + 2), (ROUND * 5 + 3, ROUND * 6 + 1), (ROUND * 6 + 2, ROUND * 6 + 3)]
    _check_all([_noise(110 + i, SMALL_LENS, dict(DEL=nd, INS=ni)) for i, (nd, ni) in enumerate(counts)])


def test_clusters_across_round_edges():
    """Clusters of six whose members are split 3/3, 1/5 and 5/1 across the edges of rounds 1, 2 and 3, and one in the
    input's last rows, each cluster in a partition of its own."""
    rng = np.random.default_rng(120)
    n = ROUND * 5 + 7
    cfg = _noise(120, SMALL_LENS, dict(DEL=n, INS=n - 2))
    for name in ("DEL", "INS"):
        ins = name == "INS"
        for k, row in enumerate((ROUND - 3, 2 * ROUND - 1, 3 * ROUND - 5, len(cfg["sigs"][name]["chrom"]) - 6)):
            pos = (3 + 2 * k) * (1 << 16) + 20000 + rng.integers(0, 200, 6)
            _put(cfg, name, row, _cols(np.zeros(6), pos, 400 + rng.integers(-5, 5, 6), rng.integers(0, 20000, 6), ins,
                                       rng.integers(0, 2, 6) if ins else None))
    _check_all([cfg])


def test_one_round_in_one_partition():
    """Every row of round 1 (DEL) and of round 2 (INS) in one partition: one run of 16 384 pairs, empty runs of that round
    for every other partition, and far more survivors than the filter's shared-memory stage holds."""
    rng = np.random.default_rng(130)
    cfg = _noise(130, SMALL_LENS, dict(DEL=ROUND * 5 + 5, INS=ROUND * 6 + 3))
    _put(cfg, "DEL", ROUND, _block(rng, ROUND, 2 * EDGE + rng.integers(0, 1 << 16, ROUND), False))
    _put(cfg, "INS", 2 * ROUND, _block(rng, ROUND, EDGE + rng.integers(0, 1 << 16, ROUND), True))
    _check_all([cfg])


def test_one_round_over_every_partition():
    """Round 1 of both types spread evenly over both contigs (a row every 2.1 kb): every partition gets a run from it."""
    rng = np.random.default_rng(140)
    cfg = _noise(140, SMALL_LENS, dict(DEL=ROUND * 5 + 2, INS=ROUND * 5 + 9))
    share = (ROUND * SMALL_LENS / SMALL_LENS.sum()).astype(np.int64)
    share[-1] = ROUND - share[:-1].sum()
    for name in ("DEL", "INS"):
        ins = name == "INS"
        parts = []
        for c, k in enumerate(share):
            pos = ((np.arange(k) + 0.5) * (SMALL_LENS[c] - 10) / k).astype(np.int64)
            parts.append(_cols(np.full(k, c), pos, 60 + rng.integers(0, 400, k), rng.integers(0, 20000, k), ins,
                               rng.integers(0, 2, k) if ins else None))
        cols = _cat(parts)
        perm = rng.permutation(ROUND)
        _put(cfg, name, ROUND, {key: None if v is None else v[perm] for key, v in cols.items()})
    _check_all([cfg])
