"""-m gpu: the grouping rounds of k_part_scatter against the oracle.

k_part_scatter groups 8192 rows per round with 16 B loads, so row counts that are not multiples of 4, of a round or of a
16 384-row chunk leave partial loads at the end of the input.  A genome of 34 Mb makes the library pick the narrowest
partitions on a 132-SM H100 (2^16 bp).  The filter is taken for 65 536 to about 100 000 rows of a type on that genome."""
import numpy as np
import pytest

from cutesv_b200 import _abi
from cutesv_b200.engine import Engine
from test_gpu_partition_filter import PARAMS, _cat, _check, _cols

pytestmark = pytest.mark.gpu

SMALL_LENS = np.array([20_000_000, 14_000_003], dtype=np.int64)


def _noise(seed, lens, n_by_type):
    """Sparse signatures over `lens` (n_by_type[name] rows each) plus one dense stretch of planted clusters in contig 0."""
    rng = np.random.default_rng(seed)
    n_reads = 20000
    weights = lens / lens.sum()
    reads_chrom = rng.choice(len(lens), n_reads, p=weights).astype(np.int32)
    r_start = (rng.random(n_reads) * (lens[reads_chrom] - 20000)).astype(np.int64)
    reads = dict(chrom=reads_chrom, start=r_start.astype(np.int32), end=(r_start + 15000).astype(np.int32),
                 read_id=np.arange(n_reads, dtype=np.int32), is_primary=np.ones(n_reads, np.uint8))
    sigs = {}
    for name, n in n_by_type.items():
        ins = name == "INS"
        n_cl = 40 * 6
        ch = rng.choice(len(lens), n - n_cl, p=weights)
        pos = (rng.random(n - n_cl) * (lens[ch] - 10)).astype(np.int64)
        parts = [_cols(ch, pos, 60 + rng.integers(0, 400, n - n_cl), rng.integers(0, n_reads, n - n_cl), ins,
                       rng.integers(0, 2, n - n_cl) if ins else None)]
        for k in range(40):   # 40 clusters of 6 a few kb apart
            p = 1_000_000 + 5000 * k + rng.integers(0, 200, 6)
            parts.append(_cols(np.zeros(6), p, 400 + rng.integers(-5, 5, 6), rng.integers(0, n_reads, 6), ins,
                               rng.integers(0, 2, 6) if ins else None))
        cols = _cat(parts)
        perm = rng.permutation(n)   # the rows of a chunk spread over every partition
        sigs[name] = {k: None if v is None else v[perm] for k, v in cols.items()}
    return dict(lens=lens, sigs=sigs, reads=reads, params=dict(PARAMS))


def test_row_counts_off_the_load_width():
    """Row counts that end inside a 4-row load, inside a round and inside a chunk, then exact multiples."""
    counts = [(70001, 90003), (16384 * 5 + 8192 + 3, 16384 * 4 + 1), (16384 * 6, 8192 * 9)]
    for i, (nd, ni) in enumerate(counts):
        cfg = _noise(10 + i, SMALL_LENS, dict(DEL=nd, INS=ni))
        eng = Engine(0, params=_abi.default_params(**cfg["params"]), contig_lens=cfg["lens"])
        try:
            assert _check(eng, cfg) > 0
        finally:
            eng.close()


def test_one_engine_inputs_of_different_sizes():
    """Larger, smaller and larger again on one engine: scratch sized by an earlier call, CUDA-graph capture and replay."""
    cfgs = [_noise(20 + i, SMALL_LENS, dict(DEL=n, INS=n + 5)) for i, n in enumerate((98001, 66001, 98001))]
    eng = Engine(0, params=_abi.default_params(**cfgs[0]["params"]), contig_lens=SMALL_LENS)
    try:
        for cfg in cfgs:
            for _ in range(2):
                assert _check(eng, cfg) > 0
    finally:
        eng.close()
