"""-m gpu: the 512-thread density filter (k_part_filter) against the oracle at the edges of its layout.

Every thread owns a strip of BP / 512 buckets (32 at W = 22, one at W = 17); at W = 16 (256 buckets) the threads at or
past 256 own none.  A radius rb longer than the strip leaves no strip interior.  One CTA step of the page walk covers four
pages of 2048 pairs, so partitions of 4 * 2048 +- 1 pairs end a step one pair early or late.  Survivors beyond the
shared-memory stage spill, buckets of more than 64 survivors are ordered by a counting sort, listed up to 256 per
partition and found by visiting every bucket past that.  The library picks the partition width W from the genome's
length and the SM count (the widest W <= 22 that still gives about two partitions per SM, at least 16), so the genomes
here are sized from the card's SM count."""
import numpy as np
import pytest
import torch

from cutesv_b200 import _abi
from cutesv_b200.engine import Engine
from test_gpu_partition_filter import PARAMS, _cat, _check, _cols

pytestmark = pytest.mark.gpu

PAGE = 2048
STEP = 4 * PAGE          # pairs per CTA step of the page walk
BKT = 256
N_READS = 20000


def _pad(params):
    p = _abi.default_params(**params)
    return max(p.bias_del, p.bias_ins, p.bias_inv, p.bias_dup, p.bias_tra, p.gt_bias_ins) + 1


def _width(lens, params):
    """The partition width run_indel picks for this genome on this card."""
    total = int(np.sum(np.asarray(lens, np.int64) + _pad(params)))
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    w = 22
    while w > 16 and (total >> w) + 1 < 2 * n_sm:
        w -= 1
    return w


def _lens_for(w, params):
    """Two contigs whose linear length makes the library pick width w."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    total = (2 * n_sm - 8) << 17 if w == 16 else (2 * n_sm + 4) << w
    first = total * 3 // 5
    lens = np.array([first, total - first - 2 * _pad(params)], dtype=np.int64)
    assert _width(lens, params) == w
    return lens


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


def _dataset(seed, lens, n_noise, planted=lambda rng: [], params=PARAMS, noise_contigs=(0, 1)):
    """n_noise rows spread over noise_contigs, plus the rows planted(rng) returns as contig-0 positions; shuffled."""
    rng = np.random.default_rng(seed)
    # INS keys carry 2 * pos: keep the noise below 2^30 bp so that 2 * pos fits int32
    top = np.minimum(lens, (1 << 30) - 1)
    sigs = {}
    for name in ("DEL", "INS"):
        ins = name == "INS"
        ch = rng.choice(np.asarray(noise_contigs), n_noise)
        pos = (rng.random(n_noise) * (top[ch] - 10)).astype(np.int64)
        parts = [_cols(ch, pos, 60 + rng.integers(0, 400, n_noise), rng.integers(0, N_READS, n_noise), ins,
                       rng.integers(0, 2, n_noise) if ins else None)]
        parts += [_rows(rng, 0, p, ins) for p in planted(rng)]
        cols = _cat(parts)
        perm = rng.permutation(len(cols["chrom"]))
        sigs[name] = {k: None if v is None else v[perm] for k, v in cols.items()}
    return dict(lens=lens, sigs=sigs, reads=_reads(rng, lens), params=dict(params))


def _run(*cfgs):
    eng = Engine(0, params=_abi.default_params(**cfgs[0]["params"]), contig_lens=cfgs[0]["lens"])
    try:
        for cfg in cfgs:
            assert _check(eng, cfg) > 0
    finally:
        eng.close()


def _clusters(rng, starts, k=9):
    """k rows within 200 bp of every start: clusters that survive the filter."""
    return [np.int64(s) + rng.integers(0, 200, k) for s in starts]


def test_w16_threads_without_a_strip():
    """W = 16: 256 buckets per partition, so threads 256 .. 511 own no strip (they still load and place pairs);
    clusters at partition starts and ends read the halo."""
    lens = _lens_for(16, PARAMS)
    part = 1 << 16
    starts = [j * part + off for j in range(3, 200, 7) for off in (0, part - 150, part // 2)]
    _run(_dataset(200, lens, 70000, lambda rng: _clusters(rng, starts)))


def test_w17_one_bucket_per_strip_no_interior_strip():
    """W = 17: 512 buckets, one per strip; rb = 2 is longer than the strip, so every strip takes the generic loop."""
    lens = _lens_for(17, PARAMS)
    part = 1 << 17
    starts = [j * part + off for j in range(2, 150, 5) for off in (0, 100, part - 300, 256 * 255)]
    _run(_dataset(210, lens, 80000, lambda rng: _clusters(rng, starts)))


def test_w22_radius_longer_than_the_strip():
    """W = 22: 32 buckets per strip with rb = 63 (bias 4000): no strip is interior, and windows reach two strips away."""
    params = dict(PARAMS, bias_del=4000, bias_ins=4000)
    lens = _lens_for(22, params)
    part = 1 << 22
    starts = [j * part + off for j in range(1, 120, 3) for off in (0, 32 * BKT * 7 - 100, part - 5000)]
    _run(_dataset(220, lens, 70000, lambda rng: [s + rng.integers(0, 16000, 6) for s in starts], params))


def test_partitions_around_a_walk_step():
    """Partitions of STEP - 1, STEP, STEP + 1 and 2 STEP + 1 pairs (and one page + 1) in the first 2^16 bp of their
    partition, the noise in contig 1 only: the CTA's last step ends one pair short of, at, or one pair into four pages.
    They spill the stage."""
    lens = _lens_for(18, PARAMS)
    part = 1 << 18
    sizes = [STEP - 1, STEP, STEP + 1, 2 * STEP + 1, PAGE + 1]
    starts = [(10 + 20 * j) * part for j in range(len(sizes))]
    cfg = _dataset(230, lens, 66000, lambda rng: [s + 512 + rng.integers(0, (1 << 16) - 1024, k) for s, k in zip(starts, sizes)],
                   noise_contigs=(1,))
    _run(cfg)


def test_pileup_spills_the_stage_and_counting_sort():
    """One bucket of 7000 rows (spill, counting sort), and in another partition five buckets of 65 .. 400 rows beside
    small ones: several listed large buckets in one partition."""
    lens = _lens_for(18, PARAMS)
    part = 1 << 18

    def planted(rng):
        out = [40 * part + 4096 + rng.integers(0, BKT, 7000)]
        out += [60 * part + 8192 + BKT * 3 * i + rng.integers(0, BKT, k) for i, k in enumerate((65, 66, 128, 257, 400))]
        out += _clusters(rng, [60 * part + 40000 + 700 * i for i in range(30)], 20)
        return out
    _run(_dataset(240, lens, 70000, planted))


def test_big_bucket_list_overflows():
    """300 consecutive buckets of 70 rows each in one partition, more than the 256 the large-bucket list holds: the CTA
    visits every bucket of the partition instead."""
    lens = _lens_for(18, PARAMS)
    part = 1 << 18

    def planted(rng):
        return [np.concatenate([30 * part + 512 + BKT * i + rng.integers(0, BKT, 70) for i in range(300)])]
    _run(_dataset(250, lens, 70000, planted))


def test_one_engine_repeated_calls():
    """One engine: the same input three times (eager, graph capture, replay), then a larger one with a pile-up and
    partitions around a walk step, then the first again: the fill counters and page table start clean every time."""
    lens = _lens_for(18, PARAMS)
    part = 1 << 18
    a = _dataset(260, lens, 70000, lambda rng: _clusters(rng, [j * part + 77 for j in range(5, 150, 4)]))
    b = _dataset(261, lens, 90000, lambda rng: [40 * part + 4096 + rng.integers(0, BKT, 7000),
                                                90 * part + 512 + rng.integers(0, (1 << 16) - 1024, STEP + 1)])
    _run(a, a, a, b, b, a)
