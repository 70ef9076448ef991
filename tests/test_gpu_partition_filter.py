"""-m gpu: the partitioned INS/DEL front end (density filter per genome partition in shared memory) against the oracle.

The front end is taken when the density filter applies (32-bit keys, min_support >= 3, sparse input, >= 65536 signatures
of the type).  Partitions are 2^W bp of the linear coordinate with W <= 22, so every multiple of 2^22 in contig 0 (whose
linear offset is 0) is a partition edge whatever W the library picks."""
import numpy as np
import pytest

from cutesv_b200 import _abi, shard
from cutesv_b200.engine import Engine
from oracle import compare_records, oracle_lib

pytestmark = pytest.mark.gpu

EDGE = 1 << 22
BKT_SHIFT = 8
PARAMS = dict(min_support=5, bias_del=100, bias_ins=100, ratio_del=0.3, ratio_ins=0.3, genotype=1)
LENS = np.array([5 * EDGE + 12345, 3 * EDGE + 777, 2 * EDGE + 5], dtype=np.int64)


def _cols(chrom, pos, ln, rid, ins, half=None):
    chrom = np.asarray(chrom, np.int32)
    pos = np.asarray(pos, np.int64)
    ln = np.asarray(ln, np.int32)
    if not ins:
        return dict(chrom=chrom, a=pos.astype(np.int32), b=ln, read_id=np.asarray(rid, np.int32), c=None)
    a = 2 * pos + (np.asarray(half, np.int64) if half is not None else 0)   # odd a: an x.5 position
    return dict(chrom=chrom, a=a.astype(np.int32), b=ln, read_id=np.asarray(rid, np.int32), c=ln.copy())


def _cat(parts):
    out = {}
    for k in ("chrom", "a", "b", "read_id", "c"):
        vs = [p[k] for p in parts]
        out[k] = None if vs[0] is None else np.concatenate(vs)
    return out


def _dataset(seed, pileup=0):
    """Sparse noise over three contigs (enough rows to take the filter) plus clusters planted across partition edges."""
    rng = np.random.default_rng(seed)
    n_noise = 110000
    n_reads = 20000
    weights = LENS / LENS.sum()
    reads_chrom = rng.choice(len(LENS), n_reads, p=weights).astype(np.int32)
    r_start = (rng.random(n_reads) * (LENS[reads_chrom] - 20000)).astype(np.int64)
    reads = dict(chrom=reads_chrom, start=r_start.astype(np.int32), end=(r_start + 15000).astype(np.int32),
                 read_id=np.arange(n_reads, dtype=np.int32), is_primary=np.ones(n_reads, np.uint8))
    sigs = {}
    for name in ("DEL", "INS"):
        ins = name == "INS"
        parts = []
        ch = rng.choice(len(LENS), n_noise, p=weights)
        pos = (rng.random(n_noise) * (LENS[ch] - 10)).astype(np.int64)
        parts.append(_cols(ch, pos, 60 + rng.integers(0, 400, n_noise), rng.integers(0, n_reads, n_noise), ins,
                           rng.integers(0, 2, n_noise) if ins else None))
        rid = iter(rng.permutation(n_reads))
        for e in range(1, 5):
            edge = e * EDGE
            # a cluster across the edge
            k = 8
            p = edge - 150 + rng.integers(0, 300, k)
            parts.append(_cols(np.zeros(k), p, 300 + rng.integers(-5, 5, k), [next(rid) for _ in range(k)], ins,
                               np.ones(k, np.int64) if ins else None))
            # three members on each side of the edge: neither side's buckets alone reach min_support (the halo decides)
            p = np.array([edge - 40, edge - 30, edge - 20, edge + 10, edge + 20, edge + 30]) + 1000 * (e % 2)
            parts.append(_cols(np.zeros(6), p, 500 + rng.integers(-3, 3, 6), [next(rid) for _ in range(6)], ins,
                               np.array([1, 0, 1, 0, 1, 1]) if ins else None))
            # x.5 INS positions at the last base before the edge
            p = np.full(5, edge - 1)
            parts.append(_cols(np.zeros(5), p, 700 + rng.integers(-2, 2, 5), [next(rid) for _ in range(5)], ins,
                               np.ones(5, np.int64) if ins else None))
        if pileup:
            # one 256-bp bucket with more survivors than a partition's shared-memory stage holds
            p = 3 * EDGE + 4096 + rng.integers(0, 256, pileup)
            parts.append(_cols(np.zeros(pileup), p, np.where(rng.random(pileup) < 0.5, 300, 900) + rng.integers(-20, 20, pileup),
                               rng.integers(0, n_reads, pileup), ins, rng.integers(0, 2, pileup) if ins else None))
        sigs[name] = _cat(parts)
    return dict(lens=LENS, sigs=sigs, reads=reads, params=dict(PARAMS))


def _filter_survivors(p, lens, cols, ins, owned=None):
    """Survivor count of the density filter's rule: +-rb 256-bp buckets of the linear key hold >= min_support."""
    ms = p.min_support
    bias = p.bias_ins if ins else p.bias_del
    pad = max(p.bias_del, p.bias_ins, p.bias_inv, p.bias_dup, p.bias_tra, p.gt_bias_ins) + 1
    mine = np.ones(len(lens), bool) if owned is None else np.asarray(owned, bool)
    step = np.where(mine, lens + pad, 0)
    off = np.concatenate([[0], np.cumsum(step)])
    total = int(off[-1])
    radius = min((ms - 1) * bias, 1 << 24)
    rb = (radius + (1 << BKT_SHIFT) - 1) >> BKT_SHIFT
    n = len(cols["chrom"])
    lam = n * (2.0 * radius + 2.0 * (1 << BKT_SHIFT)) / total
    assert n >= 65536 and lam < 0.8 * ms, "the input must take the density filter"
    pos = cols["a"].astype(np.int64) >> (1 if ins else 0)
    key = off[cols["chrom"]] + pos
    cnt = np.bincount(key >> BKT_SHIFT, minlength=(total >> BKT_SHIFT) + 1).astype(np.int64)
    pre = np.concatenate([[0], np.cumsum(cnt)])
    b = np.arange(len(cnt))
    win = pre[np.minimum(b + rb + 1, len(cnt))] - pre[np.maximum(b - rb, 0)]
    return int(cnt[win >= ms].sum())


def _check(eng, cfg, owned=None):
    p = _abi.default_params(**cfg["params"])
    got = eng.cluster(cfg["sigs"], cfg["reads"])
    ref = oracle_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"], n_threads=8)
    d = compare_records.diff_records(ref, got)
    assert not d, "\n".join(d[:5])
    dom = eng.counters()["domain"]
    for name in ("DEL", "INS"):
        assert dom[name] == _filter_survivors(p, cfg["lens"], cfg["sigs"][name], name == "INS", owned), name
    return len(ref[0])


def test_partition_edges_and_repeated_calls():
    """Clusters across partition edges (DEL, INS, INS x.5), three calls on one engine (graph capture and replay), then a
    different input on the same engine (stale buffers of the larger call)."""
    a = _dataset(1, pileup=7000)
    b = _dataset(2)
    eng = Engine(0, params=_abi.default_params(**a["params"]), contig_lens=a["lens"])
    try:
        for _ in range(3):
            assert _check(eng, a) > 0
        for _ in range(3):
            assert _check(eng, b) > 0
    finally:
        eng.close()


def test_pileup_spills_the_stage():
    """A single bucket of 7000 survivors, far more than the shared-memory stage of its partition."""
    cfg = _dataset(3, pileup=7000)
    eng = Engine(0, params=_abi.default_params(**cfg["params"]), contig_lens=cfg["lens"])
    try:
        assert _check(eng, cfg) > 0
    finally:
        eng.close()


def test_sharded_contigs():
    """csv_set_shard: contigs 0 and 2 only; the linear coordinate (and the partitions) cover the owned contigs alone."""
    cfg = _dataset(4)
    owner = np.array([0, 1, 0])
    sigs, reads, _ = shard.shard_inputs(cfg["sigs"], cfg["reads"], owner, 0)
    sub = dict(lens=cfg["lens"], sigs=sigs, reads=reads, params=cfg["params"])
    eng = Engine(0, params=_abi.default_params(**cfg["params"]), contig_lens=cfg["lens"])
    try:
        eng.set_shard(shard.owned_mask(owner, 0))
        for _ in range(3):
            assert _check(eng, sub, owned=owner == 0) > 0
    finally:
        eng.close()
