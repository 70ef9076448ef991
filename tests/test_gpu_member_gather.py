"""-m gpu: k_select_heads' member gather at its tile edges.  In record mode every 2048-element tile gathers the member
records of the kept clusters that lie in it, wherever their heads are, and sizes the clusters headed in it from its link
mask.  DEL and INS domains are built with the density filter off, so every signature is in the domain and its sorted
position is known: kept clusters start on a tile's last position, span three tiles and end on a tile's last position,
and a run of min_support - 1 signatures crosses a tile edge.  The domain covers two contigs (DEL takes a member's position
from its key in a tile that lies on one contig, and loads it in the tile that crosses the contig end).  Records are compared with the oracle, and the kept, member,
big and register-kernel counts with a numpy chain split of the planted runs."""
import numpy as np
import pytest

import cluster_tiers as ct
from cutesv_b200 import _abi
from cutesv_b200.engine import Engine
from oracle import compare_records, oracle_lib

pytestmark = pytest.mark.gpu

TILE = 2048
NEED = ct.PARAMS["min_support"]
STEP = 10      # bp between the signatures of a run: chained under both biases
GAP = 1000     # bp between runs: never chained


def _domain(t, runs, n, seed, split):
    """n signatures of type t in sorted order: the planted runs (start, length) in sorted positions, every other
    signature a cluster of one; one read per signature.  Sorted positions from `split` on lie on a second contig, so that
    one tile crosses a contig end and the later ones lie on a contig whose linear offset is not 0.  Returns the config and
    the run lengths in sorted order."""
    rng = np.random.default_rng(seed)
    size = np.ones(n, np.int64)    # run length at each run start, 0 inside a run
    for s, m in runs:
        assert size[s:s + m].min() == 1 and size[s:s + m].sum() == m
        size[s] = m
        size[s + 1:s + m] = 0
    gap = np.where(size > 0, GAP, STEP)
    gap[0] = 0
    assert size[split] > 0
    gap[split] = 0
    chrom = (np.arange(n) >= split).astype(np.int32)
    pos = np.cumsum(gap)
    pos = 20000 + pos - np.where(chrom == 1, pos[split], 0)
    ln = 300 + rng.integers(-20, 20, n)
    rid = np.arange(n, dtype=np.int32)
    if t == "DEL":
        cols = dict(chrom=chrom, a=pos.astype(np.int32), b=ln.astype(np.int32), read_id=rid, c=None)
    else:
        cols = dict(chrom=chrom, a=(2 * pos + rng.integers(0, 2, n)).astype(np.int32), b=ln.astype(np.int32),
                    read_id=rid, c=ln.astype(np.int32))
    perm = rng.permutation(n)
    cols = {k: (None if v is None else v[perm]) for k, v in cols.items()}
    lens = np.array([pos[:split].max(), pos[split:].max()], np.int64) + 100000
    reads = dict(chrom=chrom, start=np.maximum(pos - 6000, 0).astype(np.int32), end=(pos + 6000).astype(np.int32), read_id=rid,
                 is_primary=np.ones(n, np.uint8))
    cfg = dict(lens=lens, sigs={t: cols}, reads=reads, params=dict(ct.PARAMS))
    return cfg, size[size > 0]


# (start, length) in sorted positions
EDGE_RUNS = (
    (TILE - 1, 40),                   # a kept cluster that starts on tile 0's last position
    (2 * TILE - 7, TILE + 20),        # one that spans tiles 1, 2 and 3 (more than 2048 members: global scratch)
    (4 * TILE - 30, 30),              # one that ends on tile 3's last position
    (5 * TILE - 4, NEED - 1),         # a run one short of min_support across the edge of tiles 4 and 5
    (6 * TILE - NEED, NEED),          # exactly min_support, ending on a tile edge
    (6 * TILE + 100, 65),             # size-list edges inside a tile
    (6 * TILE + 300, 64),
    (6 * TILE + 500, 33),
    (6 * TILE + 700, 32),
    (7 * TILE - 20, 129),             # 129 members over the edge of tiles 6 and 7
)


@pytest.mark.parametrize("t", ["DEL", "INS"])
def test_clusters_on_tile_edges(monkeypatch, t):
    monkeypatch.setenv("CUTESV_B200_NO_PREFILTER", "1")
    n = 8 * TILE + 333
    cfg, sizes = _domain(t, EDGE_RUNS, n, 31 if t == "DEL" else 32, 3 * TILE + 1000)
    kept = sizes[sizes >= NEED]
    want = dict(kept=len(kept), members=int(kept.sum()), big=int((kept > ct.WARP_M).sum()), giant=int((kept > ct.BLOCK_M).sum()),
                small=int((kept <= ct.SMALL_M).sum()))
    assert want == dict(kept=9, members=40 + TILE + 20 + 30 + NEED + 65 + 64 + 33 + 32 + 129, big=2, giant=1, small=3)
    mask = 1 << _abi.TYPE_IDS[t]
    p = _abi.default_params(**cfg["params"])
    ref = oracle_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"], type_mask=mask, n_threads=8)
    eng = Engine(0, params=p, contig_lens=cfg["lens"])
    try:
        got = eng.cluster(cfg["sigs"], cfg["reads"], type_mask=mask)
        d = compare_records.diff_records(ref, got)
        assert not d, "\n".join(d[:5])
        c = eng.counters()
        assert dict(kept=c["kept"][t], members=c["members"][t], big=c["big"][t], giant=c["giant"][t],
                    small=c["small_path"]) == want
        assert ct.counters_view(c) == ct.expected_counters(cfg, p, (t,))
        eng.upload(cfg["sigs"], cfg["reads"])   # resident inputs: a captured graph and its replays give the same records
        for _ in range(3):
            eng.cluster_device(mask)
            d = compare_records.diff_records(ref, eng.fetch())
            assert not d, "\n".join(d[:5])
    finally:
        eng.close()
