"""-m gpu: every cluster-kernel route at its size-class boundaries (tests/cluster_tiers.py).  Each case compares the
records with the oracle, checks CIPOS / CILEN of the exact-boundary alleles against numpy directly, and asserts the route
it was written for through Engine.counters() (kept / members / big / giant / small_path, predicted by a numpy chain split)
or, on a profiled context, through the kernels that ran."""
import functools

import numpy as np
import pytest

import cluster_tiers as ct
from cutesv_b200 import _abi
from cutesv_b200.engine import Engine
from oracle import compare_records, oracle_lib

pytestmark = pytest.mark.gpu

INDEL_MASK = (1 << _abi.CSV_DEL) | (1 << _abi.CSV_INS)


@functools.lru_cache(maxsize=None)
def _layout():
    return ct.boundary_layout(seed=ct.GPU_LAYOUT_SEED)


@functools.lru_cache(maxsize=None)
def _ref(keep, mask):
    cfg = _layout()
    p = _abi.default_params(remain_reads_ratio=keep, **cfg["params"])
    return p, oracle_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"], type_mask=mask, n_threads=8)


def _engine(monkeypatch, env, cfg, p):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    return Engine(0, params=p, contig_lens=cfg["lens"])


def _types(mask):
    return tuple(t for i, t in enumerate(_abi.TYPE_NAMES) if mask >> i & 1)


def _check(eng, cfg, p, ref, mask=0x1F, small_path=True, resident=False):
    if resident:   # inputs uploaded once (Engine.upload): the call that can replay a captured CUDA graph
        eng.cluster_device(mask)
        got = eng.fetch()
    else:
        got = eng.cluster(cfg["sigs"], cfg["reads"], type_mask=mask)
    d = compare_records.diff_records(ref, got)
    assert not d, "\n".join(d[:5])
    errs = ct.allele_cipos_errors(dict(cfg, alleles=[a for a in cfg["alleles"] if a["type"] in _types(mask)]), got)
    assert not errs, "\n".join(errs[:5])
    assert ct.counters_view(eng.counters()) == ct.expected_counters(cfg, p, _types(mask), small_path)
    return got


ROUTES = {
    "default": ({}, dict()),            # then three device-resident calls
    "graphs_off": ({"CUTESV_B200_GRAPHS": "0"}, dict()),
    "lanes_off": ({}, dict(lanes=False)),
    "indel_only_pdl": ({}, dict(mask=INDEL_MASK)),
    "indel_only_pdl_off": ({"CUTESV_B200_PDL": "0"}, dict(mask=INDEL_MASK)),
    "small_path_off": ({"CUTESV_B200_SMALL_PATH": "0"}, dict(small_path=False)),
    "records_off": ({"CUTESV_B200_RECORDS": "0"}, dict()),          # gather mode
    "remain_0.6": ({}, dict(keep=0.6, small_path=False)),            # KIND 4 / 5
    "small_chain": ({"CUTESV_B200_SMALL_CHAIN": "1"}, dict()),       # DUP / INV / TRA chained sorts
}


@pytest.mark.parametrize("route", list(ROUTES))
def test_route(monkeypatch, route):
    env, o = ROUTES[route]
    cfg = _layout()
    mask = o.get("mask", 0x1F)
    p, ref = _ref(o.get("keep", 1.0), mask)
    eng = _engine(monkeypatch, env, cfg, p)
    try:
        if o.get("lanes") is False:
            eng.set_lanes(False)
        _check(eng, cfg, p, ref, mask, o.get("small_path", True))
        if route == "default":   # device-resident inputs, three calls: the second captures a graph, the third replays it
            eng.upload(cfg["sigs"], cfg["reads"])
            for i in range(3):
                before = eng.graph_replays()
                _check(eng, cfg, p, ref, mask, resident=True)
            assert eng.graph_replays() > before, "the third call replays the captured graph"
    finally:
        eng.close()


@pytest.mark.parametrize("route", ["default", "small_path_off", "small_chain"])
def test_kernels_of_route(monkeypatch, route):
    """Profiled context (graphs and the side-stream fork are off there): the register kernel runs exactly when the small
    path is on; k_gather_keys only on the chained-sorts route; the CTA kernel for the > 128-member clusters."""
    env, o = ROUTES[route]
    cfg = _layout()
    p, ref = _ref(1.0, 0x1F)
    eng = _engine(monkeypatch, env, cfg, p)
    try:
        eng.set_profiling(True)
        _check(eng, cfg, p, ref, small_path=o.get("small_path", True))
        names = list(eng.kernel_times())
    finally:
        eng.close()
    has = lambda s: any(s in k for k in names)   # noqa: E731
    small = o.get("small_path", True)
    assert has("k_cluster_small<DEL>") == small and has("k_cluster_small<INS>") == small, names
    assert has("k_gather_keys") == (route == "small_chain"), names
    assert has("k_cluster_block") and has("k_cluster_warp"), names


@pytest.mark.parametrize("ms", [2016, 2017])
def test_min_support_head_mask_limit(monkeypatch, ms):
    """2016 is the last min_support of the bit-mask head test (k_select_heads), 2017 the first of the generic
    k_select<HeadPred> (profiled context: the kernel names show which one ran)."""
    cfg = ct.boundary_layout(seed=ms, types=("DEL", "INS", "DUP"), sizes=(ms - 1, ms, 2100, 2500), min_support=ms, tiers=())
    p = _abi.default_params(**cfg["params"])
    ref = oracle_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"], n_threads=8)
    eng = _engine(monkeypatch, {}, cfg, p)
    try:
        eng.set_profiling(True)
        _check(eng, cfg, p, ref)
        assert eng.counters()["giant"]["DEL"] >= 3
        names = list(eng.kernel_times())
    finally:
        eng.close()
    generic = ms > 2016
    assert any("k_select_heads" in k for k in names) != generic, names
    assert any("k_select<HeadPred>" in k for k in names) == generic, names


def _with_background(layout_cfg, n_noise, seed):
    """Sparse INS / DEL noise on the part of contig 0 after the planted clusters (so no planted allele changes), from
    50 000 reads of 15 kb that are added to the reads table; each noise signature lies inside its read."""
    rng = np.random.default_rng(seed)
    cfg = dict(layout_cfg)
    L0 = int(cfg["lens"][0])
    lo = int(cfg["sigs"]["DEL"]["a"].max()) + 50000
    n_reads = 50000
    r0 = int(cfg["reads"]["read_id"].max()) + 1
    r_start = rng.integers(lo, L0 - 20000, n_reads)
    cfg["reads"] = {k: np.concatenate([v, extra]).astype(v.dtype) for (k, v), extra in zip(
        cfg["reads"].items(), (np.zeros(n_reads), r_start, r_start + 15000, r0 + np.arange(n_reads), np.ones(n_reads)))}
    sigs = {}
    for t, cols in cfg["sigs"].items():
        k = rng.integers(0, n_reads, n_noise)
        pos = r_start[k] + rng.integers(100, 14000, n_noise)
        ln = 60 + rng.integers(0, 400, n_noise)
        rid = r0 + k
        a = 2 * pos if t == "INS" else pos
        extra = dict(chrom=np.zeros(n_noise, np.int32), a=a.astype(np.int32), b=ln.astype(np.int32), read_id=rid.astype(np.int32),
                     c=ln.astype(np.int32) if t == "INS" else None)
        sigs[t] = {k: (None if cols[k] is None else np.concatenate([cols[k], extra[k]])) for k in cols}
    cfg["sigs"] = sigs
    return cfg


@pytest.mark.parametrize("small_path", [True, False])
def test_partitioned_front_end(monkeypatch, small_path):
    """The INS / DEL boundary clusters in a sparse background of 70 000 signatures per type: the density filter runs
    (domain < input) and k_select_heads gathers member records (list mode)."""
    L = ct.Layout(5, contig_len=120_000_000)
    for t in ("DEL", "INS"):
        for m in (10,) + ct.BOUNDARY_SIZES[:-1]:
            L.cluster(t, m)
        L.cluster(t, 33, dup=1)
        L.cluster(t, 129, shared_read=1)
    for tier in ("small", "warp", "cta"):
        for (n, kind), vs in sorted(ct.tier_vectors(tier).items()):
            if kind == "pos" and vs:
                lv = ct.tier_vectors(tier)[(n, "len")]
                for t in ("DEL", "INS"):
                    L.allele(t, vs[0][0], lv[0][0] if lv else ct.BASE + np.arange(n))
    cfg = _with_background(L.config(), 70000, 5)
    p = _abi.default_params(**cfg["params"])
    ref = oracle_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"], n_threads=8)
    env = {} if small_path else {"CUTESV_B200_SMALL_PATH": "0"}
    eng = _engine(monkeypatch, env, cfg, p)
    try:
        _check(eng, cfg, p, ref, mask=INDEL_MASK, small_path=small_path)
        dom = eng.counters()["domain"]
        for t in ("DEL", "INS"):
            assert 0 < dom[t] < len(cfg["sigs"][t]["a"]), (t, dom[t])
    finally:
        eng.close()


@pytest.mark.parametrize("t", ["DUP", "INV"])
@pytest.mark.parametrize("run", [2048, 2049])
def test_equal_primary_keys(monkeypatch, t, run):
    """A run of `run` equal primary keys ((chr, a) for DUP, (chr, strand, a) for INV): up to RUN_MAX = 2048 the run is
    ranked in place, one more takes the chained sorts (k_gather_keys)."""
    L = ct.Layout(run)
    base = L._base(100)
    rid = L._rids(run, base)
    b = base + 3000 + L.rng.integers(0, 60, run)
    L._add(t, np.zeros(run), np.full(run, base), b, rid, np.ones(run) if t == "INV" else None)
    L.cluster(t, 40)
    cfg = L.config()
    p = _abi.default_params(**cfg["params"])
    mask = 1 << _abi.TYPE_IDS[t]
    ref = oracle_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"], type_mask=mask, n_threads=8)
    eng = _engine(monkeypatch, {}, cfg, p)
    try:
        eng.set_profiling(True)
        _check(eng, cfg, p, ref, mask=mask)
        names = list(eng.kernel_times())
    finally:
        eng.close()
    assert any("k_gather_keys" in k for k in names) == (run > 2048), names


def test_pow_table_grow_and_rerun(monkeypatch):
    """One DEL allele of 70 000 distinct reads: more than the initial n ** 0.5 table (65 536 entries), so the first call
    sets ST_POW_TABLE, grows the table and reruns; the second call on the same engine needs no rerun."""
    n = 70000
    L = ct.Layout(70)
    base = L._base(200)
    rid = L._rids(n, base)
    L._add("DEL", np.zeros(n), base + L.rng.integers(0, 150, n), 500 + L.rng.integers(0, 10, n), rid)
    L.cluster("DEL", 50)
    cfg = L.config()
    p = _abi.default_params(**cfg["params"])
    ref = oracle_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"], n_threads=8)
    assert int(ref[0]["support"].max()) == n
    eng = _engine(monkeypatch, {}, cfg, p)
    try:
        l0 = eng.launch_count()
        _check(eng, cfg, p, ref, mask=0x1F)
        l1 = eng.launch_count()
        _check(eng, cfg, p, ref, mask=0x1F)
        l2 = eng.launch_count()
    finally:
        eng.close()
    assert l1 - l0 == 2 * (l2 - l1), "the first call runs the pipeline twice, the second once"


def test_sorted_domain_tile_edges(monkeypatch):
    """Density filter off (every signature in the sorted domain, so a signature's sorted index follows from the layout):
    k_select_heads works on tiles of SEL_TILE = 2048 sorted signatures.  One head at sorted index 2047 (a 40-member
    cluster across the first edge), one min_support cluster whose last member is the last of the second tile, and one
    that crosses the third edge by one member; singletons (never kept) fill the gaps."""
    ms, tile = 10, 2048
    groups = [1] * (tile - 1) + [40]
    groups += [1] * (2 * tile - ms - sum(groups)) + [ms]
    groups += [1] * (3 * tile - ms + 1 - sum(groups)) + [ms] + [1] * 50
    heads = np.cumsum([0] + groups[:-1])
    assert heads[tile - 1] == tile - 1 and groups[tile - 1] == 40
    assert (2 * tile - ms) in heads and (3 * tile - ms + 1) in heads
    rng = np.random.default_rng(17)
    n = sum(groups)
    pos = np.repeat(10000 + 1000 * np.arange(len(groups)), groups) + np.concatenate([rng.integers(0, 40, g) for g in groups])
    ln = 300 + rng.integers(-10, 10, n)
    rid = np.arange(n, dtype=np.int32)
    sigs = dict(DEL=dict(chrom=np.zeros(n, np.int32), a=pos.astype(np.int32), b=ln.astype(np.int32), read_id=rid, c=None),
                INS=dict(chrom=np.zeros(n, np.int32), a=(2 * pos).astype(np.int32), b=ln.astype(np.int32), read_id=rid,
                         c=ln.astype(np.int32)))
    reads = dict(chrom=np.zeros(n, np.int32), start=(pos - 5000).astype(np.int32), end=(pos + 8000).astype(np.int32), read_id=rid,
                 is_primary=np.ones(n, np.uint8))
    cfg = dict(lens=np.array([int(pos.max()) + 100000], np.int64), sigs=sigs, reads=reads, params=dict(ct.PARAMS, min_support=ms),
               alleles=[])
    p = _abi.default_params(**cfg["params"])
    ref = oracle_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"], n_threads=8)
    assert len(ref[0]) >= 6
    eng = _engine(monkeypatch, {"CUTESV_B200_NO_PREFILTER": "1"}, cfg, p)
    try:
        _check(eng, cfg, p, ref, mask=INDEL_MASK)
        assert eng.counters()["kept"]["DEL"] == 3
    finally:
        eng.close()
