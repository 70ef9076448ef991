"""-m gpu: the INS / DEL back-end routes at their edges.  k_select_heads sorts the kept clusters by size while it gathers
their member records: <= 32 members to the register kernel, 33 .. 64 to the end and the larger ones to the front of the
rest list, which k_cluster_warp hands out largest first; clusters of more than 128 members go on to the CTA kernel.
k_select_heads' grid is the CTAs that fit at once, so a domain of more tiles than that makes CTAs take a second tile.
Each case compares the records with the oracle and asserts the route through Engine.counters() (a numpy chain split) and,
on a profiled context, through the kernels that ran."""
import numpy as np
import pytest
import torch

import cluster_tiers as ct
from cutesv_b200 import _abi
from cutesv_b200.engine import Engine
from oracle import compare_records, oracle_lib

pytestmark = pytest.mark.gpu

INDEL_MASK = (1 << _abi.CSV_DEL) | (1 << _abi.CSV_INS)
SEL_TILE = 2048
SEL_CTAS_PER_SM = 8   # k_select_heads: 256 threads and 32 registers per thread, so eight CTAs fill an SM


def _run(monkeypatch, cfg, mask, env=None, profile=False):
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    p = _abi.default_params(**cfg["params"])
    ref = oracle_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"], type_mask=mask, n_threads=8)
    eng = Engine(0, params=p, contig_lens=cfg["lens"])
    try:
        if profile:
            eng.set_profiling(True)
        got = eng.cluster(cfg["sigs"], cfg["reads"], type_mask=mask)
        d = compare_records.diff_records(ref, got)
        assert not d, "\n".join(d[:5])
        types = tuple(t for i, t in enumerate(_abi.TYPE_NAMES) if mask >> i & 1)
        assert ct.counters_view(eng.counters()) == ct.expected_counters(cfg, p, types)
        names = list(eng.kernel_times()) if profile else []
        if not profile:   # the same inputs resident: the second call captures a graph, the third replays it
            eng.upload(cfg["sigs"], cfg["reads"])
            for _ in range(3):
                eng.cluster_device(mask)
                d = compare_records.diff_records(ref, eng.fetch())
                assert not d, "\n".join(d[:5])
            assert eng.graph_replays() > 0
        return eng.counters(), names
    finally:
        eng.close()


def _sizes_layout(sizes, seed):
    L = ct.Layout(seed)
    for t in ("DEL", "INS"):
        for m in sizes:
            L.cluster(t, m)
    return L.config()


@pytest.mark.parametrize("profile", [False, True])
def test_size_edges(monkeypatch, profile):
    """Clusters of 31 .. 33, 63 .. 65 and 127 .. 129 members: register kernel, either end of the rest list, CTA kernel."""
    cfg = _sizes_layout((10, 31, 32, 33, 63, 64, 65, 127, 128, 129), 21)
    ctr, names = _run(monkeypatch, cfg, INDEL_MASK, profile=profile)
    for t in ("DEL", "INS"):
        assert ctr["big"][t] == 1 and ctr["kept"][t] == 10
    if profile:
        for t in ("DEL", "INS"):
            assert "k_cluster_warp<%s,keep-all>" % t in names and "k_cluster_small<%s>" % t in names, names


def test_one_large_among_many_small(monkeypatch):
    """One 128-member cluster among 300 clusters of 33 members (and 60 of 64 and 65): the list holds the 128- and
    65-member clusters at its front and the others at its end."""
    cfg = _sizes_layout((33,) * 150 + (64, 65) * 30 + (128,) + (33,) * 150, 22)
    ctr, _ = _run(monkeypatch, cfg, INDEL_MASK)
    assert ctr["kept"]["DEL"] == ctr["kept"]["INS"] == 361


def test_warp_route_without_small_path(monkeypatch):
    """With the register kernel off, k_select_heads makes no size lists and k_cluster_warp takes every INS / DEL cluster."""
    cfg = _sizes_layout((10, 32, 33, 64, 65, 128, 129), 23)
    p = _abi.default_params(**cfg["params"])
    monkeypatch.setenv("CUTESV_B200_SMALL_PATH", "0")
    ref = oracle_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"], type_mask=INDEL_MASK, n_threads=8)
    eng = Engine(0, params=p, contig_lens=cfg["lens"])
    try:
        eng.set_profiling(True)
        got = eng.cluster(cfg["sigs"], cfg["reads"], type_mask=INDEL_MASK)
        assert not compare_records.diff_records(ref, got)
        assert ct.counters_view(eng.counters()) == ct.expected_counters(cfg, p, ("DEL", "INS"), small_path=False)
        names = list(eng.kernel_times())
    finally:
        eng.close()
    assert any("k_cluster_warp" in k for k in names) and not any("k_cluster_small" in k for k in names), names


@pytest.mark.parametrize("extra_tiles", [0, 1])
def test_select_tiles_around_one_wave(monkeypatch, extra_tiles):
    """A DEL domain (density filter off, so every signature is in it) of exactly one wave of k_select_heads tiles, and of
    one tile more: then one CTA takes a second tile.  The planted clusters of every route sit in the last tiles."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    wave = SEL_CTAS_PER_SM * n_sm
    sizes = (10, 32, 33, 64, 65, 128, 129, 2049)
    planted = sum(sizes)
    n_total = (wave + extra_tiles) * SEL_TILE - 100
    n_noise = n_total - planted
    spacing = 250   # > bias_del: every noise signature is a cluster of one
    first = 10000 + n_noise * spacing + 10000
    L = ct.Layout(24, contig_len=first + 2_000_000, first=first)
    for m in sizes:
        L.cluster("DEL", m)
    cfg = L.config()
    pos = 10000 + spacing * np.arange(n_noise)
    r0 = int(cfg["reads"]["read_id"].max()) + 1
    d = cfg["sigs"]["DEL"]
    noise = dict(chrom=np.zeros(n_noise, np.int32), a=pos.astype(np.int32), b=np.full(n_noise, 300, np.int32),
                 read_id=(r0 + np.arange(n_noise)).astype(np.int32))
    cfg["sigs"] = {"DEL": {k: (None if d[k] is None else np.concatenate([d[k], noise[k]])) for k in d}}
    assert len(cfg["sigs"]["DEL"]["a"]) == n_total
    tiles = (n_total + SEL_TILE - 1) // SEL_TILE
    assert tiles == wave + extra_tiles
    ctr, _ = _run(monkeypatch, cfg, 1 << _abi.CSV_DEL, env={"CUTESV_B200_NO_PREFILTER": "1"})
    assert ctr["big"]["DEL"] == 2 and ctr["giant"]["DEL"] == 1
