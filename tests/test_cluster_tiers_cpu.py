"""CPU: the exact-boundary CIPOS vectors (tests/cluster_tiers.py) tell numpy's summation order from wrong ones, the
oracle's std / cal_CIPOS give numpy's answer on them, and the one-thread emulator of the cluster templates equals the
oracle on clusters planted at every size-class boundary."""
import numpy as np
import pytest

import cluster_tiers as ct
import emul_lib
from cutesv_b200 import _abi
from oracle import compare_records, oracle_lib


@pytest.mark.parametrize("tier", list(ct.TIERS))
def test_vectors_defeat_their_mutants(tier):
    tv = ct.tier_vectors(tier)
    covered = set()
    for (n, kind), vs in tv.items():
        for v, beaten in vs:
            assert len(v) == n
            if kind == "len":
                assert all(b > a for a, b in zip(v, v[1:])), "lengths must be distinct and ascending"
            else:
                assert int(np.diff(np.sort(v)).max()) <= ct.POS_MAX_GAP
            want = float(np.std(np.asarray(v, np.int64)))
            assert ct.np_std(v) == want, "the Python restatement must equal np.std bit for bit"
            assert beaten and beaten == ct.defeated(v)
            k = ct.cal_cipos(want, n)
            for m in beaten:
                assert ct.cal_cipos(ct.np_std(v, m), n) != k, m
            covered |= beaten
    missing = ct.TIER_NEEDS[tier] - covered
    assert not missing, "%s: no vector defeats %s" % (tier, sorted(missing))


def test_planted_alleles_cover_every_tier():
    """The vectors keep what they were chosen for where the GPU sees them: on the absolute positions and lengths of the
    route tests' layout, in allele order."""
    cov = ct.planted_coverage(ct.boundary_layout(seed=ct.GPU_LAYOUT_SEED))
    for tier, need in ct.TIER_NEEDS.items():
        assert need <= cov[tier], "%s: no planted allele defeats %s" % (tier, sorted(need - cov[tier]))


@pytest.mark.parametrize("tier", list(ct.TIERS))
def test_oracle_std_and_cal_cipos(tier):
    for (n, kind), vs in ct.tier_vectors(tier).items():
        for v, _ in vs:
            for base in (0, 5000, 1 << 20):
                x = np.asarray(v, np.int64) + base
                want = float(np.std(x))
                got = oracle_lib.np_std(x.astype(np.int32))
                assert got == want, (n, kind, base)
                assert oracle_lib.lib().csvo_cal_cipos(got, n) == ct.cal_cipos(want, n)


def test_restatement_on_random_vectors():
    rng = np.random.default_rng(5)
    for n in (1, 7, 8, 9, 127, 128, 129, 136, 255, 1000, 2049, 4500):
        v = rng.integers(-10 ** 6, 10 ** 6, n)
        assert ct.np_std(v) == float(np.std(v)), n


def test_chain_split_counts_planted_sizes():
    cfg = ct.boundary_layout(tiers=())
    p = _abi.default_params(**cfg["params"])
    exp = ct.expected_counters(cfg, p)
    sizes = (p.min_support,) + ct.BOUNDARY_SIZES
    for t in ct.ALL_TYPES:
        m, dom = ct.chain_sizes(t, cfg["sigs"][t], cfg["lens"], p)
        planted = sorted(sizes + ((32,) if t not in ("DEL", "INS") else (33,)) + (129,) +
                         ((2048,) if t not in ("DEL", "INS") else (2049,)) +
                         ((20, 20, 100, 100, 500, 500, 2100, 2100) if t == "INS" else ()))
        assert sorted(m.tolist()) == planted, t
    # DEL: > 128 members: 129, 2047, 2048, 2049, 4500 and the straddling 129 and 2049; > 2048: 2049, 4500, 2049
    assert exp["big"]["DEL"] == 7 and exp["giant"]["DEL"] == 3
    assert exp["small_path"] == 2 * 3 + 2   # min_support, 31, 32 for INS and DEL; the two 20-member INS clusters
    assert exp["giant"]["DUP"] == 2     # 2049 and 4500; 2049 with one exact duplicate is a 2048-member cluster


@pytest.mark.parametrize("keep", [1.0, 0.6])
def test_emulator_equals_oracle_on_boundary_layout(keep):
    cfg = ct.boundary_layout(seed=3, tiers=("small", "warp", "cta"))
    p = _abi.default_params(remain_reads_ratio=keep, **cfg["params"])
    ref = oracle_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"], n_threads=8)
    got = emul_lib.cluster(p, cfg["lens"], cfg["sigs"], cfg["reads"])
    d = compare_records.diff_records(ref, got)
    assert not d, "\n".join(d[:5])
    errs = ct.allele_cipos_errors(cfg, ref)
    assert not errs, "\n".join(errs[:5])
