"""The round-edge inputs of tests/test_gpu_radix_library.py give the key widths they are named for: field maxima -> bits per
field -> total -> LSD rounds -> onesweep passes, by the library's rules."""
import pytest

import radix_cases as R


@pytest.mark.parametrize("name", list(R.ROUND_EDGES))
def test_round_edge_totals(name):
    svtype, maxima, total = R.ROUND_EDGES[name]
    assert set(maxima) == set(R.FIELDS[svtype])
    assert all(0 <= v < (1 << 31) for v in maxima.values())
    assert R.total_bits(svtype, maxima) == total
    if svtype == "TRA":   # c = chr2 * 4 + type: its largest value fits the contig table
        assert maxima["c"] >> 2 < R.n_contigs(svtype, maxima)


def test_round_split():
    assert R.bits_for(0) == 1 and R.bits_for(1) == 1 and R.bits_for(255) == 8 and R.bits_for(256) == 9
    want = {32: ([32], 4), 33: ([33], 5), 64: ([64], 8), 65: ([64, 1], 9), 128: ([64, 64], 16), 129: ([64, 64, 1], 17)}
    for total, (widths, passes) in want.items():
        assert R.rounds(total) == widths and R.onesweep_passes(total) == passes
    assert sorted({t for _, _, t in R.ROUND_EDGES.values()}) == sorted(want)
