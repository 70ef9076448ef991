"""-include_bed region assignment: grouping the task windows by contig gives every task exactly the region list, in the
same order, that the reference's scan of every task for every region gives (cuteSV_genotype.py:704-726)."""
import numpy as np
import pytest

from cutesv_b200 import cli


def reference_load_bed(bed_file, tasks):
    """Literal restatement of the reference's loop."""
    regions = {}
    with open(bed_file) as f:
        for line in f:
            s = line.strip().split("\t")
            regions.setdefault(s[0], []).append((int(s[1]) - 1000, int(s[2]) + 1000))
    out = [[] for _ in tasks]
    for chrom in regions:
        regions[chrom].sort()
        for item in regions[chrom]:
            for i, t in enumerate(tasks):
                if chrom == t[0] and ((t[1] <= item[0] and t[2] > item[0]) or item[0] <= t[1] < item[1]):
                    out[i].append(item)
    return out


@pytest.mark.parametrize("seed", range(12))
def test_load_bed_equals_reference_loop(tmp_path, seed):
    rng = np.random.default_rng(seed)
    n_contigs = int(rng.integers(1, 40))
    names = ["ctg%d" % k for k in rng.permutation(n_contigs)]
    lens = {n: int(rng.integers(1000, 300000)) for n in names}
    stats = [(n, int(rng.integers(0, 5000))) for n in names]
    tasks, _ = cli.task_windows(stats, lens.get, int(rng.integers(1, 17)), int(rng.choice([5000, 20000, 100000])))
    rows = []
    for _ in range(int(rng.integers(0, 200))):
        c = names[int(rng.integers(0, n_contigs))] if rng.random() < 0.9 else "absent"
        a = int(rng.integers(0, 310000))
        rows.append("%s\t%d\t%d\n" % (c, a, a + int(rng.integers(0, 30000))))
    if rows and rng.random() < 0.5:   # repeated rows
        rows += rows[:int(rng.integers(1, len(rows) + 1))]
    bed = tmp_path / "r.bed"
    bed.write_text("".join(rows))
    got = cli.load_bed(str(bed), tasks)
    assert got == reference_load_bed(str(bed), tasks)


def test_load_bed_none():
    assert cli.load_bed(None, [["a", 0, 10]]) is None
