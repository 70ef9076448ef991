"""Helpers of the SA:Z text tests: adversarial and seeded SA values, a BAM whose records carry them (the native decoder's host
reduction is the reference), and the (text, text_off) arrays csv_reduce_sa_device takes."""
import numpy as np

import bam_writer
from cutesv_b200 import bamio

CONTIGS = [("chr1", 300000), ("chr10", 200000), ("chr2", 250000), ("chrX", 100000), ("c", 5000)]
NAMES = sorted(n for n, _ in CONTIGS)
CHROM_ID = {n: i for i, n in enumerate(NAMES)}


class Rec(object):
    """The fields bam_writer reads from a record."""

    def __init__(self, i, sa):
        self.query_name = "r%d" % i
        self.cigartuples = [(0, 100)]
        self.query_sequence = None
        self.query_length = 100
        self.reference_name = "chr1"
        self.reference_start = 10 * i
        self.reference_end = 10 * i + 100
        self.mapq = 60
        self.flag = 0
        self.sa = sa

    def get_tags(self):
        return [] if self.sa is None else [("SA", self.sa)]


def adversarial_values():
    """SA values (str, or None: no tag) for every parity trap of the host reduction."""
    e = "chr1,100,+,50S100M,60,0;"
    v = [
        None, "", e, e * 3,
        e + "chr2,5,-,10M,3,1",                      # unterminated last entry: dropped
        "chr2,5,-,10M,3,1",                          # one unterminated entry
        ";;", e + ";;" + e, ";" + e + ";",            # empty entries
        "chr1,100,+,50M;", "chr1,100,+,50M,7;", "chr1,100,+,50M,7,0;", "chr1,100,+,50M,7,0,extra;",   # 4, 5, 6, 7 fields
        "chr1,100,+,50M,7,0,x,y,z;", ",,,,;", ",,,;", "chr1,,,,;",
        "chr3,1,+,5M,1,0;chr,2,+,5M,1,0;chr10,3,-,5M,1,0;chr1,4,+,5M,1,0;chr1 ,5,+,5M,1,0;CHR1,6,+,5M,1,0;",   # unknown / prefix names
        "chrX,7,+,5M,1,0;c,8,+,5M,1,0;chr10x,9,+,5M,1,0;chré,10,+,5M,1,0;",
        "chr1,1,+,5H10S20M3I4D5=6X7N8P9S,1,0;",      # H then S: the first op is H, no leading clip
        "chr1,1,+,10S20M5H,1,0;chr1,1,+,10S,1,0;chr1,1,+,S,1,0;chr1,1,+,10M5,1,0;chr1,1,+,10m5s,1,0;",
        "chr1,1,+,*,1,0;chr1,1,+,,1,0;chr1,1,+,000000000000000123M0000045S,1,0;chr1,1,+,2147483647M,1,0;",
        "chr1,1,+,1000000000M1000000000D147483647=,1,0;chr1,1,+,12=13X14N15P16I17D,1,0;",
        "chr1,-5,+,5M,1,0;chr1,+7,-,5M,1,0;chr1, 12,+,5M,1,0;chr1,\t\n-12,+,5M,1,0;chr1,12abc,+,5M,1,0;chr1,-2147483647,+,5M,1,0;",
        "chr1,2147483647,+,5M,1,0;chr1,0,+,5M,1,0;chr1,-,+,5M,1,0;chr1,+-3,+,5M,1,0;",
        "chr1,1,+,5M,255,0;chr1,1,+,5M,,0;chr1,1,+,5M,-3,0;chr1,1,+,5M,2147483647,0;chr1,1,+,5M,-2147483648,0;chr1,1,+,5M,7x;",
        "chr1,1,,5M,1,0;chr1,1,x,5M,1,0;chr1,1,++,5M,1,0;chr1,1,-+,5M,1,0;chr1,1, +,5M,1,0;",
        e + "chr2,1,+,5M,1,0\0;" + e,                # an embedded NUL ends the value
        e + "\0" + e, "\0" + e,
        "chr2,1,+,5M,1,0;" * 1000,                   # 1 000 entries
        ("chr10,%d,-,%dS%dM%dD%dS,%d,3;" % (1, 2, 3, 4, 5, 6)) * 7 + "x" * 70 + ";" + "y" * 31 + "," * 33 + ";",
    ]
    return v


def random_values(seed, n):
    """Seeded SA values built from fields that move the ';' and ',' across 32-byte strip borders."""
    rng = np.random.default_rng(seed)
    names = NAMES + ["chr3", "chr", "chr1_alt", "x"]
    ops = "MIDNSHP=X"
    out = []
    for _ in range(n):
        if rng.random() < 0.2:
            out.append(None if rng.random() < 0.5 else "")
            continue
        ents = []
        for _ in range(int(rng.choice([1, 1, 2, 3, 5, 9, 40]))):
            cig = "".join("%d%s" % (int(rng.integers(0, 10 ** int(rng.integers(1, 7)))), ops[int(rng.integers(0, len(ops)))])
                          for _ in range(int(rng.integers(0, 12))))
            f = [names[int(rng.integers(0, len(names)))], str(int(rng.integers(-5, 3_000_000))), "+-x"[int(rng.integers(0, 3))], cig,
                 str(int(rng.integers(0, 256))), str(int(rng.integers(0, 50)))]
            k = int(rng.choice([3, 4, 5, 6, 6, 6, 7]))
            ents.append(",".join((f + ["z" * int(rng.integers(0, 40))])[:k]))
        v = ";".join(ents) + ";"
        if rng.random() < 0.15:
            v = v[:int(rng.integers(0, len(v)))]   # cut anywhere, also inside an entry
        out.append(v)
    return out


def write_bam(path, values):
    bam_writer.write_bam(path, CONTIGS, [Rec(i, v) for i, v in enumerate(values)], block_bytes=7000)


def host_reduce(path):
    """The native decoder's reduction of every record's SA tag: (sa_off, dict of the seven columns)."""
    rd = bamio.BamReader(path, threads=2, keep_seq=False)
    rd.set_chrom_ids(CHROM_ID)
    pk = rd.next_packet(1 << 30)
    assert rd.next_packet(1 << 30) is None
    rd.close()
    return pk["sa_off"], pk["sa"]


def text_arrays(values, lead=5):
    """(text uint8, text_off int64) of the values as written (UTF-8), behind `lead` bytes that belong to no record."""
    parts = [b"" if v is None else v.encode() for v in values]
    off = np.zeros(len(parts) + 1, np.int64)
    np.cumsum([len(p) for p in parts], out=off[1:])
    text = np.frombuffer(b";,\0ab"[:lead] + b"".join(parts), np.uint8).copy()
    return text, off + lead


def name_table(names=NAMES):
    """(bytes, offsets, ids) of contig names sorted bytewise; name k has contig id k of the sorted list."""
    enc = sorted(n.encode() for n in names)
    off = np.zeros(len(enc) + 1, np.int64)
    np.cumsum([len(b) for b in enc], out=off[1:])
    return np.frombuffer(b"".join(enc), np.uint8).copy(), off, np.arange(len(enc), dtype=np.int32)
