"""csv_sort_sigs inputs whose key lands on the edges of the radix rounds.  The library gives every key field the bits its
largest value needs (bits_for, at least 1), concatenates the fields (contig first) and sorts the string from its least
significant end in rounds of up to 64 bits: a round of up to 32 bits on uint32 keys, a wider one on uint64 keys, each round
ceil(width / 8) onesweep passes.  Every case names the field maxima and the total key bits they must give."""

FIELDS = {"DEL": ("chrom", "a", "b", "read_id"), "TRA": ("chrom", "c", "a", "b", "read_id")}

# name: (svtype, {field: largest value}, total key bits).  TRA's c is chr2 * 4 + type, so its largest value is 4 n - 1 for
# n contigs and chrom's is n - 1.
ROUND_EDGES = {
    "DEL_32": ("DEL", dict(chrom=1, a=(1 << 10) - 1, b=(1 << 10) - 1, read_id=(1 << 11) - 1), 32),
    "DEL_33": ("DEL", dict(chrom=1, a=1 << 10, b=(1 << 10) - 1, read_id=(1 << 11) - 1), 33),
    "DEL_64": ("DEL", dict(chrom=3, a=(1 << 20) - 1, b=1 << 20, read_id=(1 << 21) - 1), 64),
    "DEL_65": ("DEL", dict(chrom=3, a=1 << 20, b=1 << 20, read_id=(1 << 21) - 1), 65),
    "TRA_32": ("TRA", dict(chrom=1, c=7, a=(1 << 9) - 1, b=(1 << 9) - 1, read_id=(1 << 10) - 1), 32),
    "TRA_33": ("TRA", dict(chrom=1, c=7, a=(1 << 9) - 1, b=(1 << 9) - 1, read_id=1 << 10), 33),
    "TRA_64": ("TRA", dict(chrom=1, c=7, a=(1 << 20) - 1, b=(1 << 20) - 1, read_id=(1 << 20) - 1), 64),
    "TRA_65": ("TRA", dict(chrom=1, c=7, a=(1 << 20) - 1, b=(1 << 20) - 1, read_id=1 << 20), 65),
    "TRA_128": ("TRA", dict(chrom=(1 << 17) - 1, c=(1 << 19) - 1, a=(1 << 30) - 1, b=(1 << 31) - 1, read_id=(1 << 31) - 1), 128),
    "TRA_129": ("TRA", dict(chrom=(1 << 17) - 1, c=(1 << 19) - 1, a=1 << 30, b=(1 << 31) - 1, read_id=(1 << 31) - 1), 129),
}


def bits_for(max_value):
    """Bits of the largest value, at least 1 (bits_for in cutesv_b200.cu)."""
    return max(1, int(max_value).bit_length())


def total_bits(svtype, maxima):
    return sum(bits_for(maxima[f]) for f in FIELDS[svtype])


def rounds(total):
    """Widths of the LSD rounds over the concatenated key: 64 bits at a time from the least significant end."""
    return [min(64, total - lo) for lo in range(0, total, 64)]


def onesweep_passes(total):
    return sum(max(1, (w + 7) // 8) for w in rounds(total))


def n_contigs(svtype, maxima):
    return maxima["chrom"] + 1
