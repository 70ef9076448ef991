"""Seeded synthetic workloads shaped like BASELINE.json's configs (SURVEY.md section 8d).

Everything is generated directly as the columnar int32 arrays the C-ABI takes (see
include/cutesv_b200.h): contig ids are ranks of the contig names in Python string order and
read ids are ranks of zero-padded read names, so id order == the reference's string order.

  config 2: 30x ONT whole genome, INS + DEL      (R = 7.75 M reads, 8 388 608 sigs per type)
  config 3: 50x HiFi, all five SV types + genotyping
  config 5: 100x ONT ultra-long (deep pile-ups)

`scale` shrinks genome length, read count and signature counts together so that coverage and
signature density (what the clustering sees) are preserved at small sizes.
"""
import numpy as np

# hg19 contigs of the reference's simulation/LASeR.bed (name, length)
HG19 = [("1", 249250621), ("2", 243199373), ("3", 198022430), ("4", 191154276), ("5", 180915260),
        ("6", 171115067), ("7", 159138663), ("8", 146364022), ("9", 141213431), ("10", 135534747),
        ("11", 135006516), ("12", 133851895), ("13", 115169878), ("14", 107349540),
        ("15", 102531392), ("16", 90354753), ("17", 81195210), ("18", 78077248), ("19", 59128983),
        ("20", 63025520), ("21", 48129895), ("22", 51304566), ("X", 155270560), ("Y", 59373566),
        ("MT", 16569)]

SEED0 = 20260924


def contigs(scale=1.0, n_contigs=None):
    """Contig names sorted in Python string order (id = rank) and their lengths."""
    tab = HG19 if n_contigs is None else HG19[:n_contigs]
    tab = sorted(tab, key=lambda x: x[0])
    names = [t[0] for t in tab]
    lens = np.array([max(int(t[1] * scale), 2000) for t in tab], dtype=np.int64)
    return names, lens


def read_name(i):
    return "read%09d" % i


def _pick_contig(rng, lens, n):
    p = lens / lens.sum()
    return rng.choice(len(lens), size=n, p=p).astype(np.int32)


def synth_reads(rng, lens, n_reads, median=9000.0, sigma=0.7, lo=500, hi=200000, primary_frac=0.97,
                normal=None):
    """reads_info_list rows (cuteSV:729-733).  Returns dict of columns + per-read arrays."""
    chrom = _pick_contig(rng, lens, n_reads)
    if normal is None:
        length = np.clip(rng.lognormal(np.log(median), sigma, n_reads), lo, hi).astype(np.int64)
    else:
        length = np.clip(rng.normal(normal[0], normal[1], n_reads), lo, hi).astype(np.int64)
    clen = lens[chrom]
    length = np.minimum(length, np.maximum(clen - 1, 1))
    start = (rng.random(n_reads) * (clen - length)).astype(np.int64)
    end = start + length
    is_primary = (rng.random(n_reads) < primary_frac).astype(np.uint8)
    read_id = np.arange(n_reads, dtype=np.int32)
    # supplementary rows carry the name of some primary read
    sup = np.flatnonzero(is_primary == 0)
    prim = np.flatnonzero(is_primary == 1)
    if len(sup) and len(prim):
        read_id[sup] = prim[rng.integers(0, len(prim), len(sup))]
    return dict(chrom=chrom, start=start.astype(np.int32), end=end.astype(np.int32), read_id=read_id,
                is_primary=is_primary)


def _covering_index(reads, lens):
    """Per-contig start-sorted views for 'which reads span position p' queries."""
    off = np.concatenate([[0], np.cumsum(lens + 1)])
    lin = off[reads["chrom"]] + reads["start"]
    order = np.argsort(lin, kind="stable")
    return off, lin[order], order


def _loci_support(rng, reads, lens, loci_chrom, loci_pos, het_p=0.5):
    """For every locus pick the reads that carry it. Returns (locus_index, read_row) pairs."""
    off, lin_sorted, order = _covering_index(reads, lens)
    maxlen = int((reads["end"].astype(np.int64) - reads["start"]).max()) if len(order) else 0
    lp = off[loci_chrom] + loci_pos
    lo = np.searchsorted(lin_sorted, lp - maxlen, side="left")
    hi = np.searchsorted(lin_sorted, lp, side="right")
    hom = rng.random(len(lp)) < 0.5
    li, ri = [], []
    ends = reads["end"].astype(np.int64)
    starts = reads["start"].astype(np.int64)
    chrom = reads["chrom"]
    for k in range(len(lp)):
        rows = order[lo[k]:hi[k]]
        if len(rows) == 0:
            continue
        rows = rows[(chrom[rows] == loci_chrom[k]) & (starts[rows] + 50 <= loci_pos[k]) &
                    (ends[rows] - 50 > loci_pos[k])]
        if len(rows) == 0:
            continue
        if not hom[k]:
            rows = rows[rng.random(len(rows)) < het_p]
        li.append(np.full(len(rows), k, dtype=np.int64))
        ri.append(rows)
    if not li:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(li), np.concatenate(ri)


def synth_indel(rng, lens, reads, n_sigs, n_loci, svtype, half_frac=0.02, short_seq_frac=0.05,
                dup_frac=0.002):
    """DEL / INS signature columns: true loci + uniform noise (SURVEY.md 8d, config 2)."""
    loci_chrom = _pick_contig(rng, lens, n_loci)
    loci_pos = (rng.random(n_loci) * np.maximum(lens[loci_chrom] - 200, 1)).astype(np.int64) + 100
    loci_len = np.clip(rng.lognormal(np.log(150.0), 1.0, n_loci), 50, 20000)
    li, ri = _loci_support(rng, reads, lens, loci_chrom, loci_pos)
    if len(li) > n_sigs:
        li, ri = li[:n_sigs], ri[:n_sigs]
    n_true = len(li)
    t_chrom = loci_chrom[li]
    t_pos = np.clip(loci_pos[li] + rng.integers(-15, 16, n_true), 0, lens[t_chrom] - 1)
    t_len = np.maximum((loci_len[li] * rng.normal(1.0, 0.04, n_true)).astype(np.int64), 10)
    t_rid = reads["read_id"][ri]
    n_noise = n_sigs - n_true
    rr = rng.integers(0, len(reads["chrom"]), n_noise)
    n_chrom = reads["chrom"][rr]
    span = np.maximum(reads["end"][rr].astype(np.int64) - reads["start"][rr], 1)
    n_pos = reads["start"][rr] + (rng.random(n_noise) * span).astype(np.int64)
    n_len = 10 + rng.geometric(0.15, n_noise)
    n_rid = reads["read_id"][rr]
    chrom = np.concatenate([t_chrom, n_chrom]).astype(np.int32)
    pos = np.concatenate([t_pos, n_pos]).astype(np.int64)
    length = np.concatenate([t_len, n_len]).astype(np.int32)
    rid = np.concatenate([t_rid, n_rid]).astype(np.int32)
    half = (rng.random(len(chrom)) < half_frac).astype(np.int64)
    seqlen = length.copy()
    short = rng.random(len(chrom)) < short_seq_frac
    seqlen[short] = (seqlen[short] * rng.random(int(short.sum()))).astype(np.int32)
    # exact duplicates (the reference's remove_duplicates_sorted must drop them)
    nd = int(len(chrom) * dup_frac)
    if nd:
        src = rng.integers(0, len(chrom), nd)
        dst = rng.integers(0, len(chrom), nd)
        for col in (chrom, pos, length, rid, half, seqlen):
            col[dst] = col[src]
    perm = rng.permutation(len(chrom))
    chrom, pos, length, rid, half, seqlen = (x[perm] for x in (chrom, pos, length, rid, half, seqlen))
    if svtype == "DEL":
        return dict(chrom=chrom, a=pos.astype(np.int32), b=length, read_id=rid, c=None)
    return dict(chrom=chrom, a=(2 * pos + half).astype(np.int32), b=length, read_id=rid, c=seqlen)


def synth_dup(rng, lens, reads, n_loci, noise):
    loci_chrom = _pick_contig(rng, lens, n_loci)
    size = np.clip(rng.lognormal(np.log(3000.0), 1.0, n_loci), 100, 80000).astype(np.int64)
    p1 = (rng.random(n_loci) * np.maximum(lens[loci_chrom] - size - 200, 1)).astype(np.int64) + 100
    li, ri = _loci_support(rng, reads, lens, loci_chrom, p1)
    n = len(li)
    a = p1[li] + rng.integers(-20, 21, n)
    b = p1[li] + size[li] + rng.integers(-20, 21, n)
    # a second allele on some loci (exercises the pos2 sub-clustering)
    alt = rng.random(n) < 0.1
    b[alt] += 2000
    rr = rng.integers(0, len(reads["chrom"]), noise)
    na = reads["start"][rr].astype(np.int64) + 10
    nb = na + rng.integers(50, 5000, noise)
    chrom = np.concatenate([loci_chrom[li], reads["chrom"][rr]]).astype(np.int32)
    aa = np.maximum(np.concatenate([a, na]), 0).astype(np.int32)
    bb = np.concatenate([b, nb]).astype(np.int32)
    rid = np.concatenate([reads["read_id"][ri], reads["read_id"][rr]]).astype(np.int32)
    perm = rng.permutation(len(chrom))
    return dict(chrom=chrom[perm], a=aa[perm], b=bb[perm], read_id=rid[perm], c=None)


def synth_inv(rng, lens, reads, n_loci, noise):
    loci_chrom = _pick_contig(rng, lens, n_loci)
    size = np.clip(rng.lognormal(np.log(5000.0), 1.0, n_loci), 100, 90000).astype(np.int64)
    p1 = (rng.random(n_loci) * np.maximum(lens[loci_chrom] - size - 200, 1)).astype(np.int64) + 100
    cols = []
    for strand in (0, 1):
        li, ri = _loci_support(rng, reads, lens, loci_chrom, p1 if strand == 0 else p1 + size)
        n = len(li)
        a = p1[li] + rng.integers(-30, 31, n) + strand * 3
        b = p1[li] + size[li] + rng.integers(-30, 31, n) + strand * 3
        cols.append((loci_chrom[li], a, b, reads["read_id"][ri], np.full(n, strand)))
    rr = rng.integers(0, len(reads["chrom"]), noise)
    na = reads["start"][rr].astype(np.int64) + 10
    cols.append((reads["chrom"][rr], na, na + rng.integers(50, 5000, noise), reads["read_id"][rr],
                 rng.integers(0, 2, noise)))
    chrom = np.concatenate([c[0] for c in cols]).astype(np.int32)
    a = np.maximum(np.concatenate([c[1] for c in cols]), 0).astype(np.int32)
    b = np.concatenate([c[2] for c in cols]).astype(np.int32)
    rid = np.concatenate([c[3] for c in cols]).astype(np.int32)
    st = np.concatenate([c[4] for c in cols]).astype(np.int32)
    perm = rng.permutation(len(chrom))
    return dict(chrom=chrom[perm], a=a[perm], b=b[perm], read_id=rid[perm], c=st[perm])


def synth_tra(rng, lens, reads, n_loci, noise):
    loci_chrom = _pick_contig(rng, lens, n_loci)
    chr2 = _pick_contig(rng, lens, n_loci)
    typ = rng.integers(0, 4, n_loci)
    p1 = (rng.random(n_loci) * np.maximum(lens[loci_chrom] - 400, 1)).astype(np.int64) + 100
    p2 = (rng.random(n_loci) * np.maximum(lens[chr2] - 400, 1)).astype(np.int64) + 100
    li, ri = _loci_support(rng, reads, lens, loci_chrom, p1)
    n = len(li)
    a = p1[li] + rng.integers(-10, 11, n)
    b = p2[li] + rng.integers(-10, 11, n)
    alt = rng.random(n) < 0.15  # second mate-position allele
    b[alt] += 500
    c = chr2[li] * 4 + typ[li]
    rr = rng.integers(0, len(reads["chrom"]), noise)
    nc2 = _pick_contig(rng, lens, noise)
    na = reads["start"][rr].astype(np.int64) + 10
    nb = (rng.random(noise) * np.maximum(lens[nc2] - 10, 1)).astype(np.int64)
    ncc = nc2 * 4 + rng.integers(0, 4, noise)
    chrom = np.concatenate([loci_chrom[li], reads["chrom"][rr]]).astype(np.int32)
    aa = np.maximum(np.concatenate([a, na]), 0).astype(np.int32)
    bb = np.maximum(np.concatenate([b, nb]), 0).astype(np.int32)
    rid = np.concatenate([reads["read_id"][ri], reads["read_id"][rr]]).astype(np.int32)
    cc = np.concatenate([c, ncc]).astype(np.int32)
    perm = rng.permutation(len(chrom))
    return dict(chrom=chrom[perm], a=aa[perm], b=bb[perm], read_id=rid[perm], c=cc[perm])


def make_config(config_id=2, scale=1.0, seed=None):
    """Build one of BASELINE.json's synthetic configs.

    Returns dict(names, lens, reads, sigs={type_name: cols}, params=dict(...), n_sigs).
    """
    rng = np.random.default_rng((SEED0 + config_id) if seed is None else seed)
    names, lens = contigs(scale)
    sigs = {}
    if config_id in (2, 4):
        n_reads = max(int(7750000 * scale), 200)
        n_sigs = max(int(8388608 * scale), 64)
        n_loci = max(int(20000 * scale), 4)
        reads = synth_reads(rng, lens, n_reads)
        sigs["DEL"] = synth_indel(rng, lens, reads, n_sigs, n_loci, "DEL")
        sigs["INS"] = synth_indel(rng, lens, reads, n_sigs, n_loci, "INS")
        # ONT preset (cuteSV_Description.py:30-46) + --genotype
        params = dict(min_support=10, bias_ins=100, ratio_ins=0.3, bias_del=100, ratio_del=0.3, genotype=1)
    elif config_id == 3:
        n_reads = max(int(8600000 * scale), 200)
        reads = synth_reads(rng, lens, n_reads, normal=(18000.0, 3000.0), lo=1000, hi=60000)
        n_loci = max(int(25000 * scale), 4)
        n_sigs = max(int(8388608 * scale / 20) + n_loci * 50, 64)
        sigs["DEL"] = synth_indel(rng, lens, reads, n_sigs, n_loci, "DEL")
        sigs["INS"] = synth_indel(rng, lens, reads, n_sigs, n_loci, "INS")
        sigs["DUP"] = synth_dup(rng, lens, reads, max(int(3000 * scale), 2), max(int(20000 * scale), 8))
        sigs["INV"] = synth_inv(rng, lens, reads, max(int(300 * scale), 2), max(int(5000 * scale), 8))
        sigs["TRA"] = synth_tra(rng, lens, reads, max(int(300 * scale), 2), max(int(5000 * scale), 8))
        # HiFi preset + --genotype
        params = dict(min_support=3, bias_ins=1000, ratio_ins=0.9, bias_del=1000, ratio_del=0.5, genotype=1)
    elif config_id == 5:
        n_reads = max(int(3100000 * scale), 200)
        reads = synth_reads(rng, lens, n_reads, median=60000.0, sigma=0.9, lo=1000, hi=1000000)
        n_loci = max(int(20000 * scale), 4)
        n_sigs = max(int(3 * 8388608 * scale), 64)
        sigs["DEL"] = synth_indel(rng, lens, reads, n_sigs, n_loci, "DEL")
        sigs["INS"] = synth_indel(rng, lens, reads, n_sigs, n_loci, "INS")
        sigs["DUP"] = synth_dup(rng, lens, reads, max(int(2000 * scale), 2), max(int(20000 * scale), 8))
        sigs["INV"] = synth_inv(rng, lens, reads, max(int(300 * scale), 2), max(int(5000 * scale), 8))
        sigs["TRA"] = synth_tra(rng, lens, reads, max(int(300 * scale), 2), max(int(5000 * scale), 8))
        params = dict(min_support=10, bias_ins=100, ratio_ins=0.3, bias_del=100, ratio_del=0.3, genotype=1)
    else:
        raise ValueError("config_id must be 2, 3, 4 or 5")
    n_total = int(sum(len(v["chrom"]) for v in sigs.values()))
    return dict(names=names, lens=lens, reads=reads, sigs=sigs, params=params, n_sigs=n_total,
                config_id=config_id, scale=scale)


def adversarial(seed, n_contigs=3, max_sigs=400):
    """Small dense cases that hit the reference's quirks: ties in pos/len, many signatures per
    read, pile-ups, odd biases, tiny supports, x.5 INS positions, short INS seqs, duplicates."""
    rng = np.random.default_rng(seed)
    names, lens = contigs(1.0, n_contigs)
    lens = np.minimum(lens, 200000).astype(np.int64)
    n_reads = int(rng.integers(5, 120))
    span = int(rng.choice([300, 2000, 30000]))
    base = rng.integers(0, 50000, n_contigs)
    rc = rng.integers(0, n_contigs, n_reads).astype(np.int32)
    rs = np.maximum(base[rc] - rng.integers(0, 20000, n_reads), 0)
    re_ = base[rc] + span + rng.integers(-span // 2, 20000, n_reads)
    re_ = np.maximum(re_, rs + 1)
    prim = (rng.random(n_reads) < 0.85).astype(np.uint8)
    rid = np.arange(n_reads, dtype=np.int32)
    sup = np.flatnonzero(prim == 0)
    pr = np.flatnonzero(prim == 1)
    if len(sup) and len(pr):
        rid[sup] = pr[rng.integers(0, len(pr), len(sup))]
    reads = dict(chrom=rc, start=rs.astype(np.int32), end=re_.astype(np.int32), read_id=rid, is_primary=prim)
    if rng.random() < 0.1:  # a contig without any reads-table row (call_gt returns [])
        keep = rc != 0
        reads = {k: v[keep] for k, v in reads.items()}

    def col(n, kind):
        chrom = rng.integers(0, n_contigs, n).astype(np.int32)
        a = base[chrom] + rng.integers(0, span, n)
        r = rng.integers(0, n_reads, n).astype(np.int32)
        if kind in ("DEL", "INS"):
            b = rng.choice([rng.integers(10, 60, n), rng.integers(10, 2000, n),
                            np.full(n, 50) + rng.integers(0, 3, n)][int(rng.integers(0, 3))], n)
            b = np.asarray(b).astype(np.int32)
            if kind == "DEL":
                return dict(chrom=chrom, a=a.astype(np.int32), b=b, read_id=r, c=None)
            half = (rng.random(n) < 0.2).astype(np.int64)
            c = np.where(rng.random(n) < 0.3, (b * rng.random(n)).astype(np.int32), b).astype(np.int32)
            return dict(chrom=chrom, a=(2 * a + half).astype(np.int32), b=b, read_id=r, c=c)
        if kind == "DUP":
            b = a + rng.integers(0, 3000, n)
            return dict(chrom=chrom, a=a.astype(np.int32), b=b.astype(np.int32), read_id=r, c=None)
        if kind == "INV":
            b = a + rng.integers(-100, 3000, n)
            return dict(chrom=chrom, a=a.astype(np.int32), b=np.maximum(b, 0).astype(np.int32), read_id=r,
                        c=rng.integers(0, 2, n).astype(np.int32))
        c2 = rng.integers(0, n_contigs, n)
        b = base[c2] + rng.integers(0, span, n)
        return dict(chrom=chrom, a=a.astype(np.int32), b=b.astype(np.int32), read_id=r,
                    c=(c2 * 4 + rng.integers(0, 4, n)).astype(np.int32))

    sigs = {}
    for kind in ("DEL", "INS", "INV", "DUP", "TRA"):
        n = int(rng.integers(0, max_sigs))
        s = col(n, kind)
        if n > 4:  # exact duplicates
            nd = n // 10
            src, dst = rng.integers(0, n, nd), rng.integers(0, n, nd)
            for k, v in s.items():
                if v is not None:
                    v[dst] = v[src]
        sigs[kind] = s
    ms = int(rng.choice([1, 2, 3, 5, 10]))
    params = dict(min_support=ms, min_size=int(rng.choice([0, 30, 50])), max_size=int(rng.choice([-1, 1000, 100000])),
                  bias_del=int(rng.choice([7, 100, 200, 1000])), bias_ins=int(rng.choice([5, 100, 1001])),
                  bias_inv=int(rng.choice([11, 500])), bias_dup=int(rng.choice([13, 500])),
                  bias_tra=int(rng.choice([3, 50, 501])), ratio_del=float(rng.choice([0.0, 0.3, 0.5, 0.9])),
                  ratio_ins=float(rng.choice([0.0, 0.3, 0.9])), ratio_tra=float(rng.choice([0.3, 0.6, 0.9])),
                  remain_reads_ratio=float(rng.choice([1.0, 1.0, 0.7, 0.5, 0.01, 2.0])),
                  genotype=int(rng.random() < 0.8))
    return dict(names=names, lens=lens, reads=reads, sigs=sigs, params=params,
                n_sigs=int(sum(len(v["chrom"]) for v in sigs.values())), config_id=0, scale=0.0)


# ----------------------------------------------------------------------------------------------
# synthetic alignment records (extraction stage): duck-typed like pysam.AlignedSegment
# ----------------------------------------------------------------------------------------------
class SynthRead(object):
    __slots__ = ("flag", "mapq", "query_length", "query_name", "query_sequence", "reference_start", "reference_end",
                 "reference_name", "cigartuples", "cigar", "tags")

    def get_tags(self):
        return self.tags


def _rand_cigar(rng, target_q, noise, sv_rate, clip):
    """Random CIGAR consuming about target_q query bases.  Returns (tuples, query_len, ref_span)."""
    ops = []
    lead = int(rng.integers(0, 400)) if clip and rng.random() < 0.5 else 0
    if lead:
        ops.append((5 if rng.random() < 0.2 else 4, lead))
    q = 0
    while q < target_q:
        m = int(rng.integers(5, 400))
        ops.append((int(rng.choice([0, 7, 8], p=[0.8, 0.15, 0.05])), m))
        q += m
        r = rng.random()
        if r < sv_rate:
            ln = int(rng.integers(30, 900))
            ops.append((1 if rng.random() < 0.5 else 2, ln))
        elif r < sv_rate + noise:
            ln = int(rng.integers(1, 25))
            op = int(rng.choice([1, 2, 3, 6]))
            ops.append((op, ln))
        if ops[-1][0] == 1:
            q += ops[-1][1]
    if ops[-1][0] not in (0, 7, 8):
        ops.append((0, int(rng.integers(5, 60))))
    trail = int(rng.integers(0, 400)) if clip and rng.random() < 0.5 else 0
    if trail:
        ops.append((5 if rng.random() < 0.2 else 4, trail))
    qlen = sum(l for o, l in ops if o in (0, 1, 4, 7, 8))
    span = sum(l for o, l in ops if o in (0, 2, 3, 7, 8))
    return ops, qlen, span


def synth_alignments(seed, n_reads=200, n_contigs=3, with_seq=True):
    """Alignment records with CIGAR indels, clips and SA tags that hit every branch of
    analysis_split_read (cuteSV:190-464).  Returns (reads, contig_names, contig_lens)."""
    rng = np.random.default_rng(seed)
    names, lens = contigs(1.0, n_contigs)
    lens = np.minimum(lens, 5000000).astype(np.int64)
    reads = []
    for i in range(n_reads):
        r = SynthRead()
        r.flag = int(rng.choice([0, 16, 2048, 2064, 256, 272, 4, 1024], p=[0.4, 0.35, 0.08, 0.07, 0.03, 0.02, 0.03, 0.02]))
        # a read name has ONE primary record; supplementary records re-use the names of other reads
        reuse = r.flag not in (0, 16) and rng.random() < 0.6
        r.query_name = read_name(int(rng.integers(0, max(n_reads // 2, 1))) if reuse else i)
        r.mapq = int(rng.choice([0, 5, 19, 20, 30, 60], p=[0.05, 0.05, 0.05, 0.1, 0.25, 0.5]))
        ch = int(rng.integers(0, n_contigs))
        r.reference_name = names[ch]
        r.reference_start = int(rng.integers(0, 200000))
        target = int(rng.choice([300, 800, 3000, 12000]))
        ops, qlen, span = _rand_cigar(rng, target, 0.25, 0.08, True)
        r.cigartuples = ops
        r.cigar = ops
        r.query_length = qlen
        r.reference_end = r.reference_start + span
        r.query_sequence = "".join(rng.choice(list("ACGT"), qlen)) if with_seq else None
        tags = [("NM", 3)]
        if rng.random() < 0.45:
            k = int(rng.choice([1, 1, 2, 2, 3, 4, 6, 9]))
            ents = []
            # total read length incl. hard clips is what the reference calls total_L = read.query_length
            L = max(qlen, 50)
            cuts = np.sort(rng.integers(0, L, 2 * k))
            for j in range(k):
                a, b = int(cuts[2 * j]), int(cuts[2 * j + 1])
                if b <= a:
                    b = a + 1
                strand = "+" if rng.random() < 0.6 else "-"
                sch = names[ch] if rng.random() < 0.7 else names[int(rng.integers(0, n_contigs))]
                mode = rng.random()
                if mode < 0.5:
                    pos = r.reference_end + int(rng.integers(-3000, 3000))
                elif mode < 0.8:
                    pos = r.reference_start + int(rng.integers(-3000, 3000))
                else:
                    pos = int(rng.integers(1, 300000))
                pos = max(pos, 1)
                mid = "%dM" % max(b - a, 1)
                if rng.random() < 0.3:
                    mid = "%dM%dD%dM" % (max((b - a) // 2, 1), int(rng.integers(1, 500)), max((b - a) - (b - a) // 2, 1))
                if rng.random() < 0.2:
                    mid = "%d=%dI%dX" % (max((b - a) // 2, 1), int(rng.integers(1, 50)), max((b - a) // 3, 1))
                lead = "%dS" % a if a > 0 and rng.random() < 0.9 else ("%dH" % a if a > 0 else "")
                trail = "%dS" % (L - b) if L - b > 0 and rng.random() < 0.9 else ("%dH" % (L - b) if L - b > 0 else "")
                if strand == "-":
                    lead, trail = trail.replace("S", "S"), lead
                ents.append("%s,%d,%s,%s%s%s,%d,%d" % (sch, pos, strand, lead, mid, trail, int(rng.choice([0, 10, 20, 60])), 7))
            tags.append(("SA", ";".join(ents) + ";"))
        r.tags = tags
        reads.append(r)
    return reads, names, lens


def synth_alignments_long(seed, n_reads=16, n_contigs=3, ops_range=(10000, 30000)):
    """BASELINE config-5-shaped records for the extraction goldens: >= 10^4 CIGAR ops per record (one op per ~7 bp), hard / soft
    clips on both ends, runs of 70-90 chained >= 10 bp insertions (more merged pieces than the kernel buffers), and 2-6 SA
    segments laid out to reach the strand patterns of analysis_split_read (cuteSV:190-464): colinear same-strand chains
    (DEL / INS / DUP rules), +-+ / -+- (INV rules), a foreign contig in the middle (BND + post-loop bridge), mixed tails.
    Returns (reads, contig_names, contig_lens)."""
    rng = np.random.default_rng(seed)
    names, lens = contigs(1.0, n_contigs)
    lens = np.minimum(lens, 40000000).astype(np.int64)
    reads = []
    for i in range(n_reads):
        r = SynthRead()
        r.flag = int(rng.choice([0, 16, 0, 16, 2048, 2064]))
        r.query_name = read_name(i if r.flag in (0, 16) else int(rng.integers(0, max(n_reads // 2, 1))))
        r.mapq = int(rng.choice([60, 60, 30, 20, 5]))
        ch = int(rng.integers(0, n_contigs))
        r.reference_name = names[ch]
        r.reference_start = int(rng.integers(1000, 2000000))
        n_pairs = int(rng.integers(ops_range[0] // 2, ops_range[1] // 2))
        m_len = 1 + rng.geometric(1.0 / 12.0, n_pairs)
        small = 1 + rng.geometric(0.6, n_pairs)
        kind = rng.random(n_pairs)
        other_op = np.where(kind < 0.47, 1, np.where(kind < 0.94, 2, np.where(kind < 0.97, 3, 6)))   # I, D, N, P
        big = rng.random(n_pairs) < 4.0 / n_pairs
        small[big] = 10 + rng.geometric(0.02, int(big.sum()))
        ops = []
        lead_kind = int(rng.choice([0, 4, 5], p=[0.2, 0.5, 0.3]))
        if lead_kind:
            ops.append((lead_kind, int(rng.integers(50, 4000))))
        chain_at = int(rng.integers(0, n_pairs)) if rng.random() < 0.6 else -1
        for k in range(n_pairs):
            ops.append((int(rng.choice([0, 7, 8], p=[0.8, 0.15, 0.05])), int(m_len[k])))
            if k == chain_at:   # 70-90 insertions of 12-20 bp, 20-60 bp apart: one merged signature with > 64 pieces
                for _ in range(int(rng.integers(70, 91))):
                    ops.append((1, int(rng.integers(12, 21))))
                    ops.append((0, int(rng.integers(20, 61))))
            ops.append((int(other_op[k]), int(small[k])))
        ops.append((0, int(rng.integers(5, 60))))
        trail_kind = int(rng.choice([0, 4, 5], p=[0.2, 0.5, 0.3]))
        if trail_kind:
            ops.append((trail_kind, int(rng.integers(50, 4000))))
        qlen = sum(l for o, l in ops if o in (0, 1, 4, 7, 8))
        span = sum(l for o, l in ops if o in (0, 2, 3, 7, 8))
        r.cigartuples = ops
        r.cigar = ops
        r.query_length = qlen
        r.reference_end = r.reference_start + span
        r.query_sequence = "".join(rng.choice(list("ACGT"), qlen))
        tags = [("NM", 3)]
        if r.flag in (0, 16) and rng.random() < 0.85:
            k = int(rng.integers(2, 7))
            pattern = int(rng.integers(0, 5))
            L = qlen
            cuts = np.sort(rng.integers(0, L, k + 1))
            own = "+" if r.flag == 0 else "-"
            flip = {"+": "-", "-": "+"}
            ents = []
            pos = r.reference_end + int(rng.integers(-2000, 2000))
            for j in range(k):
                a, b = int(cuts[j]), int(cuts[j + 1])
                if b <= a:
                    b = a + 1
                if pattern == 0:      # colinear, same strand: DEL / INS / DUP rules
                    strand, sch = own, names[ch]
                    pos += int(rng.integers(-1500, 4000))
                elif pattern == 1:    # alternating strands: + - + / - + - inversion rules
                    strand, sch = (own if j % 2 else flip[own]), names[ch]
                    pos += int(rng.integers(-500, 3000))
                elif pattern == 2:    # a foreign contig in the middle: BND rules + the post-loop bridge
                    mid = 0 < j < k - 1 or k == 2
                    strand, sch = own, (names[(ch + 1) % n_contigs] if mid else names[ch])
                    pos += int(rng.integers(-1000, 3000))
                elif pattern == 3:    # strand change at the tail (rule 4)
                    strand, sch = (flip[own] if j >= k - 2 else own), names[ch]
                    pos += int(rng.integers(-800, 2500))
                else:                 # anything
                    strand = own if rng.random() < 0.5 else flip[own]
                    sch = names[int(rng.integers(0, n_contigs))]
                    pos = int(rng.integers(1, 3000000))
                pos = max(pos, 1)
                seg = max(b - a, 1)
                mid_c = "%dM" % seg if rng.random() < 0.7 else "%dM%dD%dM" % (max(seg // 2, 1), int(rng.integers(1, 300)), max(seg - seg // 2, 1))
                lead = ("%dS" % a if rng.random() < 0.8 else "%dH" % a) if a > 0 else ""
                trail = ("%dS" % (L - b) if rng.random() < 0.8 else "%dH" % (L - b)) if L - b > 0 else ""
                if strand == "-":
                    lead, trail = trail, lead
                ents.append("%s,%d,%s,%s%s%s,%d,%d" % (sch, pos, strand, lead, mid_c, trail, int(rng.choice([60, 60, 20, 3])), 5))
            tags.append(("SA", ";".join(ents) + ";"))
        r.tags = tags
        reads.append(r)
    return reads, names, lens


def synth_bam_dataset(seed=1, n_contigs=2, contig_len=120000, coverage=22, read_len=(2500, 7000), double_ins=0.0):
    """A small coherent long-read dataset for the CLI plumbing test (BASELINE.json config 1 in
    spirit): reads tile the contigs; planted DEL / INS loci appear in the CIGAR of the reads that
    span them (position / length jitter), TRA loci as split reads with SA tags.  Returns
    dict(contigs=[(name, len)], reads=[SynthRead]), fasta {name: seq}."""
    rng = np.random.default_rng(seed)
    names = ["chrA", "chrB", "chrC"][:n_contigs]
    loci = []
    for ci, nm in enumerate(names):
        pos = 6000
        while pos < contig_len - 8000:
            kind = rng.choice(["DEL", "INS", "DEL", "INS", "TRA"]) if ci == 0 else rng.choice(["DEL", "INS"])
            loci.append((nm, int(pos), str(kind), int(rng.integers(60, 600)), bool(rng.random() < 0.5)))
            pos += int(rng.integers(5000, 9000))
    reads = []
    rid = 0
    for nm in names:
        n_reads = int(coverage * contig_len / ((read_len[0] + read_len[1]) / 2))
        starts = np.sort(rng.integers(0, contig_len - read_len[1] - 1000, n_reads))
        for st in starts:
            L = int(rng.integers(read_len[0], read_len[1]))
            r = SynthRead()
            r.query_name = read_name(rid)
            rid += 1
            r.flag = 0 if rng.random() < 0.5 else 16
            r.mapq = int(rng.choice([60, 60, 60, 30, 10]))
            r.reference_name = nm
            r.reference_start = int(st)
            ops = []
            ref = int(st)
            end = int(st) + L
            tags = [("NM", 5)]
            tra_hit = None
            here = [l for l in loci if l[0] == nm and ref + 300 < l[1] < end - 300]
            for (_, lp, kind, ln, hom) in here:
                if not hom and rng.random() < 0.5:
                    continue
                if kind == "TRA":
                    tra_hit = (lp, ln)
                    continue
                lp2 = lp + int(rng.integers(-8, 9))
                if lp2 <= ref + 20:
                    continue
                seg = lp2 - ref
                while seg > 0:  # match run with small noise indels
                    m = int(min(seg, rng.integers(80, 400)))
                    ops.append((0, m))
                    seg -= m
                    ref += m
                    if seg > 10 and rng.random() < 0.3:
                        nl = int(rng.integers(1, 9))
                        if rng.random() < 0.5:
                            ops.append((1, nl))
                        else:
                            ops.append((2, nl))
                            ref += nl
                            seg -= nl
                ln2 = max(int(ln * rng.normal(1.0, 0.03)), 30)
                if kind == "DEL":
                    ops.append((2, ln2))
                    ref += ln2
                elif double_ins > 0 and rng.random() < double_ins:
                    # the same read reports TWO insertions of equal length at the same position ("nInI"): with -mi -1 they stay
                    # two signatures that tie on (chr, int(pos), len, name) and differ only in their sequence (cuteSV:774)
                    ops.append((1, ln2))
                    ops.append((1, ln2))
                else:
                    ops.append((1, ln2))
            if tra_hit is not None:
                end = tra_hit[0] + int(rng.integers(-5, 6))
            if end > ref:
                ops.append((0, end - ref))
                ref = end
            clip = 0
            if tra_hit is not None:  # split read: the tail maps to the last contig
                clip = int(rng.integers(800, 2000))
                ops.append((4, clip))
            qlen = sum(l for o, l in ops if o in (0, 1, 4, 7, 8))
            if tra_hit is not None:
                tgt = 20000 + tra_hit[1] * 10 + int(rng.integers(-5, 6))
                tags.append(("SA", "%s,%d,+,%dS%dM,60,3;" % (names[-1], tgt, qlen - clip, clip)))
                r.flag = 0
            r.cigartuples = ops
            r.cigar = ops
            r.query_length = qlen
            r.reference_end = ref
            r.query_sequence = "".join(rng.choice(list("ACGT"), qlen))
            r.tags = tags
            reads.append(r)
    fasta = {nm: "".join(rng.choice(list("ACGT"), contig_len + 10)) for nm in names}
    return dict(contigs=[(nm, contig_len) for nm in names], reads=reads), fasta


def draft_names(n):
    """Scaffold names of a draft assembly in header order: unpadded numbers, so string order differs from numeric order."""
    return ["scaffold_%d" % k for k in range(n)]


def draft_assembly(n_contigs, seed=7, n_active=40, active_len=400000, n_reads=6000, scale=1.0, median_len=30000.0):
    """Columnar inputs (like make_config) on a draft assembly of `n_contigs` scaffolds with lognormal lengths (median
    `median_len`, at least 1000 bp; the active scaffolds at least `active_len`).  Reads and
    signatures of all five types sit on `n_active` scaffolds that include the contig ids 0, 32767, 32768 and n-1 (those that
    exist); TRA mates pair them up.  Contig ids are ranks of the names in string order, as the C-ABI requires."""
    rng = np.random.default_rng(seed)
    header = draft_names(n_contigs)
    by_name = sorted(range(n_contigs), key=header.__getitem__)   # contig id (string-order rank) -> header index
    lens = np.clip(rng.lognormal(np.log(median_len), 1.2, n_contigs), 1000, 5000000).astype(np.int64)[by_name]
    want = [i for i in (0, 32767, 32768, n_contigs - 1) if 0 <= i < n_contigs]
    pool = np.setdiff1d(np.arange(n_contigs), want)
    act = np.unique(np.concatenate([want, rng.choice(pool, min(len(pool), max(n_active - len(want), 0)), replace=False)])).astype(np.int32)
    lens[act] = np.maximum(lens[act], active_len)
    la = lens[act]
    reads = synth_reads(rng, la, n_reads, normal=(18000.0, 3000.0), lo=1000, hi=60000)
    sigs = {"DEL": synth_indel(rng, la, reads, int(40000 * scale), int(600 * scale), "DEL"),
            "INS": synth_indel(rng, la, reads, int(40000 * scale), int(600 * scale), "INS"),
            "DUP": synth_dup(rng, la, reads, int(300 * scale), int(2000 * scale)),
            "INV": synth_inv(rng, la, reads, int(100 * scale), int(1000 * scale)),
            "TRA": synth_tra(rng, la, reads, int(300 * scale), int(3000 * scale))}
    reads["chrom"] = act[reads["chrom"]]
    for t, s in sigs.items():
        s["chrom"] = act[s["chrom"]]
        if t == "TRA":
            s["c"] = (act[s["c"] >> 2] * 4 + (s["c"] & 3)).astype(np.int32)
    params = dict(min_support=3, bias_ins=1000, ratio_ins=0.9, bias_del=1000, ratio_del=0.5, genotype=1)
    names = [header[k] for k in by_name]
    return dict(names=names, lens=lens, reads=reads, sigs=sigs, params=params, active=act,
                n_sigs=int(sum(len(v["chrom"]) for v in sigs.values())))


def synth_draft_bam_dataset(seed=11, n_header=40000, n_active=30, contig_len=60000, coverage=14, read_len=(2500, 7000)):
    """Like synth_bam_dataset on a draft assembly: `n_header` scaffolds in the BAM header, reads on `n_active` of them (among
    them scaffolds whose string-order rank is above 32767), DEL / INS loci in the CIGARs and TRA loci as split reads whose
    SA mate lies on another active scaffold.  Returns dict(contigs=[(name, len)], reads=[SynthRead]), fasta of the active
    scaffolds {name: seq}."""
    rng = np.random.default_rng(seed)
    names = draft_names(n_header)
    rank = {n: i for i, n in enumerate(sorted(names))}
    lens = np.clip(rng.lognormal(np.log(3000.0), 0.8, n_header), 500, 40000).astype(np.int64)
    hi_rank = [k for k in range(n_header) if rank[names[k]] > 32767]
    act = sorted(set(rng.choice(n_header, n_active // 2, replace=False).tolist()) | set(rng.choice(hi_rank, n_active - n_active // 2, replace=False).tolist()))
    for k in act:
        lens[k] = contig_len
    loci = {}
    for k in act:
        pos, lk = 6000, []
        while pos < contig_len - 8000:
            kind = str(rng.choice(["DEL", "INS", "DEL", "INS", "TRA"]))
            mate = int(rng.choice([j for j in act if j != k]))
            lk.append((int(pos), kind, int(rng.integers(60, 600)), bool(rng.random() < 0.5), mate))
            pos += int(rng.integers(5000, 9000))
        loci[k] = lk
    reads, rid = [], 0
    for k in act:
        nm = names[k]
        n_reads = int(coverage * contig_len / ((read_len[0] + read_len[1]) / 2))
        for st in np.sort(rng.integers(0, contig_len - read_len[1] - 1000, n_reads)):
            L = int(rng.integers(read_len[0], read_len[1]))
            r = SynthRead()
            r.query_name = read_name(rid)
            rid += 1
            r.flag = 0 if rng.random() < 0.5 else 16
            r.mapq = int(rng.choice([60, 60, 60, 30, 10]))
            r.reference_name = nm
            r.reference_start = int(st)
            ops, ref, end, tags, tra_hit = [], int(st), int(st) + L, [("NM", 5)], None
            for (lp, kind, ln, hom, mate) in loci[k]:
                if not (ref + 300 < lp < end - 300) or (not hom and rng.random() < 0.5):
                    continue
                if kind == "TRA":
                    tra_hit = (lp, ln, mate)
                    break
                lp2 = lp + int(rng.integers(-8, 9))
                if lp2 <= ref + 20:
                    continue
                ops.append((0, lp2 - ref))
                ref = lp2
                ln2 = max(int(ln * rng.normal(1.0, 0.03)), 30)
                if kind == "DEL":
                    ops.append((2, ln2))
                    ref += ln2
                else:
                    ops.append((1, ln2))
            if tra_hit is not None:
                end = max(tra_hit[0] + int(rng.integers(-5, 6)), ref + 1)
            if end > ref:
                ops.append((0, end - ref))
                ref = end
            clip = 0
            if tra_hit is not None:   # split read: the tail maps to the locus' mate scaffold
                clip = int(rng.integers(800, 2000))
                ops.append((4, clip))
            qlen = sum(l for o, l in ops if o in (0, 1, 4, 7, 8))
            if tra_hit is not None:
                tgt = 20000 + tra_hit[1] * 10 + int(rng.integers(-5, 6))
                tags.append(("SA", "%s,%d,+,%dS%dM,60,3;" % (names[tra_hit[2]], tgt, qlen - clip, clip)))
                r.flag = 0
            r.cigartuples = ops
            r.cigar = ops
            r.query_length = qlen
            r.reference_end = ref
            r.query_sequence = "".join(rng.choice(list("ACGT"), qlen))
            r.tags = tags
            reads.append(r)
    fasta = {names[k]: "".join(rng.choice(list("ACGT"), contig_len + 10)) for k in act}
    return dict(contigs=[(names[k], int(lens[k])) for k in range(n_header)], reads=reads), fasta


def synth_cigar_packet(n_reads, mean_indels=850, seed=5, n_contigs=25, sa_frac=0.0):
    """Vectorised packed alignment packet (no Python objects) shaped like ONT reads: ~1 CIGAR op per
    7 bp, M / small indel alternation, ~1 qualifying (>= 10 bp) insertion and deletion per read
    (BASELINE.json config 5 stresses this CIGAR walk).  Returns a packing.pack_alignments()-style dict."""
    rng = np.random.default_rng(seed)
    names, lens = contigs(1.0, n_contigs)
    k = np.maximum(rng.poisson(mean_indels, n_reads), 1).astype(np.int64)
    n_ops = 2 * k + 1
    off = np.concatenate([[0], np.cumsum(n_ops)])
    T = int(off[-1])
    idx_in_read = np.arange(T, dtype=np.int64) - np.repeat(off[:-1], n_ops)
    is_m = (idx_in_read % 2) == 0
    op = np.where(is_m, 0, np.where(rng.random(T) < 0.5, 1, 2)).astype(np.uint32)
    ln = np.where(is_m, 1 + rng.geometric(1.0 / 12.0, T), 1 + rng.geometric(0.6, T)).astype(np.int64)
    big = (~is_m) & (rng.random(T) < 2.2 / (2.0 * mean_indels))
    ln[big] = 10 + rng.geometric(0.05, int(big.sum()))
    cigar = ((ln.astype(np.uint32) << 4) | op).astype(np.uint32)
    ref_adv = np.where(op != 1, ln, 0)
    q_adv = np.where(op != 2, ln, 0)
    span = np.add.reduceat(ref_adv, off[:-1])
    qlen = np.add.reduceat(q_adv, off[:-1])
    chrom = _pick_contig(rng, lens, n_reads)
    start = (rng.random(n_reads) * np.maximum(lens[chrom] - span - 1, 1)).astype(np.int64)
    out = dict(chrom=chrom.astype(np.int32), ref_start=start.astype(np.int32), ref_end=(start + span).astype(np.int32),
               flag=np.where(rng.random(n_reads) < 0.5, 0, 16).astype(np.int32), mapq=np.full(n_reads, 60, np.int32),
               query_len=qlen.astype(np.int32), read_id=np.arange(n_reads, dtype=np.int32), cigar_off=off.astype(np.int64),
               sa_off=np.zeros(n_reads + 1, dtype=np.int64), cigar=cigar,
               sa={k2: np.zeros(0, np.int32) for k2 in ("chrom", "pos0", "strand", "mapq", "first_clip", "last_clip", "ref_span")})
    if sa_frac > 0:
        # sa_frac of the records carry 1-6 supplementary segments (BASELINE config 5: "dense SA-tag splits"): the query is cut
        # into consecutive pieces, the primary keeps the first one; segments land near the primary (DEL / INS / DUP / INV shaped)
        # or on another contig (TRA shaped)
        has = rng.random(n_reads) < sa_frac
        n_seg = np.where(has, rng.integers(1, 7, n_reads), 0).astype(np.int64)
        sa_off = np.concatenate([[0], np.cumsum(n_seg)])
        S = int(sa_off[-1])
        owner = np.repeat(np.arange(n_reads), n_seg)
        k_in = np.arange(S, dtype=np.int64) - np.repeat(sa_off[:-1], n_seg)
        ql = qlen[owner]
        piece = np.maximum(ql // (n_seg[owner] + 1), 1)
        first_clip = piece * (k_in + 1)                       # query consumed before this segment
        last_clip = np.maximum(ql - first_clip - piece, 0)
        far = rng.random(S) < 0.25
        sa_chrom = np.where(far, rng.integers(0, len(lens), S), chrom[owner]).astype(np.int64)
        jitter = rng.integers(-3000, 3000, S)
        near_pos = start[owner] + (span[owner] * (k_in + 1)) // (n_seg[owner] + 1) + jitter
        sa_span = np.maximum(piece + rng.integers(-20, 20, S), 1)
        pos0 = np.where(far, (rng.random(S) * np.maximum(lens[sa_chrom] - sa_span - 1, 1)).astype(np.int64), near_pos)
        pos0 = np.clip(pos0, 0, np.maximum(lens[sa_chrom] - sa_span - 1, 0))
        same = (out["flag"][owner] == 16).astype(np.int64)
        strand = np.where(rng.random(S) < 0.8, same, 1 - same)
        out["sa_off"] = sa_off.astype(np.int64)
        out["sa"] = dict(chrom=sa_chrom.astype(np.int32), pos0=pos0.astype(np.int32), strand=strand.astype(np.int32),
                         mapq=np.where(rng.random(S) < 0.9, 60, 5).astype(np.int32), first_clip=first_clip.astype(np.int32),
                         last_clip=last_clip.astype(np.int32), ref_span=sa_span.astype(np.int32))
        # the primary of a split read is soft-clipped at its end by what the segments consume
        # (the CIGAR stays as generated: the clip only matters to the split-read engine through query_len / segment bounds)
    return out, names, lens


def synth_config1_dataset(loci, contig="22", contig_len=51304566, seed=20260924, reads_per_locus=15):
    """BASELINE.json configs[0] (SURVEY 8d config 1): BED-driven chr22 INS+DEL, ~5k synthetic reads.
    loci: [[kind, start, length], ...] (chr22 rows of the reference's simulation BEDs, committed as
    tests/golden/sim_chr22_loci.json).  ~15 reads per locus, read length lognormal(median 9 kb, sigma 0.7)
    clipped to [500, 200k], 50 % het / 50 % hom, CIGAR = M runs with small noise indels + the SV op
    (+-15 bp position jitter, +-4 % length jitter), 10 % of the SVs expressed as an SA split instead of a
    CIGAR op.  Returns (dict(contigs, reads), fasta_as_function)."""
    rng = np.random.default_rng(seed)
    reads = []
    rid = 0
    for kind, pos, ln in loci:
        hom = rng.random() < 0.5
        for _ in range(reads_per_locus):
            carries = hom or rng.random() < 0.5
            L = int(np.clip(rng.lognormal(np.log(9000.0), 0.7), 500, 200000))
            left = int(rng.integers(int(0.1 * L), int(0.9 * L) + 1))
            st = max(pos - left, 0)
            r = SynthRead()
            r.query_name = read_name(rid)
            rid += 1
            r.flag = 0 if rng.random() < 0.5 else 16
            r.mapq = 60
            r.reference_name = contig
            r.reference_start = st
            ops = []
            tags = [("NM", 7)]
            ref = st

            def m_run(n, ref):
                while n > 0:
                    m = int(min(n, rng.integers(60, 300)))
                    ops.append((0, m))
                    n -= m
                    ref += m
                    if n > 12 and rng.random() < 0.10:
                        nl = int(rng.integers(1, 10))
                        if rng.random() < 0.5:
                            ops.append((1, nl))
                        else:
                            ops.append((2, nl))
                            ref += nl
                            n -= nl
                return ref
            split = carries and rng.random() < 0.10
            if carries and not split:
                p2 = pos + int(rng.integers(-15, 16))
                ref = m_run(max(p2 - ref, 1), ref)
                l2 = max(int(round(ln * (1.0 + rng.uniform(-0.04, 0.04)))), 30)
                if kind == "DEL":
                    ops.append((2, l2))
                    ref += l2
                else:
                    ops.append((1, l2))
                ref = m_run(max(st + L - ref, 50), ref)
            elif split:
                # primary covers the left flank and soft-clips the rest; the SA entry maps the right flank
                ref = m_run(max(pos - ref, 1), ref)
                tail = max(L - (pos - st), 200)
                l2 = max(int(round(ln * (1.0 + rng.uniform(-0.04, 0.04)))), 30)
                ops.append((4, tail + (l2 if kind == "INS" else 0)))
                qlen_now = sum(l for o, l in ops if o in (0, 1, 4, 7, 8))
                sa_pos = pos + (l2 if kind == "DEL" else 0) + 1
                strand = "+" if r.flag == 0 else "-"
                lead = qlen_now - tail
                sa_cig = ("%dS%dM" % (lead, tail)) if r.flag == 0 else ("%dM%dS" % (tail, lead))
                tags.append(("SA", "%s,%d,%s,%s,60,5;" % (contig, sa_pos, strand, sa_cig)))
                if r.flag == 16:  # reverse-strand records store the clip on the other side
                    ops = [ops[-1]] + ops[:-1]
            else:
                ref = m_run(L, ref)
            r.cigartuples = ops
            r.cigar = ops
            r.query_length = sum(l for o, l in ops if o in (0, 1, 4, 7, 8))
            r.reference_end = st + sum(l for o, l in ops if o in (0, 2, 3, 7, 8))
            r.query_sequence = "".join(rng.choice(list("ACGT"), r.query_length))
            r.tags = tags
            reads.append(r)
    return dict(contigs=[(contig, contig_len)], reads=reads)


def pseudo_fasta_line(contig, length, seed=3, width=60):
    """Deterministic pseudo-random reference sequence, generated in chunks (used for the 51 Mb chr22 fixture)."""
    rng = np.random.default_rng(seed)
    alphabet = np.frombuffer(b"ACGT", dtype=np.uint8)
    return alphabet[rng.integers(0, 4, length)].tobytes().decode()


def random_params(seed):
    """Flag combinations well away from the presets (every cuteSV clustering / genotyping flag), for parity sweeps."""
    rng = np.random.default_rng(seed)
    ms = int(rng.choice([1, 2, 3, 5, 8, 10]))
    return dict(min_support=ms, min_size=int(rng.choice([1, 30, 50, 200])), max_size=int(rng.choice([-1, 1000, 100000])),
                bias_del=int(rng.choice([1, 20, 100, 200, 1000])), bias_ins=int(rng.choice([1, 20, 100, 1000])),
                bias_inv=int(rng.choice([10, 500, 2000])), bias_dup=int(rng.choice([10, 500, 2000])), bias_tra=int(rng.choice([5, 50, 400])),
                ratio_del=float(rng.choice([0.0, 0.1, 0.3, 0.5, 0.9, 2.0])), ratio_ins=float(rng.choice([0.0, 0.2, 0.3, 0.9, 1.5])),
                ratio_tra=float(rng.choice([0.1, 0.6, 1.0])), remain_reads_ratio=float(rng.choice([0.3, 0.5, 0.8, 1.0, 1.7])),
                genotype=int(rng.integers(0, 2)), gt_round=int(rng.choice([1, 5, 50, 500])))   # (gt_bias_ins is the reference's constant 1000, resolveINDEL.py:312)
