"""Chain clusters planted at the size-class boundaries of the cluster kernels, the counters they must produce, and integer
vectors whose CIPOS / CILEN sits exactly on an integer so that a summation order other than numpy's changes the record.

Size classes of a kept chain cluster of m members (m counted before duplicate removal):
  m <= 32     k_cluster_small (INS / DEL, every member kept, small path on): inline std of indel_cluster_small
  m <= 128    k_cluster_warp: register bitonic sorts at M = 32 / 64 / 128, warp_np_std2
  m <= 2048   k_cluster_block on its shared-memory arena: np_pairwise_sum on two lanes
  m >  2048   k_cluster_block on global scratch

Exact-boundary vectors.  cal_CIPOS is int(1.96 * sqrt(S / n) / n ** 0.5) with S = sum((x - mean) ** 2).  With
S = (25 k n / 49) ** 2 and 49 | 25 k n the exact value is the integer k, and the float result lands a few ulp on either
side of it.  Which side depends on the last bits of the computed S, and those depend on the summation order as long as the
mean is not dyadic: sum(x) = r (mod n) with n | r * r and r / n not dyadic.  Deviations d = x - base therefore satisfy
sum(d) = r and sum(d * d) = S + r * r / n (which needs sum(d * d) = sum(d) mod 2).  The generator draws n - 2 deviations,
walks them until the last two are the integer roots of a + b = R, a * a + b * b = Q, and keeps the vector only when numpy's
answer differs from one of the MUTANTS below.  The test is made on the values as planted, BASE + d: the rounding of the mean
and of every x - mean depends on the magnitude of x, so a vector chosen at one base says nothing about another.  Every
planted allele therefore sits at BASE, on a contig of its own, and has length BASE + its length deviation.  Nothing here
calls the oracle or the library."""
import functools
import math

import numpy as np

from cutesv_b200 import _abi

SMALL_M, WARP_M, BLOCK_M = 32, 128, 2048
ALL_TYPES = _abi.TYPE_NAMES

# ---------------------------------------------------------------------------------------------------------------------
# numpy's pairwise summation (np.add.reduce on float64) and wrong orders a kernel could plausibly use
# ---------------------------------------------------------------------------------------------------------------------
MUTANTS = ("sequential",   # one running sum
           "pair4",        # leaf tree (r0+r4)+(r2+r6)+... : a xor butterfly run at distances 4, 2, 1
           "tail_first",   # the n % 8 tail summed first and the tree added to it
           "no_split",     # one leaf for any n (no recursion above 128)
           "split_half")   # recursion at n / 2 without rounding down to a multiple of 8


def _leaf(x, lo, n, mutant):
    if n < 8:
        res = 0.0
        for i in range(lo, lo + n):
            res += float(x[i])
        return res
    n8 = n - n % 8
    r = x[lo:lo + 8].copy()
    for i in range(lo + 8, lo + n8, 8):
        r += x[i:i + 8]   # eight independent accumulators, elementwise IEEE adds
    r = [float(v) for v in r]
    if mutant == "pair4":
        res = ((r[0] + r[4]) + (r[2] + r[6])) + ((r[1] + r[5]) + (r[3] + r[7]))
    else:
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    if mutant == "tail_first":
        tail = 0.0
        for i in range(lo + n8, lo + n):
            tail += float(x[i])
        return tail + res
    for i in range(lo + n8, lo + n):
        res += float(x[i])
    return res


def pairwise_sum(x, mutant=None):
    """numpy's pairwise_sum (blocks of 128, eight accumulators per block, split rounded down to a multiple of 8);
    `mutant` names one of MUTANTS instead."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    if mutant == "sequential":
        res = 0.0
        for v in x.tolist():   # (not builtin sum: it compensates float rounding)
            res += v
        return res

    def rec(lo, n):
        if n <= 128 or mutant == "no_split":
            return _leaf(x, lo, n, mutant)
        n2 = n // 2
        if mutant != "split_half":
            n2 -= n2 % 8
        return rec(lo, n2) + rec(lo + n2, n - n2)
    return rec(0, len(x))


def np_std(v, mutant=None):
    """np.std of an integer list in the given order (mean = exact integer sum / n, sqrt(pairwise(d * d) / n))."""
    v = np.asarray(v, dtype=np.int64)
    mean = float(int(v.sum())) / len(v)
    d = v.astype(np.float64) - mean
    return math.sqrt(pairwise_sum(d * d, mutant) / len(v))


def cal_cipos(std, n):
    """cal_CIPOS (cuteSV_genotype.py): the integer CIPOS / CILEN of an allele of n reads."""
    return int(1.96 * std / n ** 0.5)


def defeated(v):
    """The mutants whose cal_CIPOS of v differs from numpy's."""
    want = cal_cipos(float(np.std(np.asarray(v, dtype=np.int64))), len(v))
    return {m for m in MUTANTS if cal_cipos(np_std(v, m), len(v)) != want}


# ---------------------------------------------------------------------------------------------------------------------
# exact-boundary vectors
# ---------------------------------------------------------------------------------------------------------------------
# tier -> ((n, r), ...): n | r * r, r / n not dyadic.  2304 halves to multiples of 8 all the way down, so no vector of
# that size can tell the rounded split from the plain one; 2401 can.
TIERS = {
    "small": ((25, 5),),
    "warp": ((36, 12), (49, 7), (100, 20)),        # M = 64 and M = 128 register sorts
    "cta": ((147, 21), (225, 15), (2025, 45)),
    "giant": ((2304, 96), (2401, 49)),
}
# mutants each tier's planted vectors must defeat.  Giant: the bounded search (80 vectors per size) finds no 2401-value
# vector on which the unrounded split changes cal_CIPOS, and 2304 cannot show it at all; only the CTA tier covers that
# mutant.
TIER_NEEDS = {"small": {"sequential", "pair4"}, "warp": {"sequential", "pair4"},
              "cta": {"sequential", "pair4", "no_split", "split_half"}, "giant": {"sequential", "pair4", "no_split"}}
POS_MAX_GAP = 90     # sorted neighbours of a position vector stay closer than the INS / DEL bias (100 / 200)
BASE = 40000         # planted position and length of an exact-boundary allele = BASE + deviation (above every deviation)


def _boundary_vector(rng, n, r, k, distinct, max_gap, steps=40000):
    """Deviations d (len n) with sum(d) = r and sum((d - r/n) ** 2) = (25 k n / 49) ** 2, or None."""
    S = (25 * k * n // 49) ** 2
    Q_all = S + r * r // n
    sd = math.sqrt(S / n)
    # n - 2 values spread evenly over [-a, a] with jitter (variance ~ sd ** 2, small gaps, distinct), centred on r / n
    a = sd * math.sqrt(3.0) * (n - 1) / n
    grid = np.linspace(-a, a, n - 2)
    h = 0.45 * (grid[1] - grid[0])
    d = np.rint(grid + rng.uniform(-h, h, n - 2)).astype(np.int64)
    if distinct and len(np.unique(d)) != n - 2:
        return None
    d = [int(v) for v in d]
    R = r - sum(d)
    Q = Q_all - sum(v * v for v in d)
    used = set(d)
    lim = 2 * int(a) + 2
    # |p - q| = sqrt(X) <= a keeps the two free values inside the spread of the others (no gap in the chain)
    lo_x, hi_x = sd * sd / 16, a * a
    mid = a * a / 4
    m = len(d)
    for _ in range(steps):
        X = 2 * Q - R * R
        if X > 0:
            s = math.isqrt(X)
            if s * s == X:
                p, q = (R + s) // 2, (R - s) // 2
                if p != q and max(abs(p), abs(q)) <= lim and (not distinct or (p not in used and q not in used)):
                    vec = d + [p, q]
                    if max_gap is None or int(np.diff(np.sort(vec)).max()) <= max_gap:
                        return vec
        # paired move d_i += t, d_j -= t (R unchanged, X = (p - q) ** 2 changes by -4 t (d_i - d_j) - 4 t t); outside
        # its window X is steered back, with steps sized to the distance
        i, j = int(rng.integers(0, m)), int(rng.integers(0, m))
        if i == j:
            continue
        diff = d[i] - d[j]
        if lo_x <= X <= hi_x:
            t = 1 if rng.random() < 0.5 else -1
        else:
            t = max(1, int(abs(X - mid) / (8 * abs(diff) + 8)))
            if X < lo_x:   # shrink the others' sum of squares: t against diff, |t| <= |diff| / 2
                t = -min(t, max(1, abs(diff) // 2)) * (1 if diff > 0 else -1)
            elif diff < 0:  # grow it: t with diff
                t = -t
        ni, nj = d[i] + t, d[j] - t
        if abs(ni) > lim or abs(nj) > lim:
            continue
        if distinct and (ni in used or nj in used or ni == nj):
            continue
        if distinct:
            used.discard(d[i]); used.discard(d[j]); used.add(ni); used.add(nj)
        Q -= ni * ni + nj * nj - d[i] * d[i] - d[j] * d[j]
        d[i], d[j] = ni, nj
    return None


def _k_step(n):
    return 49 // math.gcd(49, n)    # smallest k with 49 | 25 k n


def _splits_differ(n):
    """numpy's split (n / 2 rounded down to a multiple of 8) and the plain n / 2 differ somewhere in the recursion."""
    if n <= 128:
        return False
    h = n // 2
    h8 = h - h % 8
    return h8 != h or _splits_differ(h8) or _splits_differ(n - h8)


def mutants_for(n):
    """The mutants an exact-boundary vector of n values can tell apart from numpy's order at all."""
    need = {"sequential", "pair4"}
    if n % 8 >= 2:
        need.add("tail_first")
    if n > 128:
        need.add("no_split")
        if _splits_differ(n):
            need.add("split_half")
    return need


# search seed per size (default 7): with seed 7 the budget finds no 2304-value vector that defeats the (r0+r4) pairing
SEEDS = {2304: 1}


@functools.lru_cache(maxsize=None)
def boundary_vectors(n, r, kind, seed=None, budget=None, keep=4):
    """Exact-boundary vectors of n values as planted (BASE + deviation): kind "pos" (any order) or "len" (distinct,
    ascending).  Returns ((values, frozenset(defeated mutants)), ...) with at most `keep` vectors: each kept one defeats a mutant no
    earlier kept vector defeats.  Fixed seed; at most `budget` vectors are built, fewer once every mutant of
    mutants_for(n) is defeated."""
    seed = SEEDS.get(n, 7) if seed is None else seed
    rng = np.random.default_rng([seed, n, r, 0 if kind == "pos" else 1])
    step = _k_step(n)
    target_sd = 100.0 if n < 1000 else 1100.0
    k0 = max(1, int(round(target_sd * 49 / (25 * math.sqrt(n)) / step))) * step
    budget = budget or (120 if n <= 256 else 80)
    need = mutants_for(n)
    out, covered = [], set()
    # sum(d * d) = sum(d) (mod 2) holds only for some k
    ks = [k for k in range(k0, k0 + 8 * step, step) if ((25 * k * n // 49) ** 2 + r * r // n - r) % 2 == 0]
    assert ks, (n, r)
    for _ in range(budget):
        if need <= covered:
            break
        k = ks[int(rng.integers(0, len(ks)))]
        d = _boundary_vector(rng, n, r, k, distinct=kind == "len", max_gap=POS_MAX_GAP if kind == "pos" else None)
        if d is None:
            continue
        v = sorted(d) if kind == "len" else list(rng.permutation(d))
        v = [BASE + int(x) for x in v]
        got = defeated(v)
        if (got & need) - covered:
            out.append((tuple(v), frozenset(got)))
            covered |= got
            if len(out) >= keep:
                break
    return tuple(out)


def tier_vectors(tier):
    """{(n, kind): vectors} of one tier."""
    return {(n, kind): boundary_vectors(n, r, kind) for n, r in TIERS[tier] for kind in ("pos", "len")}


# ---------------------------------------------------------------------------------------------------------------------
# planted layouts
# ---------------------------------------------------------------------------------------------------------------------
BOUNDARY_SIZES = (31, 32, 33, 63, 64, 65, 127, 128, 129, 2047, 2048, 2049, 4500)
PARAMS = dict(min_support=10, genotype=1)
SPACING = 20000       # between planted clusters: far more than any bias and any spread of a planted cluster
ALLELE_CONTIG_LEN = 300000   # contig of one exact-boundary allele: room for BASE + deviation + deletion length


class Layout(object):
    """Signature columns of each type built cluster by cluster on contig 0 (TRA mates on contig 1, exact-boundary alleles
    on contigs 2, 3, ...); every cluster gets reads of its own unless told otherwise."""

    def __init__(self, seed=0, contig_len=None, first=10000):
        self.rng = np.random.default_rng(seed)
        self.cols = {t: [] for t in ALL_TYPES}
        self.next_pos = first
        self.next_rid = 0
        self.read_rows = []      # (chrom, start, end, rids)
        self.n_allele_contigs = 0
        self.alleles = []        # exact-boundary alleles: dict(type, rids, pos, len)
        self.contig_len = contig_len

    def _base(self, spread):
        b = self.next_pos + spread
        self.next_pos = b + spread + SPACING
        return b

    def _rids(self, m, base, chrom=0):
        rids = np.arange(self.next_rid, self.next_rid + m, dtype=np.int32)
        self.next_rid += m
        self.read_rows.append((chrom, max(base - 6000, 0), base + 12000, rids))
        return rids

    def _add(self, t, chrom, a, b, rid, c=None):
        self.cols[t].append((np.asarray(chrom, np.int64), np.asarray(a, np.int64), np.asarray(b, np.int64),
                             np.asarray(rid, np.int64), None if c is None else np.asarray(c, np.int64)))

    def cluster(self, t, m, dup=0, shared_read=0, seq=None, span=80):
        """m signatures of type t within `span` bp (one chain cluster of exactly m members).  dup: the last `dup`
        signatures are exact copies of the first ones; shared_read: the last `shared_read` signatures reuse the reads of
        the first ones (other positions / lengths); seq (INS): None = long enough, "none" = no member's sequence is long
        enough, "last" = only the longest member's is."""
        rng = self.rng
        base = self._base(4 * span)
        rid = self._rids(m, base).copy()
        pos = base + rng.integers(0, span, m)
        if seq is not None:
            ln = 1000 + rng.permutation(m)            # one allele, distinct lengths: allele order = ascending length
        else:
            ln = np.where(rng.random(m) < 0.5, 300, 900) + rng.integers(-20, 20, m)
        for q in range(shared_read):
            rid[m - 1 - q] = rid[q]
        if t == "DEL":
            a, b, c = pos, ln, None
        elif t == "INS":
            a, b = 2 * pos + rng.integers(0, 2, m), ln
            c = ln.copy()
            if seq == "none":
                c[:] = ln.min() - 1
            elif seq == "last":
                c[:] = 0
                c[np.argmax(ln)] = ln.max()
        elif t == "DUP":
            a, b, c = pos, pos + 3000 + rng.integers(-20, 20, m), None
        elif t == "INV":
            a, b, c = pos, pos + 5000 + rng.integers(-20, 20, m), np.full(m, 1)
        else:
            a, b, c = pos, 50000 + rng.integers(0, 40, m), np.full(m, 4 * 1 + 0)
        a, b = np.asarray(a).copy(), np.asarray(b).copy()
        c = None if c is None else np.asarray(c).copy()
        for q in range(dup):
            a[m - 1 - q], b[m - 1 - q], rid[m - 1 - q] = a[q], b[q], rid[q]
            if c is not None:
                c[m - 1 - q] = c[q]
        self._add(t, np.zeros(m), a, b, rid, c)

    def allele(self, t, pos, ln):
        """One INS / DEL allele on a contig of its own: member i has position pos[i] and length ln[i] (values as returned
        by boundary_vectors); ln must be strictly ascending, so that the allele's order (ascending length, one read
        each) is i."""
        n = len(pos)
        pos = np.asarray(pos, np.int64)
        ln = np.asarray(ln, np.int64)
        assert len(ln) == n and np.all(np.diff(ln) > 0) and pos.min() > 0 and ln.min() > 0
        assert int(pos.max() + ln.max()) < ALLELE_CONTIG_LEN
        chrom = 2 + self.n_allele_contigs
        self.n_allele_contigs += 1
        rid = self._rids(n, BASE, chrom)
        if t == "DEL":
            self._add(t, np.full(n, chrom), pos, ln, rid)
        else:
            self._add(t, np.full(n, chrom), 2 * pos, ln, rid, ln)
        self.alleles.append(dict(type=t, rids=rid, pos=dict(zip(rid.tolist(), pos.tolist())),
                                 len=dict(zip(rid.tolist(), ln.tolist()))))

    def config(self, params=None):
        sigs = {}
        for t, parts in self.cols.items():
            if not parts:
                continue
            cat = [np.concatenate([p[f] for p in parts]) for f in range(4)]
            has_c = parts[0][4] is not None
            perm = self.rng.permutation(len(cat[0]))
            sigs[t] = dict(chrom=cat[0][perm].astype(np.int32), a=cat[1][perm].astype(np.int32), b=cat[2][perm].astype(np.int32),
                           read_id=cat[3][perm].astype(np.int32),
                           c=np.concatenate([p[4] for p in parts])[perm].astype(np.int32) if has_c else None)
        ch, st, en = (np.concatenate([np.full(len(row[3]), row[f]) for row in self.read_rows]) for f in range(3))
        rid = np.concatenate([row[3] for row in self.read_rows])
        rid, first = np.unique(rid, return_index=True)
        reads = dict(chrom=ch[first].astype(np.int32), start=st[first].astype(np.int32), end=en[first].astype(np.int32),
                     read_id=rid.astype(np.int32), is_primary=np.ones(len(rid), np.uint8))
        L = self.contig_len or self.next_pos + 100000
        lens = np.array([L, 200000] + [ALLELE_CONTIG_LEN] * self.n_allele_contigs, dtype=np.int64)
        return dict(lens=lens, sigs=sigs, reads=reads, params=dict(PARAMS if params is None else params), alleles=self.alleles)


GPU_LAYOUT_SEED = 11    # the layout of tests/test_gpu_cluster_tiers.py's route tests


def boundary_layout(seed=0, types=ALL_TYPES, sizes=None, min_support=PARAMS["min_support"], tiers=tuple(TIERS), params=None):
    """Every type: clusters of min_support and BOUNDARY_SIZES members, the straddle cases (33 with one exact duplicate,
    129 with two signatures of one read, 2049 with one duplicate), INS clusters without a long-enough sequence and with
    only the last member's, and one INS and one DEL allele per exact-boundary vector of the given tiers."""
    L = Layout(seed)
    sizes = (min_support,) + BOUNDARY_SIZES if sizes is None else sizes
    for t in types:
        for m in sizes:
            L.cluster(t, m)
        L.cluster(t, 33, dup=1)
        L.cluster(t, 129, shared_read=1)
        L.cluster(t, 2049, dup=1)
        if t == "INS":
            for m in (20, 100, 500, 2100):
                L.cluster(t, m, seq="none")
                L.cluster(t, m, seq="last")
    for tier in tiers:
        for (n, kind), vs in sorted(tier_vectors(tier).items()):
            if kind != "pos":
                continue
            lens_v = [v for v, _ in tier_vectors(tier)[(n, "len")]]
            pos_v = [v for v, _ in vs]
            for i in range(max(len(pos_v), len(lens_v))):
                pv = pos_v[i % len(pos_v)] if pos_v else BASE + L.rng.integers(0, 80, n)
                lv = lens_v[i % len(lens_v)] if lens_v else BASE + np.arange(n)
                for t in ("DEL", "INS"):
                    if t in types:
                        L.allele(t, pv, lv)
    p = dict(PARAMS if params is None else params)
    p["min_support"] = min_support
    return L.config(p)


# ---------------------------------------------------------------------------------------------------------------------
# expected counters: the chain split in numpy
# ---------------------------------------------------------------------------------------------------------------------
def chain_sizes(t, cols, lens, p):
    """Sizes of the chain clusters of one type: over the linear key for INS / DEL, over the reference's full sort order
    without exact duplicates for DUP / INV / TRA.  p: _abi.csv_params."""
    chrom = np.asarray(cols["chrom"], np.int64)
    if len(chrom) == 0:
        return np.zeros(0, np.int64), 0
    a = np.asarray(cols["a"], np.int64)
    b = np.asarray(cols["b"], np.int64)
    rid = np.asarray(cols["read_id"], np.int64)
    c = np.zeros(len(a), np.int64) if cols.get("c") is None else np.asarray(cols["c"], np.int64)
    if t in ("DEL", "INS"):
        pad = max(p.bias_del, p.bias_ins, p.bias_inv, p.bias_dup, p.bias_tra, p.gt_bias_ins) + 1
        off = np.concatenate([[0], np.cumsum(np.asarray(lens, np.int64) + pad)])
        key = np.sort(off[chrom] + (a >> 1 if t == "INS" else a))
        link = np.diff(key) <= (p.bias_ins if t == "INS" else p.bias_del)
        dom = len(key)
    else:
        ck = c if t in ("INV", "TRA") else np.zeros_like(c)
        o = np.lexsort((c, rid, b, a, ck, chrom))
        rows = np.stack([chrom[o], ck[o], a[o], b[o], rid[o], c[o]], 1)
        keep = np.ones(len(rows), bool)
        keep[1:] = np.any(rows[1:] != rows[:-1], axis=1)
        rows = rows[keep]
        dom = len(rows)
        bias = {"DUP": p.bias_dup, "INV": p.bias_inv, "TRA": p.bias_tra}[t]
        same = (rows[1:, 0] == rows[:-1, 0]) & (rows[1:, 1] == rows[:-1, 1])
        link = same & (np.diff(rows[:, 2]) <= bias)
        if t == "INV":
            link &= np.diff(rows[:, 3]) <= bias
    starts = np.concatenate([[0], np.nonzero(~link)[0] + 1, [len(link) + 1]])
    return np.diff(starts), dom


def expected_counters(cfg, p, types=ALL_TYPES, small_path=True):
    """kept / members / big (m > 128) / giant (m > 2048) per type and small_path (INS + DEL clusters of m <= 32 that the
    register kernel takes: every member kept and the small path on)."""
    out = dict(kept={}, members={}, big={}, giant={}, small_path=0)
    for t in ALL_TYPES:
        m = np.zeros(0, np.int64)
        if t in types and t in cfg["sigs"]:
            m, _ = chain_sizes(t, cfg["sigs"][t], cfg["lens"], p)
            m = m[m >= p.min_support]
        out["kept"][t] = int(len(m))
        out["members"][t] = int(m.sum())
        out["big"][t] = int((m > WARP_M).sum())
        out["giant"][t] = int((m > BLOCK_M).sum())
        if t in ("DEL", "INS") and small_path and p.remain_reads_ratio >= 1.0:
            out["small_path"] += int((m <= SMALL_M).sum())
    return out


def counters_view(ctr):
    """The part of Engine.counters() that expected_counters() predicts."""
    return dict(kept=dict(ctr["kept"]), members=dict(ctr["members"]), big=dict(ctr["big"]), giant=dict(ctr["giant"]),
                small_path=int(ctr["small_path"]))


def allele_cipos_errors(cfg, recs):
    """Every exact-boundary allele of cfg must appear as one record whose CIPOS / CILEN equal cal_CIPOS of np.std over
    the positions / lengths in the record's own `names` order.  Returns a list of messages (empty: all good)."""
    cands, _, names = recs
    first = {}
    for i in range(len(cands)):
        o, n = int(cands[i]["names_off"]), int(cands[i]["names_cnt"])
        if n:
            first.setdefault(int(names[o]), []).append(i)
    errs = []
    for al in cfg["alleles"]:
        want_t = _abi.TYPE_IDS[al["type"]]
        rids = set(al["rids"].tolist())
        hit = [i for r in rids for i in first.get(r, []) if int(cands[i]["svtype"]) == want_t]
        if len(hit) != 1:
            errs.append("%s allele of %d reads: %d records" % (al["type"], len(rids), len(hit)))
            continue
        c = cands[hit[0]]
        nm = names[int(c["names_off"]):int(c["names_off"]) + int(c["names_cnt"])].tolist()
        if nm != al["rids"].tolist():   # the order the vectors were chosen in
            errs.append("%s allele of %d reads: record names %d of them, in another order" % (al["type"], len(rids), len(set(nm) & rids)))
            continue
        pos = [al["pos"][r] for r in nm]
        ln = [al["len"][r] for r in nm]
        n = len(nm)
        want = (cal_cipos(float(np.std(pos)), n), cal_cipos(float(np.std(ln)), n))
        got = (int(c["cipos"]), int(c["cilen"]))
        if got != want:
            errs.append("%s allele n=%d: (cipos, cilen) %s, numpy %s" % (al["type"], n, got, want))
    return errs


def tier_of(n):
    for tier, sizes in TIERS.items():
        if any(n == m for m, _ in sizes):
            return tier
    return None


def planted_coverage(cfg):
    """{tier: mutants defeated by the positions or the lengths of a planted exact-boundary allele of cfg}, evaluated on the
    absolute values in allele order (the order the allele's record names its reads in)."""
    cov = {tier: set() for tier in TIERS}
    for al in cfg["alleles"]:
        rids = al["rids"].tolist()
        cov[tier_of(len(rids))] |= defeated([al["pos"][r] for r in rids]) | defeated([al["len"][r] for r in rids])
    return cov
