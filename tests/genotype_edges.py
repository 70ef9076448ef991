"""Planted layouts for csv_cluster's genotype pass (k_permute -> k_scan_excl -> k_windows -> k_reads_pass -> k_pairs_test ->
k_finalize) at the edges where its kernels could go wrong without the whole-run parity tests noticing: rows that start or end
one base either side of a window bound, x.5 windows and windows clamped at 0, the DUP / INV union, every index of the
supporting-id scan, windows at bin and bin-map word edges, the shift and 32-bit-route thresholds of the linear coordinate,
the 1024-contig shared table, tile tails, and rows that run past their contig.

A case is built in two phases: its signatures are clustered once without reads (`cluster_fn`, the oracle or the library) to
read each candidate's windows, then the reads table is built relative to those windows.  Every planted candidate sits on a
contig of its own, so its rows touch no other window.  Each case also states the DR it plants per contig as a literal, so
that the three references (the oracle, `rule_genos` below and the standalone call_gt) cannot all be wrong the same way.

The linear coordinate (cutesv_b200.cu csv_set_contigs / enqueue_cluster): off[c] = sum over i < c of (len_i + pad) with
pad = max(six biases) + 1; shift = the smallest value >= 10 with total >> shift <= 2^20; a window is binned by
(off[c] + s) >> shift; the 32-bit pair route runs iff total + 4096 < 2^32.  Nothing here calls the library."""
import numpy as np

from cutesv_b200 import _abi

FRESH_ID = 1_000_000   # read ids of rows that support nothing
EMPTY_READS = dict(chrom=np.zeros(0, np.int32), start=np.zeros(0, np.int32), end=np.zeros(0, np.int32),
                   read_id=np.zeros(0, np.int32), is_primary=np.zeros(0, np.uint8))


# ---------------------------------------------------------------------------------------------------------------------
# the linear coordinate and the windows
# ---------------------------------------------------------------------------------------------------------------------
def pad_of(p):
    return max(p.bias_del, p.bias_ins, p.bias_inv, p.bias_dup, p.bias_tra, p.gt_bias_ins) + 1


def layout(p, lens):
    lens = np.asarray(lens, np.int64)
    pad = pad_of(p)
    off = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens + pad, out=off[1:])
    total = int(off[-1])
    shift = 10
    while (total >> shift) > (1 << 20):
        shift += 1
    return dict(pad=pad, off=off, total=total, shift=shift, n_bins=(total >> shift) + 2, lin32=total + 4096 < (1 << 32))


def windows_of_candidates(cands, p):
    """csv_cluster's genotype windows (call_gt of resolveINDEL.py:450-451, resolveDUP.py:146-151, resolveINV.py:218-221), half units."""
    t = cands["svtype"]
    w = np.zeros((len(cands), 2), dtype=_abi.WINDOW_DTYPE)
    w["chrom"] = cands["chrom"][:, None]
    b = np.where(t == _abi.CSV_INS, p.gt_bias_ins, p.bias_del).astype(np.int64)
    sp = cands["search_pos"].astype(np.int64)
    w["s2"][:, 0], w["e2"][:, 0] = 2 * np.maximum(sp - b, 0), 2 * (sp + b)
    nb = np.where(t == _abi.CSV_DUP, np.minimum(p.bias_dup, cands["pos2"].astype(np.int64) - cands["pos"]), p.bias_inv)
    for k, x in ((0, cands["pos"].astype(np.int64)), (1, cands["pos2"].astype(np.int64))):
        two = (t == _abi.CSV_DUP) | (t == _abi.CSV_INV)
        w["s2"][two, k], w["e2"][two, k] = np.maximum(2 * x - nb, 0)[two], (2 * x + nb)[two]
    return w


def n_windows(cands):
    t = cands["svtype"]
    return np.where((t == _abi.CSV_DEL) | (t == _abi.CSV_INS), 1, np.where((t == _abi.CSV_DUP) | (t == _abi.CSV_INV), 2, 0))


def int_bounds(w):
    """Integer bounds of a half-unit window: a row with integer ends covers it iff start <= s and end >= e."""
    return int(w["s2"]) // 2, (int(w["e2"]) + 1) // 2


# ---------------------------------------------------------------------------------------------------------------------
# the rule, stated with numpy
# ---------------------------------------------------------------------------------------------------------------------
def rule_dr(cands, names, reads, p):
    """DR per candidate: primary rows of the candidate's own contig with 2 * start <= s2 and 2 * end >= e2 for one of its
    windows (DUP / INV: the union of the two covers, a row counted once), less those whose read id supports the candidate.
    -1 where the candidate has no window, -2 where its contig has no rows at all (CSV_F_NO_READS)."""
    win = windows_of_candidates(cands, p)
    nw = n_windows(cands)
    ch = np.asarray(reads["chrom"])
    order = np.argsort(ch, kind="stable")
    bounds = np.searchsorted(ch[order], np.arange(int(cands["chrom"].max(initial=0)) + 2))
    rs2, re2 = 2 * np.asarray(reads["start"], np.int64), 2 * np.asarray(reads["end"], np.int64)
    dr = np.full(len(cands), -1, np.int64)
    for i in range(len(cands)):
        if nw[i] == 0:
            continue
        c = int(cands["chrom"][i])
        rows = order[bounds[c]:bounds[c + 1]]
        if not len(rows):
            dr[i] = -2
            continue
        rows = rows[np.asarray(reads["is_primary"])[rows] != 0]
        cov = np.zeros(len(rows), bool)
        for k in range(nw[i]):
            cov |= (rs2[rows] <= win["s2"][i, k]) & (re2[rows] >= win["e2"][i, k])
        sup = names[cands["names_off"][i]:cands["names_off"][i] + cands["names_cnt"][i]]
        cov &= ~np.isin(np.asarray(reads["read_id"])[rows], sup)
        dr[i] = int(cov.sum())
    return dr


def rule_genos(cands, names, reads, p, cal_gl):
    """The csv_geno records the rule gives: cal_GL(DR, DV) from `cal_gl` (the oracle's restatement), status 1 and DR -1
    where the contig has no rows; also the expected CSV_F_NO_READS mask."""
    dr = rule_dr(cands, names, reads, p)
    g = np.zeros(len(cands), _abi.GENO_DTYPE)
    for i in range(len(cands)):
        if dr[i] >= 0:
            g[i] = cal_gl(int(dr[i]), int(cands["names_cnt"][i]))
            g[i]["dr"], g[i]["dv"] = dr[i], cands["names_cnt"][i]
        else:
            g[i]["dr"], g[i]["dv"], g[i]["gt"], g[i]["status"] = -1, cands["names_cnt"][i], -1, 1
    return g, dr == -2


def diff_genos(want, got, fields=("dr", "dv", "gt", "pl", "gq", "status", "qual")):
    bad = []
    for k in fields:
        ne = np.flatnonzero(np.any(np.asarray(want[k]).reshape(len(want), -1) != np.asarray(got[k]).reshape(len(got), -1), axis=1))
        bad += ["%s differs at %s: want %s got %s" % (k, i, want[k][i], got[k][i]) for i in ne[:3]]
    return bad


def dr_by_contig(cands, genos):
    """{contig: total DR of its windowed candidates}, -1 where one has none (NO_READS)."""
    out = {}
    for i in np.flatnonzero(n_windows(cands) > 0):
        c, d = int(cands["chrom"][i]), int(genos["dr"][i])
        out[c] = -1 if d < 0 or out.get(c, 0) < 0 else out.get(c, 0) + d
    return out


# ---------------------------------------------------------------------------------------------------------------------
# building blocks
# ---------------------------------------------------------------------------------------------------------------------
def _sig(chrom, a, b, ids, c=None):
    n = len(ids)
    return dict(chrom=np.full(n, chrom, np.int32), a=np.full(n, a, np.int32), b=np.full(n, b, np.int32),
                read_id=np.asarray(ids, np.int32), c=None if c is None else np.full(n, c, np.int32))


def _cat(parts):
    out = {}
    for t in _abi.TYPE_NAMES:
        ps = [d for tt, d in parts if tt == t]
        if ps:
            out[t] = {k: (None if ps[0][k] is None else np.concatenate([d[k] for d in ps])) for k in ps[0]}
    return out


class Sigs(object):
    """Signature clusters of identical members: a DEL / INS at `pos`, a DUP from `pos` to `pos2`, an INV (strand 0)."""

    def __init__(self):
        self.parts, self.next_id = [], 1

    def _ids(self, k):
        ids = list(range(self.next_id, self.next_id + k))
        self.next_id += k
        return ids

    def dele(self, chrom, pos, length=300, k=3):
        self.parts.append(("DEL", _sig(chrom, pos, length, self._ids(k))))

    def ins(self, chrom, pos, length=300, k=3):
        self.parts.append(("INS", _sig(chrom, 2 * pos, length, self._ids(k), length)))

    def dup(self, chrom, pos, pos2, k=3):
        self.parts.append(("DUP", _sig(chrom, pos, pos2, self._ids(k))))

    def inv(self, chrom, pos, pos2, k=3):
        self.parts.append(("INV", _sig(chrom, pos, pos2, self._ids(k), 0)))

    def cols(self):
        return _cat(self.parts)


class Rows(object):
    def __init__(self):
        self.ch, self.st, self.en, self.rid, self.pr = [], [], [], [], []
        self.next_id = FRESH_ID

    def add(self, chrom, start, end, rid=None, primary=1):
        if rid is None:
            rid, self.next_id = self.next_id, self.next_id + 1
        self.ch.append(chrom); self.st.append(start); self.en.append(end); self.rid.append(rid); self.pr.append(primary)

    def bounds9(self, chrom, s, e):
        """Rows from s-1, s, s+1 to e-1, e, e+1 (starts below 0 left out); returns how many of them cover [s, e]."""
        n = 0
        for ds in (-1, 0, 1):
            for de in (-1, 0, 1):
                if s + ds >= 0:
                    self.add(chrom, s + ds, e + de)
                    n += ds <= 0 <= de
        return n

    def table(self):
        return dict(chrom=np.asarray(self.ch, np.int32), start=np.asarray(self.st, np.int32), end=np.asarray(self.en, np.int32),
                    read_id=np.asarray(self.rid, np.int32), is_primary=np.asarray(self.pr, np.uint8))


def on_contig(cands, chrom):
    i = np.flatnonzero((cands["chrom"] == chrom) & (n_windows(cands) > 0))
    assert len(i) == 1, (chrom, i)
    return int(i[0])


def supporters(cands, names, i):
    return names[cands["names_off"][i]:cands["names_off"][i] + cands["names_cnt"][i]]


class Case(object):
    """params, lens, sigs; reads(cands, names) -> reads table; planted {contig: DR} (-2: NO_READS) after reads() ran;
    edges(cands, names, reads) -> {edge name: bool}, every one of which the layout must hit."""

    def __init__(self, name, params, lens, sigs, reads, edges=None):
        self.name, self.params, self.lens, self.sigs = name, params, np.asarray(lens, np.int64), sigs
        self._reads, self._edges = reads, edges
        self.planted = {}

    def lay(self):
        return layout(self.params, self.lens)

    def reads(self, cands, names):
        self.planted = {}
        return self._reads(self, cands, names)

    def edges(self, cands, names, reads):
        return self._edges(self, cands, names, reads) if self._edges else {}


def build(case, cluster_fn):
    """The two phases: candidates without reads, then the reads table relative to their windows.  Returns the reads table."""
    cands, _, names = cluster_fn(case.params, case.lens, case.sigs, EMPTY_READS)
    return case.reads(cands, names)


def params(**kw):
    kw.setdefault("min_support", 2)
    kw.setdefault("genotype", 1)
    return _abi.default_params(**kw)


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------
def _bounds_rows(case, cands, names, contigs):
    """bounds9 around every window of the candidate on each contig; planted DR = the covering rows."""
    R = Rows()
    win = windows_of_candidates(cands, case.params)
    for c in contigs:
        i = on_contig(cands, c)
        n = 0
        for k in range(n_windows(cands[i:i + 1])[0]):
            s, e = int_bounds(win[i, k])
            n += R.bounds9(c, s, e)
        case.planted[c] = n
    return R


def window_bounds():
    """DEL, INS (gt_bias_ins, not bias_ins), DUP with pos2 - pos odd, even and above bias_dup, INV with an odd bias (x.5
    windows), windows clamped at 0 on contig 0 and on later contigs (an INV with 2x - nb < 0), and the DUP / INV union."""
    p = params(bias_inv=501, gt_bias_ins=1000, bias_ins=100)
    S = Sigs()
    S.dele(0, 150)              # clamped at 0 on contig 0
    S.dele(1, 50_000)
    S.ins(2, 50_000)
    S.ins(3, 700)               # clamped at 0 (gt_bias_ins 1000) on a later contig
    S.dup(4, 50_000, 50_301)    # odd: x.5 windows
    S.dup(5, 50_000, 50_300)    # even
    S.dup(6, 50_000, 54_000)    # above bias_dup
    S.inv(7, 50_000, 53_000)    # odd bias_inv
    S.inv(8, 200, 3_000)        # 2 * 200 - 501 < 0: first window clamped at 0
    S.dup(9, 50_000, 54_000)    # union
    S.inv(10, 50_000, 53_000)   # union

    def reads(case, cands, names):
        R = _bounds_rows(case, cands, names, range(9))
        win = windows_of_candidates(cands, case.params)
        for c in (9, 10):
            i = on_contig(cands, c)
            (s0, e0), (s1, e1) = int_bounds(win[i, 0]), int_bounds(win[i, 1])
            R.add(c, s0 - 5, e0 + 5)                  # only the first window
            R.add(c, s1 - 5, e1 + 5)                  # only the second
            R.add(c, s0 - 5, e1 + 5)                  # both: counted once
            R.add(c, s0 - 5, e1 + 5, rid=int(supporters(cands, names, i)[0]))   # a supporter covering both
            case.planted[c] = 3
        return R.table()

    def edges(case, cands, names, reads):
        win = windows_of_candidates(cands, case.params)
        i_dup = [on_contig(cands, c) for c in (4, 5, 6)]
        i_inv = on_contig(cands, 8)
        return {"x.5 start": win["s2"][i_dup[0], 0] % 2 == 1, "even DUP": (cands["pos2"] - cands["pos"])[i_dup[1]] % 2 == 0,
                "DUP above bias": (cands["pos2"] - cands["pos"])[i_dup[2]] > case.params.bias_dup,
                "INV x.5": case.params.bias_inv % 2 == 1 and win["e2"][i_inv, 1] % 2 == 1,
                "clamped contig 0": win["s2"][on_contig(cands, 0), 0] == 0, "clamped INS": win["s2"][on_contig(cands, 3), 0] == 0,
                "clamped x.5": 2 * int(cands["pos"][i_inv]) - case.params.bias_inv < 0 and win["s2"][i_inv, 0] == 0,
                "INS uses gt_bias_ins": win["e2"][on_contig(cands, 2), 0] - win["s2"][on_contig(cands, 2), 0] == 4 * case.params.gt_bias_ins}
    return Case("window_bounds", p, [100_000] * 11, S.cols(), reads, edges)


def names_scan():
    """names_cnt 1 .. 9 with the covering supporter at every index: the four-wide unrolled scan and its tail."""
    p = params(min_support=1, min_support_allele=1)
    S = Sigs()
    combos = [(k, j) for k in range(1, 10) for j in range(k)]
    for c, (k, _) in enumerate(combos):
        S.dele(c, 20_000, k=k)

    def reads(case, cands, names):
        R = Rows()
        win = windows_of_candidates(cands, case.params)
        for c, (k, j) in enumerate(combos):
            i = on_contig(cands, c)
            s, e = int_bounds(win[i, 0])
            sup = supporters(cands, names, i)
            assert len(sup) == k
            for m, r in enumerate(sup):
                R.add(c, s - 10 if m == j else s + 10, e + 10, rid=int(r))   # only supporter j covers
            R.add(c, s - 10, e + 10)                                          # one covering row that supports nothing
            case.planted[c] = 1
        return R.table()

    def edges(case, cands, names, reads):
        return {"names_cnt 1..9": sorted(set(cands["names_cnt"].tolist())) == list(range(1, 10))}
    return Case("names_scan", p, [50_000] * len(combos), S.cols(), reads, edges)


def bin_edges():
    """Window starts at k * 2^shift - 1, k * 2^shift and k * 2^shift + 1; windows at bit 0 and bit 31 of a bin-map word with
    rows whose bin range ends exactly there; long rows crossing empty map words to a window in their last or a middle word;
    a row in an occupied bin that covers nothing; a bin holding many windows."""
    p = params()
    lens = [400_000] * 9
    lay = layout(p, lens)
    off, sh = lay["off"], lay["shift"]
    bias = p.bias_del

    def del_at(S, c, lin_start):   # a DEL whose window starts at linear coordinate lin_start
        S.dele(c, int(lin_start - off[c]) + bias)

    def bin_after(c, x, mod=None):   # first bin of contig c past local coordinate x, optionally with bin % 32 == mod
        b = (int(off[c]) + x) >> sh
        while mod is not None and b % 32 != mod:
            b += 1
        return b

    S = Sigs()
    k0 = bin_after(0, 50_000)
    del_at(S, 0, (k0 << sh) - 1)
    del_at(S, 1, bin_after(1, 50_000) << sh)
    del_at(S, 2, (bin_after(2, 50_000) << sh) + 1)
    del_at(S, 3, (bin_after(3, 50_000, 0) << sh) + 10)     # bit 0
    del_at(S, 4, (bin_after(4, 50_000, 31) << sh) + 10)    # bit 31
    del_at(S, 5, (bin_after(5, 200_000, 31) << sh) + 10)   # bit 31, reached by a row from three words before
    del_at(S, 6, (bin_after(6, 200_000, 5) << sh) + 10)    # a middle word of a long row
    # many windows in one bin: DELs and INSs 300 bp apart (more than their biases), a DUP and an INV
    b7 = bin_after(7, 100_000, 7)
    base7 = int((b7 << sh) - off[7]) + 5
    for d in (0, 300, 600):
        S.dele(7, base7 + bias + d)
        S.ins(7, base7 + p.gt_bias_ins + d + 2)
    S.dup(7, base7 + 500, base7 + 50_000)
    S.inv(7, base7 + 900, base7 + 100_000)

    def reads(case, cands, names):
        R = Rows()
        win = windows_of_candidates(cands, case.params)
        for c in range(5):
            s, e = int_bounds(win[on_contig(cands, c), 0])
            R.add(c, s, e)                     # ends exactly at e: its bin range ends in the window's bin (c = 3, 4)
            R.add(c, s - 3, e + 1)
            R.add(c, s + 1, e + 50)            # starts inside: in an occupied bin, covers nothing
            case.planted[c] = 2
        s, e = int_bounds(win[on_contig(cands, 5), 0])
        R.add(5, s - 100 * (1 << sh), e)       # from three map words before, through empty words, ends in the window's bin
        R.add(5, s - 40 * (1 << sh), e + 3)
        case.planted[5] = 2
        s, e = int_bounds(win[on_contig(cands, 6), 0])
        R.add(6, s - 100 * (1 << sh), e + 100 * (1 << sh))   # the window is in a middle word of the row's range
        case.planted[6] = 1
        # contig 7: one row covers every window of the crowded bin (and the second windows of its DUP and INV)
        sel = np.flatnonzero(cands["chrom"] == 7)
        lo = min(int_bounds(win[i, 0])[0] for i in sel)
        hi = max(int_bounds(win[i, k])[1] for i in sel for k in range(n_windows(cands[i:i + 1])[0]))
        R.add(7, lo, hi)
        case.planted[7] = 8
        R.add(8, 10, 300_000)                 # a contig without windows
        return R.table()

    def edges(case, cands, names, reads):
        lay = case.lay()
        win = windows_of_candidates(cands, case.params)

        def lin_s(c):
            i = on_contig(cands, c)
            return int(lay["off"][c]) + int_bounds(win[i, 0])[0]

        def lin_e(c):
            i = on_contig(cands, c)
            return int(lay["off"][c]) + int_bounds(win[i, 0])[1]
        m = (1 << lay["shift"]) - 1
        out = {"start k*2^shift - 1": lin_s(0) & m == m, "start k*2^shift": lin_s(1) & m == 0, "start k*2^shift + 1": lin_s(2) & m == 1,
               "bit 0": (lin_s(3) >> lay["shift"]) % 32 == 0, "bit 31": (lin_s(4) >> lay["shift"]) % 32 == 31,
               "row ends in the bit-0 bin": lin_e(3) >> lay["shift"] == lin_s(3) >> lay["shift"],
               "row ends in the bit-31 bin": lin_e(4) >> lay["shift"] == lin_s(4) >> lay["shift"]}
        b5 = lin_s(5) >> lay["shift"]
        r5 = int(lay["off"][5] + reads["start"][reads["chrom"] == 5].min()) >> lay["shift"]
        out["long row crosses empty words to its last word"] = (b5 >> 5) - (r5 >> 5) >= 2 and lin_e(5) >> lay["shift"] == b5
        b6 = lin_s(6) >> lay["shift"]
        r6 = reads["chrom"] == 6
        out["window in a middle word"] = (int(lay["off"][6] + reads["start"][r6][0]) >> lay["shift"] >> 5) < (b6 >> 5) < \
            (int(lay["off"][6] + reads["end"][r6][0]) >> lay["shift"] >> 5)
        sel = np.flatnonzero(cands["chrom"] == 7)
        bins7 = {(int(lay["off"][7]) + int_bounds(win[i, 0])[0]) >> lay["shift"] for i in sel}
        out["a bin with many windows"] = len(bins7) == 1 and len(sel) >= 8
        return out
    c = Case("bin_edges", p, lens, S.cols(), reads, edges)
    return c


def _route_case(name, total):
    """A planted DEL / DUP / INV set on small contigs, then large empty contigs that bring the linear coordinate to `total`."""
    p = params(bias_inv=501)
    small = [100_000] * 3
    pad = pad_of(p)
    rest = total - sum(x + pad for x in small)
    big = []
    while rest > 0:
        take = min(rest, (1 << 31) - 1 + pad)
        big.append(take - pad)
        rest -= take
    S = Sigs()
    S.dele(0, 50_000)
    S.dup(1, 50_000, 50_301)
    S.inv(2, 50_000, 53_000)

    def reads(case, cands, names):
        R = _bounds_rows(case, cands, names, range(3))
        R.add(3, 0, 1000)    # a row on the first large contig
        return R.table()
    case = Case(name, p, small + big, S.cols(), reads)
    assert case.lay()["total"] == total
    return case


ROUTES = {   # name -> (total linear length, shift, 32-bit route)
    "shift10_top": ((1 << 30) + 1023, 10, True), "shift11_bottom": ((1 << 30) + 1024, 11, True),
    "shift11_top": ((1 << 31) + 2047, 11, True), "shift12_bottom": ((1 << 31) + 2048, 12, True),
    "lin32_top": ((1 << 32) - 4097, 12, True), "lin64_bottom": ((1 << 32) - 4096, 12, False),
}


def route_case(name):
    return _route_case(name, ROUTES[name][0])


def contig_table():
    """Candidates on contigs 1022 .. 1025 and 1099 (the shared-memory table holds contigs below 1024; the others take the global
    has_rows path), a contig whose rows are all secondary (DR 0, not NO_READS) and contigs with candidates and no rows."""
    p = params()
    S = Sigs()
    with_rows = (3, 1022, 1023, 1024, 1025, 1099)
    for c in with_rows + (5, 7, 1050):
        S.dele(c, 5_000)

    def reads(case, cands, names):
        R = Rows()
        win = windows_of_candidates(cands, case.params)
        for c in with_rows:
            s, e = int_bounds(win[on_contig(cands, c), 0])
            R.add(c, s - 1, e + 1)
            R.add(c, s, e)
            R.add(c, s + 1, e)
            case.planted[c] = 2
        s, e = int_bounds(win[on_contig(cands, 5), 0])
        R.add(5, s - 1, e + 1, primary=0)
        R.add(5, 0, 9_000, primary=0)
        case.planted[5] = 0
        case.planted[7] = case.planted[1050] = -2
        R.add(1070, 0, 9_000)   # rows on a contig without candidates
        return R.table()

    def edges(case, cands, names, reads):
        ch = set(cands["chrom"].tolist())
        return {"contig 1023": 1023 in ch, "contig 1024": 1024 in ch, "contig past 1024": 1099 in ch}
    return Case("contig_table", p, [10_000] * 1100, S.cols(), reads, edges)


TILE_SIZES = (4 * 900, 4 * 900 + 1, 4 * 900 + 3, 1024 * 3 - 1, 1024 * 3, 1024 * 3 + 1)


def tiles(n_reads):
    """window_bounds' rows inside `n_reads` rows: filler rows on a contig without windows, half of the planted rows in the
    middle and half at the end with zero-length rows (tiles of 1024 rows, four per thread; the tail tile takes the strided
    mapping)."""
    base = window_bounds()
    lens = list(base.lens) + [100_000]
    filler_c = len(lens) - 1

    def reads(case, cands, names):
        planted = base.reads(cands, names)
        case.planted = dict(base.planted)
        win = windows_of_candidates(cands, case.params)
        R = Rows()
        for c in (1, 4):   # zero-length rows at a window's bounds
            s, e = int_bounds(win[on_contig(cands, c), 0])
            R.add(c, e, e)
            R.add(c, s, s)   # last row of the table: starts in the window's bin, so it makes pairs in the tail tile
        extra = R.table()
        n_fill = n_reads - len(planted["chrom"]) - len(extra["chrom"])
        assert n_fill > 0
        rng = np.random.default_rng(n_reads)
        st = rng.integers(0, 90_000, n_fill).astype(np.int32)
        fill = dict(chrom=np.full(n_fill, filler_c, np.int32), start=st, end=st + rng.integers(0, 5000, n_fill).astype(np.int32),
                    read_id=np.arange(2 * FRESH_ID, 2 * FRESH_ID + n_fill, dtype=np.int32), is_primary=np.ones(n_fill, np.uint8))
        # half of the planted rows inside full tiles, the other half (and the zero-length rows) last: they make pairs in the
        # tail tile, which takes the strided mapping when n_reads is not a multiple of 1024
        half = len(planted["chrom"]) // 2
        return {k: np.concatenate([fill[k][:n_fill // 2], planted[k][:half], fill[k][n_fill // 2:], planted[k][half:], extra[k]])
                for k in fill}
    return Case("tiles_%d" % n_reads, base.params, lens, base.sigs, reads)


def overhang():
    """Rows of contig 0 that run past its end by pad - 1, pad and pad + the end of the first window of contig 1 (BAM allows
    reference_end past the contig's length).  In the linear coordinate the last two reach contig 1's windows; a row counts
    only on its own contig."""
    p = params(bias_del=1000, gt_bias_ins=1000)
    L = 100_000
    S = Sigs()
    S.dele(0, L - 500)     # window [L - 1500, L + 500]: covered by all three rows
    S.dele(1, 1_500)       # window [500, 2500]

    def reads(case, cands, names):
        pad = pad_of(case.params)
        win = windows_of_candidates(cands, case.params)
        i1 = on_contig(cands, 1)
        e1 = int_bounds(win[i1, 0])[1]
        R = Rows()
        for r in supporters(cands, names, i1):
            R.add(1, 0, 5_000, rid=int(r))
        R.add(1, 0, 5_000)
        for over in (pad - 1, pad, pad + e1):
            R.add(0, 90_000, L + over)
        case.planted[0], case.planted[1] = 3, 1
        return R.table()

    def edges(case, cands, names, reads):
        lay = case.lay()
        win = windows_of_candidates(cands, case.params)
        s1 = int(lay["off"][1]) + int_bounds(win[on_contig(cands, 1), 0])[0]
        ends = lay["off"][0] + reads["end"][reads["chrom"] == 0].astype(np.int64)
        return {"row reaches contig 1's window": bool((ends >= s1).any()), "row ends at pad - 1": int(ends.min()) == lay["off"][1] - 1}
    return Case("overhang", p, [L, L], S.cols(), reads, edges)


def all_cases():
    return [window_bounds(), names_scan(), bin_edges(), contig_table(), overhang()] + [route_case(n) for n in ROUTES]


# ---------------------------------------------------------------------------------------------------------------------
# TRA: count_coverage over the BAM-order all-alignments table (k_tra_genotype's warp steps)
# ---------------------------------------------------------------------------------------------------------------------
def py_count_coverage(recs, s, e, sup, up_bound, itround, acc, xs, xe):
    """count_coverage (cuteSV_genotype.py:72-93) as a plain loop over one contig's records (start, end, read id, primary) in
    BAM order: fetch(s, e) yields the records with start < e and end > s.  acc = [nset, dr] accumulates; a third entry, if
    present, receives the index in `recs` of the record that returns."""
    it = pr = 0
    for k, (st, en, rid, prim) in enumerate(recs):
        if len(acc) > 2:
            acc[2] = k
        if st >= e:
            break
        if en <= s:
            continue
        it += 1
        if not prim:
            continue
        pr += 1
        if st < s and en > e:
            if not (xs <= xe and st < xs and en > xe):
                acc[0] += 1
                acc[1] += rid not in sup
            if acc[0] >= up_bound:
                return 1
        if it >= itround:
            return 1 if pr / it <= 0.2 else -1
    return 0


def py_tra_dr(cand, sup, aln, p, lens):
    """call_gt of resolveTRA.py:260-309: DR of a TRA candidate, or -1 when the region is too noisy ('.', status 2)."""
    chr1, chr2 = int(cand["chrom"]), int(cand["aux"]) >> 2
    n = len(sup)
    up = 20 * n if n <= 2 else 9 * n if n <= 5 else 7 * n if n <= 15 else 5 * n
    recs = {c: [(int(a), int(b), int(r), bool(q)) for ch, a, b, r, q in zip(aln["chrom"], aln["start"], aln["end"], aln["read_id"],
                                                                          aln["is_primary"]) if ch == c] for c in {chr1, chr2}}
    sup = set(int(x) for x in sup)
    acc = [0, 0]
    s, e = max(int(cand["pos"]) - p.bias_tra, 0), min(int(cand["pos"]) + p.bias_tra, int(lens[chr1]))
    st = py_count_coverage(recs[chr1], s, e, sup, up, p.gt_round, acc, 1, 0)
    if st == -1:
        return -1
    if st == 0:
        s2, e2 = max(int(cand["pos2"]) - p.bias_tra, 0), min(int(cand["pos2"]) + p.bias_tra, int(lens[chr2]))
        py_count_coverage(recs[chr2], s2, e2, sup, up, p.gt_round, acc, s, e) if chr2 == chr1 else \
            py_count_coverage(recs[chr2], s2, e2, sup, up, p.gt_round, acc, 1, 0)
    return acc[1]


def tra_genos(cands, names, aln, p, lens, cal_gl):
    """The csv_geno of every TRA candidate by py_tra_dr and cal_GL; {contig: DR} of them (-1: '.')."""
    sel = np.flatnonzero(cands["svtype"] == _abi.CSV_TRA)
    g = np.zeros(len(sel), _abi.GENO_DTYPE)
    by = {}
    for k, i in enumerate(sel):
        sup = supporters(cands, names, i)
        dr = py_tra_dr(cands[i], sup, aln, p, lens)
        if dr < 0:
            g[k]["dr"], g[k]["dv"], g[k]["gt"], g[k]["status"] = -1, len(sup), -1, 2
        else:
            g[k] = cal_gl(dr, len(sup))
            g[k]["dr"], g[k]["dv"] = dr, len(sup)
        by[int(cands["chrom"][i])] = dr
    return sel, g, by


class TraCase(object):
    """TRA candidates of one supporter each (up_bound = threshold_ref_count(1) = 20), one per contig; aln(cands, names) builds
    the all-alignments table around their windows and fills `planted` {contig: DR, -1 for '.'}; `lanes` {spot: (contig, lane
    of the record that returns, 32-record step)} for the CPU test's layout check."""

    def __init__(self, name, params, lens, sigs, aln):
        self.name, self.params, self.lens, self.sigs, self._aln = name, params, np.asarray(lens, np.int64), sigs, aln
        self.planted, self.lanes = {}, {}

    def aln(self, cands, names):
        self.planted, self.lanes = {}, {}
        recs = self._aln(self, cands, names)
        ch = np.array([r[0] for r in recs], np.int32)
        st = np.array([r[1] for r in recs], np.int32)
        order = np.lexsort((np.arange(len(recs)), st, ch))
        cols = dict(chrom=ch, start=st, end=np.array([r[2] for r in recs], np.int32), read_id=np.array([r[3] for r in recs], np.int32),
                    is_primary=np.array([r[4] for r in recs], np.uint8))
        return {k: v[order] for k, v in cols.items()}


def build_tra(case, cluster_fn):
    cands, _, names = cluster_fn(case.params, case.lens, case.sigs, EMPTY_READS)
    return case.aln(cands, names)


def _tra_sigs(spots, last):
    """spot -> (chr1, pos, chr2, pos2); one supporter each, read ids 1, 2, ..."""
    cols = {k: [] for k in ("chrom", "a", "b", "read_id", "c")}
    for k, (c1, pos, c2, pos2) in enumerate(spots.values()):
        for f, v in zip(cols, (c1, pos, pos2, k + 1, (last if c2 is None else c2) * 4)):
            cols[f].append(v)
    return {"TRA": {f: np.asarray(v, np.int32) for f, v in cols.items()}}


def _tra_window(cands, c, p, lens, which=0):
    i = int(np.flatnonzero((cands["svtype"] == _abi.CSV_TRA) & (cands["chrom"] == c))[0])
    x = int(cands["pos2" if which else "pos"][i])
    cc = c if not which else int(cands["aux"][i]) >> 2
    return i, max(x - p.bias_tra, 0), min(x + p.bias_tra, int(lens[cc]))


TRA_UP_LANES = {"up_lane31": 31, "up_next_lane0": 32, "up_step1_lane31": 63, "up_step2_lane0": 64}


def tra_steps():
    """gt_round 500.  up_bound (20) reached by the record at index 31, 32, 63 and 64 of the scan (lanes 31 and 0 of
    consecutive 32-record steps), with the supporter spanning first (counted in the set, not in DR) and spanning records after
    the one that returns; an intra-contig pair whose second window's spanning reads are already in the set; windows clamped at
    0 and at the contig length; a first record found exactly at the max_span lower bound."""
    p = params(min_support=1, min_support_allele=1)
    L = 100_000
    spots = {name: (k, 50_000, None, 50_000) for k, name in enumerate(TRA_UP_LANES)}
    spots.update(intra=(4, 50_000, 4, 50_300), clamp0=(5, 30, 6, 50_000), clamp_len=(7, L - 30, None, 50_000),
                 max_span=(8, 50_000, None, 50_000))
    last = 9

    def aln(case, cands, names):
        recs = []
        fresh = iter(range(FRESH_ID, 2 * FRESH_ID))
        for k, (name, idx) in enumerate(TRA_UP_LANES.items()):
            i, s, e = _tra_window(cands, k, p, case.lens)
            sup = int(supporters(cands, names, i)[0])
            n_fill = idx - 19
            recs += [(k, s - 100, s - 50, next(fresh), 1) for _ in range(n_fill)]   # end <= s: not fetched, but scanned
            recs.append((k, s - 20, e + 20, sup, 1))                                # the supporter: in the set, not in DR
            recs += [(k, s - 20, e + 20, next(fresh), 1) for _ in range(19 + 5)]   # the 20th spanning record returns
            case.planted[k] = 19
            case.lanes[name] = (k, idx % 32, idx // 32)
        i, s, e = _tra_window(cands, 4, p, case.lens)
        _, s2, e2 = _tra_window(cands, 4, p, case.lens, 1)
        recs += [(4, s - 50, e2 + 50, next(fresh), 1), (4, s - 50, e + 50, next(fresh), 1), (4, s2 - 50, e2 + 50, next(fresh), 1)]
        case.planted[4] = 3
        i, s, e = _tra_window(cands, 5, p, case.lens)
        _, s2, e2 = _tra_window(cands, 5, p, case.lens, 1)
        recs += [(5, 0, e + 100, next(fresh), 1), (6, s2 - 10, e2 + 10, next(fresh), 1), (6, s2 - 10, e2 + 10, next(fresh), 1)]
        case.planted[5] = 2
        i, s, e = _tra_window(cands, 7, p, case.lens)
        recs += [(7, s - 10, L + 10, next(fresh), 1), (7, s - 10, L + 25, next(fresh), 1)]   # end > e only with e clamped at L
        case.planted[7] = 2
        i, s, e = _tra_window(cands, 8, p, case.lens)
        span = (e + 5) - (s - 600)
        recs += [(8, s - span - 1, s - span + 10, next(fresh), 1), (8, s - span, s - span + 20, next(fresh), 1),
                 (8, s - 600, e + 5, next(fresh), 1)]
        case.planted[8] = 1
        return recs
    return TraCase("tra_steps", p, [L] * (last + 1), _tra_sigs(spots, last), aln)


def tra_rounds():
    """gt_round 20: the round reached on a secondary record (4 primaries of 20: no return until the next primary, 5 of 21:
    '.'), primary / iteration exactly 0.2 (returns 1), and up_bound and the round reached on the same record (1 wins)."""
    p = params(min_support=1, min_support_allele=1, gt_round=20)
    spots = dict(round_secondary=(0, 50_000, None, 50_000), exact=(1, 50_000, None, 50_000), both=(2, 50_000, None, 50_000))
    last = 3

    def aln(case, cands, names):
        recs = []
        fresh = iter(range(FRESH_ID, 2 * FRESH_ID))
        _, s, e = _tra_window(cands, 0, p, case.lens)
        recs += [(0, s + 1, e + 20, next(fresh), int(j < 4 or j == 20)) for j in range(21)]
        case.planted[0] = -1
        _, s, e = _tra_window(cands, 1, p, case.lens)
        recs += [(1, s - 20, e + 20, next(fresh), 1) for _ in range(3)]
        recs += [(1, s + 1, e + 20, next(fresh), int(j == 16)) for j in range(17)]
        case.planted[1] = 3
        _, s, e = _tra_window(cands, 2, p, case.lens)
        recs += [(2, s - 20, e + 20, next(fresh), 1) for _ in range(25)]
        case.planted[2] = 20
        return recs
    return TraCase("tra_rounds", p, [100_000] * (last + 1), _tra_sigs(spots, last), aln)


def tra_cases():
    return [tra_steps(), tra_rounds()]
