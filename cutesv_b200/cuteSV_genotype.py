"""Drop-ins for the reference's cuteSV_genotype helpers:

- cal_GL (cuteSV_genotype.py:33-56): special cases + rescale on the device (csv_cal_gl), the libm part from the host-built table.
- overlap_cover (:95-159): the device overlap/cover pass (csv_overlap_cover) over any window list and reads slice.
- assign_gt (:161-173): DR from the given sets on the host, cal_GL batched through csv_cal_gl.
- cal_CIPOS (:58-60) and threshold_ref_count (:62-70): host arithmetic, the same expressions.

count_coverage (:72-93) takes a pysam handle and fills the caller's name set, so it has no drop-in of its own; its one
caller, resolveTRA's call_gt, has one (cuteSV_resolveTRA.call_gt, csv_tra_call_gt), which scans a table of the records
decoded around its windows.
call_gt of resolveINDEL / resolveDUP / resolveINV uses call_gt_genos below (csv_call_gt)."""
import numpy as np

from . import _abi, rows, runtime

Genotype = ["0/0", "0/1", "1/1"]


def _gl_tuple(g, c0, c1):
    """(GT, "PL0,PL1,PL2", GQ, QUAL) of one csv_geno, typed like cal_GL's return value."""
    qual = float(g["qual"])
    return Genotype[int(g["gt"])], "%d,%d,%d" % (int(g["pl"][0]), int(g["pl"][1]), int(g["pl"][2])), int(g["gq"]), (
        qual if (c0, c1) in ((3, 1), (6, 2)) else np.float64(qual))


def cal_GL(c0, c1):
    """(GT, "PL0,PL1,PL2", GQ, QUAL) like cuteSV_genotype.py:33-56."""
    return _gl_tuple(runtime.get_engine().cal_gl([int(c0)], [int(c1)])[0], c0, c1)


def cal_GL_batch(c0, c1):
    return runtime.get_engine().cal_gl(c0, c1)


qual_str = rows.qual_str


def cal_CIPOS(std, num):
    pos = int(1.96 * std / num ** 0.5)
    return "-%d,%d" % (pos, pos)


def threshold_ref_count(num):
    if num <= 2:
        return 20 * num
    elif 3 <= num <= 5:
        return 9 * num
    elif 6 <= num <= 15:
        return 7 * num
    else:
        return 5 * num


def half_units(values):
    """Window bounds -> the half units of csv_window: 2v when v is a multiple of 0.5, otherwise 2*floor(v) + 1, which compares
    with the integer coordinates of reads rows exactly as v does."""
    a = np.asarray(values, dtype=np.float64)
    t = a * 2
    return np.where(t == np.floor(t), t, 2 * np.floor(a) + 1).astype(np.int64)


def first_key_error(s, e, start, end):
    """Index overlap_cover raises KeyError with, or None.  Its sweep removes an element at every right-hand event; a window with
    e <= s or a row with end < start reaches its right-hand event first.  The first such event in the sweep's order
    (coordinate, then sv-right 0 < read-right 2, then insertion order: rows before windows) decides."""
    cand = []
    br = np.flatnonzero(end < start)
    if len(br):
        i = int(br[np.lexsort((br, end[br]))[0]])
        cand.append(((float(end[i]), 2, 2 * i + 1), i))
    bw = np.flatnonzero(e <= s)
    if len(bw):
        j = int(bw[np.lexsort((bw, e[bw]))[0]])
        cand.append(((float(e[j]), 0, 2 * len(start) + 2 * j + 1), j))
    return min(cand)[1] if cand else None


def _bounds(svs_list):
    return (np.asarray([w[0] for w in svs_list], dtype=np.float64).reshape(-1), np.asarray([w[1] for w in svs_list], dtype=np.float64).reshape(-1))


def reads_columns(reads_list):
    """Reference reads rows [start, end, is_primary, name, ...] of one contig -> (reads columns on contig 0, id -> name list,
    name -> id dict).  Ids are first-seen ranks; only rows with is_primary == 1 count as primary, as in overlap_cover."""
    name_id = {}
    ids = np.fromiter((name_id.setdefault(r[3], len(name_id)) for r in reads_list), dtype=np.int32, count=len(reads_list))
    n = len(reads_list)
    cols = dict(chrom=np.zeros(n, np.int32), start=np.fromiter((r[0] for r in reads_list), dtype=np.int64, count=n).astype(np.int32),
                end=np.fromiter((r[1] for r in reads_list), dtype=np.int64, count=n).astype(np.int32), read_id=ids,
                is_primary=np.fromiter((r[2] == 1 for r in reads_list), dtype=np.uint8, count=n))
    return cols, list(name_id), name_id


def windows_of(s, e):
    """Window bounds -> csv_window array on contig 0."""
    return _abi.make_windows(np.zeros(len(s), np.int32), half_units(s), half_units(e))


def overlap_cover(svs_list, reads_list):
    """(iteration_dict, primary_num_dict, cover_dict, overlap_dict) like cuteSV_genotype.py:95-159: keyed by window index in the
    reference's key order, the last two holding Python sets of read names."""
    cols, names, _ = reads_columns(reads_list)
    s, e = _bounds(svs_list)
    bad = first_key_error(s, e, cols["start"], cols["end"])
    if bad is not None:
        raise KeyError(bad)
    if not svs_list:
        return {}, {}, {}, {}
    r = runtime.get_engine().overlap_cover(windows_of(s, e), cols)
    it, pn = r["iteration"].tolist(), r["primary_num"].tolist()
    co, ci, oo, oi = r["cover_off"].tolist(), r["cover_ids"].tolist(), r["overlap_off"].tolist(), r["overlap_ids"].tolist()
    iteration_dict, primary_num_dict, cover_dict, overlap_dict = {}, {}, {}, {}
    # keys in the order of the windows' left events: by s, ties by index
    for i in np.argsort(s, kind="stable").tolist():
        iteration_dict[i] = it[i]
        primary_num_dict[i] = pn[i]
        cover_dict[i] = {names[k] for k in ci[co[i]:co[i + 1]]}
        overlap_dict[i] = {names[k] for k in oi[oo[i]:oo[i + 1]]}
    return iteration_dict, primary_num_dict, cover_dict, overlap_dict


def assign_gt(iteration_dict, primary_num_dict, cover_dict, read_id_dict):
    """[[DV, DR, GT, GL, GQ, QUAL], ...] like cuteSV_genotype.py:161-173 (one cal_GL batch for all entries)."""
    dv, dr = [], []
    for idx in read_id_dict:
        iteration_dict[idx], primary_num_dict[idx]   # the reference reads both: a missing key raises KeyError
        sup = set(read_id_dict[idx])
        dr.append(sum(1 for q in cover_dict[idx] if q not in sup))
        dv.append(len(read_id_dict[idx]))
    if not dv:
        return []
    genos = runtime.get_engine().cal_gl(dr, dv)
    return [[dv[k], dr[k]] + list(_gl_tuple(genos[k], dr[k], dv[k])) for k in range(len(dv))]


def call_gt_genos(reads_list, svs_list, windows_per_cand, supports):
    """The genotype part of the resolvers' call_gt: svs_list in the reference's layout (all first windows, then all second
    windows), supports = every candidate's list of supporting read names.  Returns one csv_geno per candidate."""
    cols, _, name_id = reads_columns(reads_list)
    s, e = _bounds(svs_list)
    bad = first_key_error(s, e, cols["start"], cols["end"])
    if bad is not None:
        raise KeyError(bad)
    n = len(supports)
    order = np.arange(n * windows_per_cand).reshape(windows_per_cand, n).T.reshape(-1)   # candidate-major
    w = windows_of(s, e)[order]
    off = np.zeros(n + 1, np.int64)
    np.cumsum([len(sup) for sup in supports], out=off[1:])
    ids = np.fromiter((name_id.get(q, -1) for sup in supports for q in sup), dtype=np.int32, count=int(off[-1]))
    return runtime.get_engine().call_gt(w, windows_per_cand, off, ids, cols)


def geno_fields(g):
    """(DR, GT, GL, GQ, QUAL) strings of one call_gt row (str() of assign_gt's values)."""
    return (str(int(g["dr"])), Genotype[int(g["gt"])], "%d,%d,%d" % (int(g["pl"][0]), int(g["pl"][1]), int(g["pl"][2])), str(int(g["gq"])),
            qual_str(g["qual"]))
