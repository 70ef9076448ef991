"""Stores what the UNMODIFIED reference's signature phases compute (tests/golden/sigs_dropin.json.gz):

  single_pipe                 every task window of the cases of tests/sigs_dropin_data.py, read through tests/fake_pysam, the
                              windows spread over three fixed fake worker pids: the lists each call appends per type
  process_process_sigs_type   over the three pids' pickles, with write_old_sigs: the rebuilt per-contig lists, the index keys,
                              reads_count and the .sigs text of every type
  run_del .. run_tra          the clustering phase on that work dir (tests/sigs_dropin_data.py resolve_calls): the rows

The cases must contain exact duplicates across pids, INS ties broken by sequence, x.5 INS positions next to integer ones,
-include_bed, -p -1 (at most 64 segments per record), all five types on several contigs and a draft assembly of more than
32 768 contigs; the generator checks each of these.

Needs the reference (ref_harness.py):  CUTESV_REF_SRC=<cuteSV checkout>/src python -m oracle.gen_sigs_dropin_golden
"""
import gzip
import json
import os
import pickle
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_harness  # noqa: E402
import sigs_dropin_data as D  # noqa: E402


class _Proc(object):
    pid = 0


def run_case(main, case):
    ds, tasks, bed = D.dataset(case)
    out = dict(name=case["name"], tasks=tasks, task_pid=[D.PIDS[i % len(D.PIDS)] for i in range(len(tasks))], bed=bed, windows=[])
    with tempfile.TemporaryDirectory() as d:
        tmp = d + "/"
        os.mkdir(tmp + "signatures")
        bam = tmp + "in.bam"
        D.write_fake_bam(bam, ds)
        main.init_reading_process(bam, None)
        proc = _Proc()
        main.current_process = lambda: proc   # fixed fake worker pids
        for i, task in enumerate(tasks):
            proc.pid = out["task_pid"][i]
            main.single_pipe(*D.task_args(case, tmp, task, None if bed is None else bed[i]))
            out["windows"].append({t: D.read_pid_dumps("%ssignatures/%s%s.pickle" % (tmp, proc.pid, t))[-1] for t in D.TYPES})
        main.cleanup()
        out["rebuilt"], out["index_keys"], out["reads_count"], out["sigs_text"] = {}, {}, {}, {}
        sigs_index = {}
        for t in D.TYPES:
            sv, index, rc = main.process_process_sigs_type((t, tmp, list(D.PIDS), True))
            assert sv == t
            sigs_index[t] = index
            if t == "reads":
                sigs_index["reads_count"] = rc
            with open("%s/%s.pickle" % (tmp, t), "rb") as f:
                per = []
                for chrom, off in index.items():
                    f.seek(off)
                    per.append([chrom, pickle.load(f)])
            out["rebuilt"][t] = per
            out["index_keys"][t] = list(index)
            out["reads_count"][t] = rc
            with open("%s/%s.sigs" % (tmp, t)) as f:
                out["sigs_text"][t] = f.read()
        # the reference's clustering phase on the rebuilt work dir (cuteSV:1113-1199, run serially)
        mods = ref_harness.modules()
        run = {"DEL": mods["indel"].run_del, "INS": mods["indel"].run_ins, "INV": mods["inv"].run_inv, "DUP": mods["dup"].run_dup,
               "TRA": mods["tra"].run_tra}
        out["resolved"] = [[t, chrom, list(run[t](args))] for t, chrom, args in D.resolve_calls(tmp, sigs_index)]
    return out, ds


def check(case, g, ds):
    """The situations the goldens must contain (asserted, so a change of the seeds cannot drop one silently)."""
    seen = {}
    n_cat = {t: sum(len(w[t]) for w in g["windows"]) for t in D.TYPES}
    n_out = {t: sum(len(v) for _, v in g["rebuilt"][t]) for t in D.TYPES}
    seen["dedup"] = any(n_out[t] < n_cat[t] for t in D.TYPES if t != "reads")
    pid_of = {}
    cross = False
    for w, pid in zip(g["windows"], g["task_pid"]):
        for t in ("DEL", "DUP", "INV", "TRA"):
            for x in w[t]:
                k = (t, tuple(x))
                if k in pid_of and pid_of[k] != pid:
                    cross = True
                pid_of.setdefault(k, pid)
    seen["cross_pid_duplicates"] = cross
    ins = [x for _, v in g["rebuilt"]["INS"] for x in v]
    seen["ins_tie_by_sequence"] = any(a[-1] == b[-1] and int(a[0]) == int(b[0]) and a[1:3] == b[1:3] and a[3] != b[3]
                                      for a, b in zip(ins, ins[1:]))
    seen["ins_half_next_to_int"] = any(isinstance(a[0], float) and a[0] % 1 == 0.5 for a in ins) and any(isinstance(a[0], int) for a in ins)
    seen["types_on_contigs"] = {t: len(g["rebuilt"][t]) for t in D.TYPES}
    seen["n_contigs"] = len(ds["contigs"])
    seen["max_sa_segments"] = max((len(tag[1].split(";")) - 1 for r in ds["reads"] for tag in r.get_tags() if tag[0] == "SA"), default=0)
    return seen


def main():
    m = ref_harness.modules()["main"]
    cases, seen = [], {}
    for case in D.CASES:
        g, ds = run_case(m, case)
        seen[case["name"]] = check(case, g, ds)
        cases.append(g)
    s3, s5, dr = seen["mixed_s3"], seen["bed_split_all_s5"], seen["draft_33k"]
    assert s3["dedup"] and s3["cross_pid_duplicates"], s3
    assert s3["ins_tie_by_sequence"], s3
    assert s3["ins_half_next_to_int"] or s5["ins_half_next_to_int"], (s3, s5)
    assert all(s3["types_on_contigs"][t] >= 2 for t in D.TYPES), s3
    assert D.CASES[1]["bed"] and D.CASES[1]["params"]["max_split_parts"] == -1 and s5["max_sa_segments"] + 1 <= 64, s5
    assert dr["n_contigs"] > 32768, dr
    blob = json.dumps(dict(cases=cases), separators=(",", ":")) + "\n"
    with open(D.GOLDEN, "wb") as f, gzip.GzipFile(fileobj=f, mode="wb", mtime=0, filename="") as z:   # mtime 0: reproducible bytes
        z.write(blob.encode())
    print("wrote %s (%d bytes)" % (D.GOLDEN, os.path.getsize(D.GOLDEN)))
    for k, v in seen.items():
        print(k, v)


if __name__ == "__main__":
    main()
