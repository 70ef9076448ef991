"""Extraction goldens of the planted edge layouts (tests/extract_edges.py) from the REAL reference's parse_read (cuteSV:606-681),
under every parameter set of extract_edges.PARAMS.  Only the reference's output tuples are committed; the records are rebuilt
from the builder's seeds.  Authoring container only:  python -m oracle.gen_extract_edges_golden"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import extract_edges  # noqa: E402
from oracle import ref_harness  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "extract_edges.json")


def reference(case, pname):
    c, r = ref_harness.run_parse_reads(case["reads"], extract_edges.params(pname))
    return dict(candidate={k: [list(t) for t in v] for k, v in c.items()}, rows=[list(t) for t in r])


def main():
    out = dict(params=extract_edges.PARAMS, cases={})
    for name in extract_edges.CASES:
        case = extract_edges.case(name)
        out["cases"][name] = {pname: reference(case, pname) for pname in extract_edges.PARAMS}
        print(name, {p: {k: len(v) for k, v in g["candidate"].items() if v} for p, g in out["cases"][name].items()})
    with open(OUT, "w") as f:
        json.dump(out, f, sort_keys=True)


if __name__ == "__main__":
    main()
