"""CPU: the planted edge layouts of k_extract (tests/extract_edges.py) hit the edges they are named for, their literals equal the
REAL reference's parse_read (tests/golden/extract_edges.json, oracle/gen_extract_edges_golden.py), and the emulator
(extract_core.h through tests/emul) equals the golden record by record, in parse_read's order within each record."""
import collections
import json
import os

import pytest

import device_packet_util as dpu
import emul_lib
import extract_edges as E
import golden_util
from oracle import compare_extract, ref_harness

_GOLDEN = None


def golden(name, pname):
    global _GOLDEN
    if _GOLDEN is None:
        with open(os.path.join(golden_util.GOLDEN, "extract_edges.json")) as f:
            _GOLDEN = json.load(f)
    assert _GOLDEN["params"][pname] == E.PARAMS[pname]
    g = _GOLDEN["cases"][name][pname]
    return {k: [tuple(t) for t in v] for k, v in g["candidate"].items()}, [tuple(t) for t in g["rows"]]


def emulated(c, pname):
    p = E.params(pname)
    ex = emul_lib.extract(p, c["pk"])
    return ex, compare_extract.tuples_from_columns(ex, c["names"], c["rnames"], lambda rec: c["reads"][rec].query_sequence,
                                                   dpu.cigar_of_packet(c["pk"]), (p.min_siglength, p.merge_ins_threshold))


def _by_label(c):
    return {info["label"]: info for info in c["records"] if info["label"]}


def _hits(info):
    return {s["i"]: s for s in info["sigs"]}


def test_lengths_case_hits_every_length_d0_and_index():
    c = E.case("lengths")
    recs = _by_label(c)
    seen = collections.defaultdict(set)
    for info in recs.values():
        assert info["n_ops"] == info["L"] and info["cigar_off"] % 4 == info["d0"]
        seen[info["L"]].add(info["d0"])
        L, hits = info["L"], _hits(info)
        if L == 1:
            assert set(hits) == {0}
            continue
        want = {1} | {i for i in E.EDGE_IDX if i < L - (info["shape"] == "clip")}
        want.add(L - 2 if info["shape"] == "clip" else L - 1)
        assert set(hits) == want, info["label"]
        ops = c["reads"][info["rec"]].cigartuples
        if info["shape"] == "clip":
            assert ops[0][0] == E.S and ops[-1][0] == E.S
        else:
            assert ops[0][0] == E.H and ops[-1][0] in (E.I, E.D)
        for i, s in hits.items():
            assert (s["tile"], s["lane"], s["item"], s["chunk"], s["slot"]) == (i // 256, i % 256 // 8, i % 8, i // 512, i // 512 % 2)
        # adjacent qualifying ops are one I and one D: no merge under the defaults
        for i in hits:
            if i + 1 in hits:
                assert {hits[i]["kind"], hits[i + 1]["kind"]} == {"INS", "DEL"}
    assert seen == {L: {0, 1, 2, 3} for L in E.LENGTHS}
    # every edge index at every d0, as an I and as a D
    at = collections.defaultdict(set)
    for s in E.planted(c):
        at[s["i"]].add((s["d0"], s["kind"]))
    for i in E.EDGE_IDX:
        assert at[i] == {(d, k) for d in range(4) for k in ("INS", "DEL")}, i
    # the fillers in front of planted records: 1-3 ops, and every skip rule among them
    fill = [x for x in c["records"] if not x["label"]]
    assert {x["n_ops"] for x in fill} == {1, 2, 3}
    assert {(x["flag"], x["mapq"] < 20) for x in fill} >= {(256, False), (272, False), (0, True), (16, False)}
    assert any(c["reads"][x["rec"]].query_length < 500 for x in fill)


def test_lanes_case_fills_every_lane_and_one_lane_with_four():
    c = E.case("lanes")
    for info in c["records"]:
        if not info["label"]:
            continue
        tile = collections.defaultdict(set)
        for s in info["sigs"]:
            tile[s["tile"]].add((s["lane"], s["item"]))
        if info["label"].startswith("every_lane"):
            assert tile[1] == {(lane, it) for lane in range(32) for it in (0, 7)}
        else:
            assert tile[2] == {(5, 0), (5, 2), (5, 4), (5, 6)}
            assert [s["kind"] for s in info["sigs"] if s["tile"] == 2] == ["INS", "INS", "DEL", "DEL"]


def test_gaps_case_spacing_clips_and_gap_classes():
    c = E.case("gaps")
    for info in (x for x in c["records"] if x["label"]):
        tiles = sorted({s["tile"] for s in info["sigs"]})
        assert tiles == [0, 1, 3, 6, 11]
        assert [b - a for a, b in zip(tiles, tiles[1:])] == [1, 2, 3, 5]
        ops = c["reads"][info["rec"]].cigartuples
        first = info["sigs"][0]
        assert first["kind"] == "INS" and all(op in (E.H, E.S) for op, _ in ops[:first["i"]]) and first["i"] >= 1
        gap = [ops[i] for i in range(len(ops)) if i not in _hits(info) and i >= first["i"]]
        assert {op for op, _ in gap} == {E.M, E.EQ, E.X, E.N, E.P, E.I, E.D}
        assert all(ln == E.MIN_SIG - 1 for op, ln in gap if op in (E.I, E.D)) and all(ln > 0 for _, ln in gap)
    assert {c["records"][i]["d0"] for i in range(len(c["records"])) if c["records"][i]["label"]} == {0, 1, 2, 3}


def test_thresholds_case_sits_on_tile_and_chunk_edges():
    c = E.case("thresholds")
    seen = set()
    for info in (x for x in c["records"] if x["label"]):
        ops = c["reads"][info["rec"]].cigartuples
        for e in (256, 512):
            pair = [ops[e - 1], ops[e]]
            assert sorted(ln for _, ln in pair) == [E.MIN_SIG - 1, E.MIN_SIG]
            hit = [s for s in info["sigs"] if s["i"] in (e - 1, e)]
            assert len(hit) == 1 and hit[0]["len"] == E.MIN_SIG
            seen.add((e, hit[0]["i"] == e, pair[0][0], pair[1][0]))
    assert len(seen) == 16


def test_merges_case_chains_and_del_pairs():
    c = E.case("merges")
    recs = _by_label(c)
    for k in E.CHAINS:
        info = recs["ins_chain_%d" % k]
        ins = [s for s in info["sigs"] if s["kind"] == "INS"]
        assert len(ins) == k and ins[0]["i"] == 511 and (ins[0]["tile"], ins[0]["lane"], ins[0]["item"], ins[0]["chunk"]) == (1, 31, 7, 0)
        assert ins[-1]["chunk"] == 1
        if k == E.CHAINS[-1]:
            assert ins[-1]["i"] == info["n_ops"] - 1
    for pname, n_pieces in (("defaults", list(E.CHAINS)), ("merge", list(E.CHAINS)), ("zero", [1])):
        ex = E.expected(c, pname)
        got = sorted({x[3] for k in E.CHAINS for x in ex[recs["ins_chain_%d" % k]["rec"]][1]})
        assert got == sorted(set(n_pieces)), pname
    # the first DEL of a record joins the next one under the first-signature rule only; a later pair of the same spacing does not
    for first in (255, 511, 1023):
        info = recs["del_pairs_from_%d" % first]
        dels, _ = E.expected(c, "merge")[info["rec"]]
        assert dels[0][1] == 140 and all(ln in (80, 60) for _, ln in dels[1:])
        assert len(E.expected(c, "defaults")[info["rec"]][0]) == len(dels) + 1


def test_one_op_records():
    c = E.case("one_op")
    ones = [c["reads"][x["rec"]].cigartuples for x in c["records"] if x["n_ops"] == 1 and x["label"]]
    assert sorted(o[0][0] for o in ones) == [E.M, E.I, E.D, E.S, E.H]


@pytest.mark.parametrize("pname", list(E.PARAMS))
@pytest.mark.parametrize("name", E.CASES)
def test_literals_match_reference_golden(name, pname):
    """The builder's planted literals (positions, lengths, query slices, merged per generate_combine_sigs) are what the reference
    emits, record by record in its order, and its reads rows."""
    c = E.case(name)
    cand, rows = golden(name, pname)
    assert E.ordered(cand) == E.expected_ordered(c, pname)
    assert rows == E.expected_rows(c, pname)
    assert not any(cand[k] for k in ("DUP", "INV", "TRA"))


@pytest.mark.parametrize("pname", list(E.PARAMS))
@pytest.mark.parametrize("name", E.CASES)
def test_emulator_matches_reference_golden(name, pname):
    c = E.case(name)
    ex, (gc, gr) = emulated(c, pname)
    cand, rows = golden(name, pname)
    assert not compare_extract.diff_extract(cand, rows, gc, gr)
    assert E.ordered(gc) == E.ordered(cand)
    if name == "merges" and pname != "zero":   # the chains of more insertions than the open-piece buffer holds
        cnt = sorted(ex["piece_cnt"].tolist())
        assert cnt.count(E.MAX_OPEN_PIECES) == 1 and cnt.count(E.MAX_OPEN_PIECES - 1) == 1
        assert (ex["pieces"][:, 3] == 2).sum() == 2


@pytest.mark.skipif(not ref_harness.available(), reason="CUTESV_REF_SRC does not name a cuteSV checkout's src/ directory")
@pytest.mark.parametrize("pname", list(E.PARAMS))
@pytest.mark.parametrize("name", E.CASES)
def test_emulator_matches_live_reference(name, pname):
    c = E.case(name)
    _, (gc, gr) = emulated(c, pname)
    cand, rows = ref_harness.run_parse_reads(c["reads"], E.params(pname))
    assert not compare_extract.diff_extract(cand, rows, gc, gr)
    assert E.ordered(gc) == E.ordered(cand)
