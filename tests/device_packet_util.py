"""Helpers of the device-extraction tests: packets with BAM-packed bases, their torch CUDA copies, and the host strings the
device-built INS sequences must equal."""
import numpy as np

from cutesv_b200 import packing


def with_bases(pk, queries):
    """The packet plus seq_off / seq4 packed from one query string (or None: no stored bases) per record."""
    out = dict(pk)
    out["seq4"], out["seq_off"] = packing.pack_bases(list(queries))
    return out


def to_device(pk, device=0):
    """torch CUDA copies of every array of a packet (the CIGAR as int32: torch has no uint32 arithmetic everywhere)."""
    import torch
    dev = torch.device("cuda", device)

    def t(a):
        a = np.ascontiguousarray(a)
        if a.dtype == np.uint32:
            a = a.view(np.int32)
        return torch.from_numpy(a.copy()).to(dev)
    out = {k: t(v) for k, v in pk.items() if k not in ("sa", "seq_lo", "seq_hi")}
    out["sa"] = {k: t(v) for k, v in pk["sa"].items()}
    return out


def host_ins_strings(ex, query_of, cigar_of, merge, rec_base=0):
    """INS strings the host builds from the piece list (packing.ins_sequence), by INS row."""
    s = ex["sigs"]["INS"]
    return [packing.ins_sequence(ex["pieces"], int(ex["piece_off"][i]), int(ex["piece_cnt"][i]), lambda rec: query_of(rec - rec_base),
                                 (lambda rec: cigar_of(rec - rec_base)) if cigar_of else None, merge) for i in range(len(s["chrom"]))]


def cigar_of_packet(pk):
    return lambda rec: (pk["cigar"][pk["cigar_off"][rec]:pk["cigar_off"][rec + 1]], int(pk["ref_start"][rec]))


def flat_seq(pk):
    """A subset packet of bamio.subset_packet (seq_lo / seq_hi into its parent's bases) with its bases regathered under seq_off."""
    if "seq_lo" not in pk:
        return pk
    out = {k: v for k, v in pk.items() if k not in ("seq_lo", "seq_hi", "seq4")}
    lo, hi = pk["seq_lo"].astype(np.int64), pk["seq_hi"].astype(np.int64)
    off = np.zeros(len(lo) + 1, dtype=np.int64)
    np.cumsum(hi - lo, out=off[1:])
    out["seq_off"] = off
    out["seq4"] = np.concatenate([pk["seq4"][a:b] for a, b in zip(lo.tolist(), hi.tolist())]) if len(lo) else np.zeros(0, np.uint8)
    return out
