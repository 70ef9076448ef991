"""Helpers of the read-name tests: adversarial name sets, their byte packing, Python's dense `sorted` ranks, and named device
packets built from a packet's names."""
import uuid

import numpy as np


def pack_names(names):
    """(uint8 bytes, int64 offsets with n + 1 entries) of a list of str (UTF-8) or bytes."""
    raw = [n.encode("utf-8") if isinstance(n, str) else bytes(n) for n in names]
    off = np.zeros(len(raw) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in raw], out=off[1:])
    return np.frombuffer(b"".join(raw), dtype=np.uint8).copy(), off


def dense_ranks(names):
    """Rank of every name among the distinct names in Python `sorted` order."""
    srt = {nm: i for i, nm in enumerate(sorted(set(names)))}
    return np.array([srt[nm] for nm in names], dtype=np.int32)


def _rand_str(rng, k, alphabet="ab0"):
    return "".join(alphabet[i] for i in rng.integers(0, len(alphabet), k))


def name_sets(seed=0):
    """{set name: list of str}: the shapes of real read names and the cases a byte-word radix sort can get wrong."""
    rng = np.random.default_rng(seed)
    out = {}
    out["ont_uuid"] = [str(uuid.UUID(bytes=rng.bytes(16), version=4)) for _ in range(3000)]
    out["pacbio_ccs"] = ["m64011_190830_220126/%d/ccs" % z for z in rng.integers(0, 180_000_000, 3000)]
    for k in (7, 8, 9, 16, 64, 250):
        pre = _rand_str(rng, k, "xyz")
        out["prefix%d" % k] = [pre + _rand_str(rng, int(rng.integers(0, 5))) for _ in range(600)]
    base = ["a", "a\x00", "a\x00\x00", "a\x00b", "ab", "a" * 8, "a" * 8 + "\x00", "a" * 9, "a" * 7 + "\x00", "", "\x00", "\x00\x00",
            "b", "a" * 16, "a" * 16 + "\x00", "a" * 15]
    out["prefixes_nul"] = base + [base[i] for i in rng.integers(0, len(base), 200)]
    out["utf8"] = ["réad_%d" % i for i in range(40)] + ["读取_%d" % i for i in range(40)] + ["\U0001f9ec%d" % i for i in range(40)] + \
        ["read_%d" % i for i in range(40)] + ["ü", "u", "z", "￿", "Ā"]
    out["len254"] = [_rand_str(rng, 254, "ab") for _ in range(300)] + ["c" * 250 + _rand_str(rng, 4) for _ in range(300)] + ["a" * 254, "a" * 253]
    out["one"] = ["only_read"]
    dup = ["dup_%d" % i for i in rng.integers(0, 50, 400)]
    out["duplicates"] = dup
    return out


def named(pk, names, device=0):
    """torch CUDA copy of a device packet (dict of tensors) with read_id replaced by the records' names."""
    import torch
    b, off = pack_names(names)
    out = {k: v for k, v in pk.items() if k != "read_id"}
    dev = torch.device("cuda", device)
    out["names"] = torch.from_numpy(b).to(dev)
    out["name_off"] = torch.from_numpy(off).to(dev)
    return out
