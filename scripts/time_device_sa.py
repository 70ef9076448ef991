"""Times SA:Z text -> SA columns on the device (Engine.reduce_sa, csv_reduce_sa_device) against the route a caller with the text in
GPU memory has without it: D2H of the text and its offsets, the host reduction, H2D of sa_off and the seven columns.  The host
reduction is the statement of cutesv_b200/csrc/sa_core.h compiled with g++ -O2 for one CPU thread (tests/emul/emul_sa.cpp, built
into a temporary directory); the native BAM decoder runs the same parse spread over its parser threads.  Both routes must give
equal columns.  Prints the card, its power limit, and per route the median with min / max over the repetitions (the routes
alternate).

    python scripts/time_device_sa.py [--records 200000] [--reps 5] [--seed 1]

The packet: records with 0 to 4 supplementary alignments (about half without an SA tag), names among 25 contigs, CIGARs of
clips around one match, 1 % ultra-long reads with 200 entries."""
import argparse
import ctypes as C
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from cutesv_b200 import _abi  # noqa: E402
from cutesv_b200.engine import Engine  # noqa: E402


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except Exception as e:   # reported, not guessed
        pl = "unknown (%s)" % e
    return torch.cuda.get_device_name(0), pl


def stats(xs):
    xs = sorted(xs)
    return "median %.2f ms (min %.2f, max %.2f, n=%d)" % (1e3 * xs[len(xs) // 2], 1e3 * xs[0], 1e3 * xs[-1], len(xs))


def make_values(n, seed, names):
    rng = np.random.default_rng(seed)
    k = rng.choice([0, 0, 0, 1, 1, 2, 3, 4], n)
    k[rng.random(n) < 0.01] = 200
    out = []
    for i in range(n):
        ents = []
        for _ in range(int(k[i])):
            a, m, b = (int(x) for x in rng.integers(0, 20000, 3))
            ents.append("%s,%d,%s,%dS%dM%dS,%d,%d;" % (names[int(rng.integers(0, len(names)))], int(rng.integers(1, 2 ** 28)), "+-"[i & 1],
                                                      a, m + 1, b, int(rng.integers(0, 61)), int(rng.integers(0, 500))))
        out.append("".join(ents).encode())
    off = np.zeros(n + 1, np.int64)
    np.cumsum([len(v) for v in out], out=off[1:])
    return np.frombuffer(b"".join(out), np.uint8).copy(), off


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    import torch
    tmp = tempfile.mkdtemp()
    so = os.path.join(tmp, "libemul_sa.so")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "emul", "emul_sa.cpp")])
    L = C.CDLL(so)
    L.emul_sa_reduce.restype = C.c_uint32
    names = ["chr%d" % k for k in range(1, 23)] + ["chrX", "chrY", "chrM"]
    srt = sorted(names)
    nb = np.frombuffer("".join(srt).encode(), np.uint8).copy()
    noff = np.zeros(len(srt) + 1, np.int64)
    np.cumsum([len(s) for s in srt], out=noff[1:])
    nid = np.arange(len(srt), dtype=np.int32)
    text, off = make_values(a.records, a.seed, names)
    dev = torch.device("cuda", 0)
    d_text, d_off = torch.from_numpy(text).to(dev), torch.from_numpy(off).to(dev)
    eng = Engine(0, contig_lens=np.full(len(srt), 10 ** 8, np.int64))
    eng.set_contigs(np.full(len(srt), 10 ** 8, np.int64), names=srt)
    n = a.records
    cap = len(text) // 10 + 1

    def p(x, t):
        return x.ctypes.data_as(C.POINTER(t))

    def host_route():
        h_text, h_off = d_text.cpu(), d_off.cpu()   # synchronous D2H
        t, o = h_text.numpy(), h_off.numpy()
        sa_off = np.empty(n + 1, np.int64)
        cols = np.empty((7, cap), np.int32)
        nr = C.c_int64(0)
        bad = L.emul_sa_reduce(p(nb, C.c_uint8), p(noff, C.c_int64), p(nid, C.c_int32), C.c_int64(len(nid)), p(t, C.c_uint8), p(o, C.c_int64),
                               C.c_int64(len(t)), C.c_int64(n), p(sa_off, C.c_int64), p(cols, C.c_int32), C.c_int64(cap), C.byref(nr))
        assert bad == 0
        m = nr.value
        out = torch.from_numpy(sa_off).to(dev), {f: torch.from_numpy(np.ascontiguousarray(cols[k, :m])).to(dev) for k, f in enumerate(_abi.SA_FIELDS)}
        torch.cuda.synchronize()
        return out

    def device_route():
        out = eng.reduce_sa(d_text, d_off)   # returns when the columns are complete
        torch.cuda.synchronize()
        return out

    w_host, w_dev = host_route(), device_route()   # warm-up, and the routes must agree
    assert w_host[0].equal(w_dev[0]) and all(w_host[1][f].equal(w_dev[1][f]) for f in _abi.SA_FIELDS)
    t_host, t_dev = [], []
    for _ in range(a.reps):
        for fn, acc in ((host_route, t_host), (device_route, t_dev)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            acc.append(time.perf_counter() - t0)
    name, pl = card()
    print("card: %s, power limit %s" % (name, pl))
    print("packet: %d records, %d SA entries, %.1f MB of SA text" % (n, int(w_dev[0][-1]), len(text) / 1e6))
    print("host route (D2H text, host reduction on one thread, H2D columns): %s" % stats(t_host))
    print("device route (csv_reduce_sa_device): %s" % stats(t_dev))
    eng.close()


if __name__ == "__main__":
    main()
