#!/usr/bin/env python
"""Config 2 (bench.py's workload and seed) end to end with host-resident vs GPU-resident inputs, at the same sizes.

  host    pinned host columns -> csv_cluster_host (H2D + kernels + D2H) -> host records
  device  torch CUDA tensors -> csv_upload_*_device (device-to-device copies) -> csv_cluster -> Engine.result_tensors()

Both paths are timed with CUDA events on the engine's stream after warm-up, every step between its own pair of events; the
device path is also split into its upload and its csv_cluster.  Prints the card, its power limit and max SM clock, then one
JSON line.  The two paths' records are asserted byte-identical.

  python scripts/time_device_inputs.py [--steps 20] [--warmup 3] [--scale 1.0]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cutesv_b200 import _abi, synth  # noqa: E402


def stats(ms):
    ms = np.asarray(ms)
    return {"median_ms": float(np.median(ms)), "p10_ms": float(np.percentile(ms, 10)), "p90_ms": float(np.percentile(ms, 90))}


def canonical(res):
    """Records with the names buffer's layout taken out (it is filled through an atomic append cursor, so names_off and the
    kept-cluster slot differ from run to run): every other byte, and each candidate's supporting read ids."""
    cands, genos, names = res
    c = np.array(cands, copy=True)
    slices = np.concatenate([names[o:o + n] for o, n in zip(c["names_off"], c["names_cnt"])] + [np.zeros(0, np.int32)])
    c["names_off"] = 0
    c["cluster"] = 0
    return c.tobytes(), np.asarray(genos).tobytes(), slices.tobytes(), len(names)


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() if q.returncode == 0 else "unavailable"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    import torch
    from cutesv_b200.engine import Engine

    torch.cuda.set_device(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    cfg = synth.make_config(2, args.scale, seed=synth.SEED0 + 2)   # bench.py's workload(2, scale, rank 0)
    params = _abi.default_params(**cfg["params"])
    eng = Engine(0, stream=stream.cuda_stream, params=params, contig_lens=cfg["lens"])
    type_mask = sum(1 << _abi.TYPE_IDS[k] for k in cfg["sigs"])

    def pinned(cols):
        out = {}
        for k, v in cols.items():
            out[k] = None if v is None else torch.from_numpy(np.ascontiguousarray(v)).pin_memory()
        return out

    def on_device(cols):
        return {k: (None if v is None else v.to("cuda:0", non_blocking=True)) for k, v in cols.items()}

    sigs_p = {k: pinned(v) for k, v in cfg["sigs"].items()}
    reads_p = pinned(cfg["reads"])
    sigs_h = {k: {c: (None if v is None else v.numpy()) for c, v in s.items()} for k, s in sigs_p.items()}
    reads_h = {c: v.numpy() for c, v in reads_p.items()}
    sigs_d = {k: on_device(v) for k, v in sigs_p.items()}
    reads_d = on_device(reads_p)
    stream.synchronize()
    in_bytes = sum(v.nbytes for s in sigs_h.values() for v in s.values() if v is not None) + sum(v.nbytes for v in reads_h.values())

    eng.upload(sigs_h, reads_h)
    eng.cluster_device(type_mask)
    n_cand, n_names = eng.counts()
    cap_c, cap_n = 2 * n_cand + 1024, 2 * n_names + 1024
    pin = [torch.empty(cap_c * 64, dtype=torch.uint8, pin_memory=True), torch.empty(cap_c * 40, dtype=torch.uint8, pin_memory=True),
           torch.empty(cap_n * 4, dtype=torch.uint8, pin_memory=True)]
    out = (pin[0].numpy().view(_abi.CAND_DTYPE), pin[1].numpy().view(_abi.GENO_DTYPE), pin[2].numpy().view(np.int32))

    def timed(step, k):
        ts = []
        for _ in range(k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            res = step()
            e1.record(stream)
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return ts, res

    def step_host():
        return eng.cluster(sigs_h, reads_h, type_mask, out=out)

    def step_device():
        eng.upload(sigs_d, reads_d, stream=stream)
        eng.cluster_device(type_mask)
        return eng.result_tensors()

    def step_upload():
        eng.upload(sigs_d, reads_d, stream=stream)

    def step_cluster():
        eng.cluster_device(type_mask)
        return eng.result_tensors()

    def step_resident():   # bench.py's `value`: inputs already resident, no upload
        eng.cluster_device(type_mask)

    res = {}
    host_res = dev_res = None
    for name, fn in (("host", step_host), ("device", step_device), ("resident", step_resident)):
        timed(fn, args.warmup)
        ts, r = timed(fn, args.steps)
        res[name] = stats(ts)
        if name == "host":
            host_res = tuple(np.array(x, copy=True) for x in r)
        elif name == "device":
            dev_res = (r[0].cpu().numpy().view(_abi.CAND_DTYPE)[:, 0], r[1].cpu().numpy().view(_abi.GENO_DTYPE)[:, 0], r[2].cpu().numpy())
    # the device path split: upload alone (the producer stream waits for the copies) and csv_cluster + result_tensors alone,
    # alternating so that both see the same state
    up, cl = [], []
    for k in range(args.warmup + args.steps):
        t_up, _ = timed(step_upload, 1)
        t_cl, _ = timed(step_cluster, 1)
        if k >= args.warmup:
            up += t_up
            cl += t_cl
    res["device_upload"] = stats(up)
    res["device_cluster"] = stats(cl)
    for e, g, what in zip(canonical(host_res), canonical(dev_res), ("candidate records", "genotype records", "names", "names count")):
        assert e == g, "host and device inputs give different %s" % what
    line = {"workload": "config2 (bench.py seed), %d signatures, %d reads rows, --genotype" % (cfg["n_sigs"], len(cfg["reads"]["chrom"])),
            "input_bytes": int(in_bytes), "steps": args.steps, "warmup": args.warmup, "card": card(), "n_cand": int(len(host_res[0])),
            "records_equal": True, "ms": res, "graph_replays": eng.graph_replays()}
    print(json.dumps(line))
    eng.close()


if __name__ == "__main__":
    main()
