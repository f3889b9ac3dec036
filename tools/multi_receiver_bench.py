#!/usr/bin/env python3
"""Throughput of K NBFM receivers on one 2.4 MS/s capture of u8 I/Q bytes held in memory, K in {1, 2, 4, 8}.

Plans:
  merged     run(): the receivers are one device DAG, the u8 file source its first node -- the bytes cross PCIe once, at
             2 B per sample
  per_chain  run(device_dag=False): one flow graph per receiver; with K >= 2 the source converts its bytes on its own and
             every chain uploads the complex64 samples (8 B per sample, K times); with K = 1 the chain absorbs the source
Configurations: the reference's 8192-sample source vectors, and the same with superchunk = 2^20.  Each (plan,
configuration) is warmed up on 2^20 samples, then the plans are alternated `--reps` times with a wall clock around run(),
which ends after the flush; the median and the spread (max - min) are reported.  The outputs of the two plans are
compared once per configuration, at the stream tolerance of tests/test_gpu_dag_boundary.py (1e-5 of max(1, |ref|)): the
calls differ in length, so the FIR kernels do.

    python tools/multi_receiver_bench.py --out profiles/h100_<W>w_multi_receiver_bench.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import luaradio_b200 as radio                                   # noqa: E402
from luaradio_b200 import _lib                                  # noqa: E402

RATE = 2.4e6
VECTOR = 8192
SUPERCHUNK = 1 << 20
DECIMATION = 50                                                 # 48 kHz per receiver


def offsets(k):
    return [-1.05e6 + 2.1e6 * (i + 0.5) / 8 for i in range(k)]


def capture(n, k_max=8, seed=1):
    """u8 I/Q bytes: an NBFM carrier at every receiver's offset plus noise; 2^22 samples generated, then repeated."""
    rng = np.random.default_rng(seed)
    m = min(n, 1 << 22)
    t = np.arange(m) / RATE
    x = np.zeros(m, np.complex128)
    for i, f in enumerate(offsets(k_max)):
        tone = np.sin(2 * np.pi * (600 + 300 * i) * t)
        x += 0.1 * np.exp(1j * (2 * np.pi * f * t + 2 * np.pi * 3e3 * np.cumsum(tone) / RATE))
    x += 0.02 * (rng.uniform(-1, 1, m) + 1j * rng.uniform(-1, 1, m))
    raw = np.clip(np.round(np.stack([x.real, x.imag], 1).reshape(-1) * 127.5 + 127.5), 0, 255).astype(np.uint8)
    return np.resize(raw, 2 * n)


def top_block(raw, k):
    src = radio.IQFileSource(raw, "u8", RATE, chunk=VECTOR)
    top, sinks = radio.CompositeBlock(), []
    for f in offsets(k):
        sinks.append(radio.ArraySink())
        top.connect(src, radio.TunerBlock(f, 20e3, DECIMATION), radio.NBFMDemodulator(5e3, 4e3), sinks[-1])
    return top, sinks


def timed(raw, k, superchunk, device_dag):
    top, sinks = top_block(raw, k)
    t0 = time.perf_counter()
    top.run(superchunk=superchunk, device_dag=device_dag)
    return time.perf_counter() - t0, [s.result() for s in sinks], top.describe_gpu_graph()


def max_rel_err(got, ref):
    if any(len(g) != len(r) for g, r in zip(got, ref)):
        return float("inf")
    return max(float(np.max(np.abs(g.astype(np.float64) - r), initial=0)) / max(1.0, float(np.max(np.abs(r), initial=0)))
               for g, r in zip(got, ref))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=26, help="log2 of the capture's samples")
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    _lib.require_device()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    n = 1 << args.n
    raw = capture(n)
    warm = raw[:2 << 20]
    rows = []
    for k in [int(v) for v in args.ks.split(",")]:
        for cfg, sc in (("vector", 0), ("superchunk", SUPERCHUNK)):
            plans = {"merged": True, "per_chain": False}
            for dd in plans.values():
                timed(warm, k, sc, dd)
            times, outs, desc = {p: [] for p in plans}, {}, {}
            for _ in range(args.reps):
                for p, dd in plans.items():
                    t, o, d = timed(raw, k, sc, dd)
                    times[p].append(t)
                    outs[p], desc[p] = o, d
            err = max_rel_err(outs["merged"], outs["per_chain"])
            for p in plans:
                med = float(np.median(times[p]))
                row = {"receivers": k, "config": cfg, "superchunk": sc, "plan": p, "samples": n, "seconds": times[p],
                       "median_s": med, "spread_s": max(times[p]) - min(times[p]), "msps": n / med / 1e6,
                       "describe": desc[p], "max_rel_err_vs_per_chain": err, "outputs_equal": err <= 1e-5}
                rows.append(row)
                print(json.dumps({kk: v for kk, v in row.items() if kk != "describe"}), flush=True)
            del outs
    rec = {"gpu": smi, "input_rate": RATE, "vector": VECTOR, "decimation": DECIMATION, "format": "u8", "results": rows}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
