#!/usr/bin/env python3
"""Throughput of PLLBlock's two GPU forms on DEVICE calls of 2^26 samples, for the receivers' three loops (stereo pilot,
RDS, AM synchronous; tests/pll_ref.py LOOPS), on a noisy locked pilot and on the same pilot with 1 % and 10 % of its
length in zero stretches (4 and 10 stretches), with the re-run counts of lrb200_pll_chunk_counts.  Mode 1 is timed as
the median of --reps calls after a warm-up call, mode 0 (serial, seconds per call) with one call; each call is timed
with a host clock around the execute and a synchronise of the library stream.

With --ab LIB, mode 1 on the locked pilot is also timed with another build of the library (LRB200_LIB=LIB), in
alternating subprocesses, --ab-rounds times each, so that the two builds share the card's state.

    python tools/pll_bench.py --out profiles/h100_<W>w_pll_bench.json [--ab /path/to/parent/libluaradio_b200.so]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N = 1 << 26
INPUTS = {"locked": (0, 0), "zeros_1pct": (4, 0.01), "zeros_10pct": (10, 0.10)}


def make_input(lp, kind):
    from tests import pll_ref as R
    x = R.pilot(lp, N, "noisy", seed=51)
    k, frac = INPUTS[kind]
    for j in range(k):
        a = int((j + 0.5) * N / k)
        x[a:a + int(frac * N / k)] = 0
    return x


def time_calls(loop_name, kind, mode, reps, counts=True):
    """[seconds per call], (chunks, reruns) of the last call, in this process with the library _lib loads."""
    from luaradio_b200 import _lib
    from tests import pll_ref as R
    lib = _lib.require_device()
    lp = R.Loop(*R.LOOPS[loop_name])
    x = make_input(lp, kind)
    bufs = [_lib.check_handle(lib.lrb200_malloc(N * s), "buffer") for s in (8, 8, 4)]
    times, cnt = [], None
    try:
        _lib.check(lib.lrb200_memcpy_h2d(bufs[0], x.ctypes.data, N * 8), "h2d")
        _lib.check(lib.lrb200_sync(), "sync")
        xa, ya, no = (ctypes.c_void_p * 1)(bufs[0]), (ctypes.c_void_p * 2)(bufs[1], bufs[2]), ctypes.c_size_t()
        for r in range(reps + (1 if mode == 1 else 0)):
            bw, fmin, fmax, m, rate = lp.args
            h = _lib.check_handle(lib.lrb200_pll_create(bw, fmin, fmax, m, rate, _lib.LRB200_DEVICE), "pll")
            _lib.check(lib.lrb200_pll_set_mode(h, mode), "pll_set_mode")
            _lib.check(lib.lrb200_sync(), "sync")
            t0 = time.perf_counter()
            _lib.check(lib.lrb200_block_execute_multi(h, xa, 1, N, ya, 2, ctypes.byref(no)), "execute")
            _lib.check(lib.lrb200_sync(), "sync")
            t = time.perf_counter() - t0
            if counts:
                c, rr = ctypes.c_uint64(), ctypes.c_uint64()
                _lib.check(lib.lrb200_pll_chunk_counts(h, ctypes.byref(c), ctypes.byref(rr)), "pll_chunk_counts")
                cnt = (c.value, rr.value)
            lib.lrb200_block_destroy(h)
            if mode == 0 or r > 0:                                   # mode 1: the first call warms up
                times.append(t)
    finally:
        for b in bufs:
            lib.lrb200_free(b)
    return times, cnt


def child(args):
    if args.no_counts:                  # a build from before lrb200_pll_chunk_counts (the --ab baseline)
        from luaradio_b200 import _lib
        _lib._PROTOS.pop("lrb200_pll_chunk_counts", None)
    times, cnt = time_calls(args.loop, args.kind, args.mode, args.reps, counts=not args.no_counts)
    print(json.dumps({"times": times, "counts": cnt}))


def run_child(lib_path, loop_name, kind, mode, reps, no_counts=False):
    env = dict(os.environ)
    if lib_path:
        env["LRB200_LIB"] = lib_path
    cmd = [sys.executable, os.path.abspath(__file__), "--child", "--loop", loop_name, "--kind", kind, "--mode", str(mode),
           "--reps", str(reps)] + (["--no-counts"] if no_counts else [])
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True).stdout
    return json.loads(out.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--loops", default="stereo,rds,am_sync")
    ap.add_argument("--ab", default=None, help="another build of libluaradio_b200.so to alternate with (mode 1, locked)")
    ap.add_argument("--ab-rounds", type=int, default=3)
    ap.add_argument("--ab-only", action="store_true", help="skip the table of modes and inputs")
    ap.add_argument("--modes", default="1,0", help="the modes of the table")
    ap.add_argument("--child", action="store_true")
    ap.add_argument("--loop", default="stereo")
    ap.add_argument("--kind", default="locked")
    ap.add_argument("--mode", type=int, default=1)
    ap.add_argument("--no-counts", action="store_true")
    args = ap.parse_args()
    if args.child:
        return child(args)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    rows = []
    for name in ([] if args.ab_only else args.loops.split(",")):
        for kind in INPUTS:
            for mode in [int(v) for v in args.modes.split(",")]:
                r = run_child(None, name, kind, mode, args.reps if mode == 1 else 1)
                t = float(np.median(r["times"]))
                row = {"loop": name, "input": kind, "mode": mode, "samples": N, "seconds": t, "all_s": r["times"],
                       "msps": N / t / 1e6}
                if mode == 1:
                    row["chunks"], row["reruns"] = r["counts"]
                rows.append(row)
                print(json.dumps(row), flush=True)
    ab = []
    if args.ab:
        for name in args.loops.split(","):
            for rnd in range(args.ab_rounds):
                for which, path in (("parent", args.ab), ("this", None)):
                    r = run_child(path, name, "locked", 1, args.reps, no_counts=which == "parent")
                    t = float(np.median(r["times"]))
                    row = {"loop": name, "input": "locked", "mode": 1, "build": which, "round": rnd, "seconds": t,
                           "all_s": r["times"], "msps": N / t / 1e6}
                    ab.append(row)
                    print(json.dumps(row), flush=True)
    rec = {"gpu": smi, "samples": N, "results": rows, "ab_mode1_locked": ab}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
