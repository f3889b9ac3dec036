"""IIRFilterBlock with 11..64 taps (iir_order.cu): 256 Mi samples in one DEVICE-mode call, real and complex, feedback
order q = 10, 16, 32, 63.  CUDA events around each call after a warm-up call; GS/s and the share of the HBM roofline
(8 B/sample real, 16 B/sample complex, 3.35 TB/s data-sheet HBM3 bandwidth of the H100 SXM).

    python tools/iir_order_bench.py [--n LOG2] [--reps R] [--out FILE]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from luaradio_b200 import _lib  # noqa: E402

HBM = 3.35e12


def taps(q):
    """a stable all-pole-plus-zeros design of order q: poles at radius 0.9 spread over the circle, b = ones / q"""
    poles = 0.9 * np.exp(2j * np.pi * (np.arange(q) + 0.5) / q)
    a = np.poly(poles).real.astype(np.float32)
    b = np.full(q + 1, 1.0 / (q + 1), np.float32)
    return b, a


# timing-only variants of iir_order.cu (their outputs are wrong), built in a temporary copy of the package
ABLATIONS = {
    "no_lookback": [("for (int d = 1; d <= dlast; ++d) {", "for (int d = 1; d <= 0; ++d) {")],
    "no_chains": [("for (int t = 0; t < IO_THREADS; ++t) {", "for (int t = 0; t < 0; ++t) {")],
    "no_lookback_no_chains": [("for (int d = 1; d <= dlast; ++d) {", "for (int d = 1; d <= 0; ++d) {"),
                              ("for (int t = 0; t < IO_THREADS; ++t) {", "for (int t = 0; t < 0; ++t) {")],
}


def ablate(name, n_log2, reps):
    """run this script on a patched copy of the package; returns its result rows"""
    import shutil
    import tempfile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with tempfile.TemporaryDirectory() as tmp:
        for d in ("luaradio_b200", "include", "tools"):
            shutil.copytree(os.path.join(root, d), os.path.join(tmp, d), copy_function=shutil.copy2)
        src = os.path.join(tmp, "luaradio_b200", "csrc", "iir_order.cu")
        text = open(src).read()
        for old, new in ABLATIONS[name]:
            assert old in text, old
            text = text.replace(old, new)
        open(src, "w").write(text)
        subprocess.run([sys.executable, "-m", "luaradio_b200.build"], cwd=tmp, check=True, capture_output=True)
        out = os.path.join(tmp, "rows.json")
        subprocess.run([sys.executable, os.path.join(tmp, "tools", "iir_order_bench.py"), "--n", str(n_log2), "--reps",
                        str(reps), "--out", out], cwd=tmp, check=True, capture_output=True)
        return json.load(open(out))["results"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ablations", action="store_true", help="also time the no-look-back / no-chain variants")
    ap.add_argument("--n", type=int, default=28)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    lib = _lib.require_device()
    n = 1 << args.n
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows = []
    for cplx in (False, True):
        dt = torch.complex64 if cplx else torch.float32
        x = torch.randn(n, dtype=dt, device="cuda")
        y = torch.empty_like(x)
        for q in (10, 16, 32, 63):
            b, a = taps(q)
            fn = lib.lrb200_iir_create_crcf if cplx else lib.lrb200_iir_create_rrrf
            h = _lib.check_handle(fn(b.ctypes.data, len(b), a.ctypes.data, len(a), _lib.LRB200_DEVICE), "iir")
            no = ctypes.c_size_t()
            _lib.check(lib.lrb200_block_execute(h, x.data_ptr(), n, y.data_ptr(), ctypes.byref(no)), "warm-up")
            _lib.check(lib.lrb200_sync(), "sync")
            stream = torch.cuda.ExternalStream(lib.lrb200_get_stream())
            times = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                _lib.check(lib.lrb200_block_execute(h, x.data_ptr(), n, y.data_ptr(), ctypes.byref(no)), "execute")
                e1.record(stream)
                e1.synchronize()
                times.append(e0.elapsed_time(e1) * 1e-3)
            lib.lrb200_block_destroy(h)
            t = float(np.median(times))
            bps = 16 if cplx else 8
            rows.append({"complex": cplx, "q": q, "nb": len(b), "samples": n, "median_s": t, "all_s": times,
                         "gsps": n / t / 1e9, "roofline_share": n * bps / HBM / t})
            print(json.dumps(rows[-1]), flush=True)
    rec = {"gpu": smi, "hbm_bytes_per_s": HBM, "results": rows}
    if args.ablations:
        rec["ablations"] = {name: ablate(name, args.n, args.reps) for name in ABLATIONS}
        for name, r in rec["ablations"].items():
            print(json.dumps({name: [(v["complex"], v["q"], round(v["gsps"], 2)) for v in r]}), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)
    print(json.dumps({"gpu": smi}))


if __name__ == "__main__":
    main()
