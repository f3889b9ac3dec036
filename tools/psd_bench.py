#!/usr/bin/env python3
"""Device throughput of the PSD kernels (aux_blocks.cu psd_kernel / psd1024_kernel for N <= 4096, psd_long.cu above) at
the spectrum sinks' frame lengths and the long ones, complex and real input, logarithmic output, 256 Mi samples per
call in DEVICE mode, timed with CUDA events.

Roofline bytes are what the PSD must move: 8 B in + 4 B out per complex sample, 4 + 4 per real one.  The two-pass
form (N >= 32768) also writes and reads its scratch buffer, 16 B per sample more; `hbm_GBs_with_scratch` counts them.

    python tools/psd_bench.py [out.json] [log2_samples]
"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [1024, 4096, 8192, 16384, 65536, 1 << 17, 1 << 18, 1 << 20]
STEPS, WARMUP = 5, 2


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                   # the record still names the device through torch
        return {"nvidia_smi_error": str(e)}


def main():
    import torch
    import bench
    from luaradio_b200 import _lib
    from luaradio_b200.utilities import window_utils
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    n = 1 << (int(sys.argv[2]) if len(sys.argv) > 2 else 28)
    lib = _lib.require_device(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    _lib.check(lib.lrb200_set_stream(ctypes.c_void_p(stream.cuda_stream)))
    peak, peak_src = bench.peaks()
    x = torch.empty(n, dtype=torch.complex64, device="cuda")
    y = torch.empty(n, dtype=torch.float32, device="cuda")
    _lib.check(lib.lrb200_synth_white_iq(ctypes.c_void_p(x.data_ptr()), 0, n, 1))
    rows = []
    for N in SIZES:
        win = np.array(window_utils.window(N, "hamming", True), np.float32)
        scale = 2.0 * float(np.sum(win.astype(np.float64) ** 2))
        for cplx in (True, False):
            h = _lib.check_handle(lib.lrb200_psd_create(N, win.ctypes.data, scale, 1, int(cplx), _lib.LRB200_DEVICE), "psd")
            no = ctypes.c_size_t(0)

            def step():
                _lib.check(lib.lrb200_block_execute(h, ctypes.c_void_p(x.data_ptr()), n, ctypes.c_void_p(y.data_ptr()),
                                                    ctypes.byref(no)), "psd")
            for _ in range(WARMUP):
                step()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(STEPS):
                step()
            e1.record(stream)
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / STEPS
            lib.lrb200_block_destroy(h)
            roof = 12 if cplx else 8
            extra = 16 if N >= 32768 else 0
            gbs = roof * n / (ms * 1e-3) / 1e9
            rows.append({"N": N, "input": "complex" if cplx else "real", "samples": n, "ms": round(ms, 3),
                         "msamples_per_s": round(n / ms / 1e3, 1), "roofline_bytes_per_sample": roof,
                         "scratch_bytes_per_sample": extra, "hbm_GBs_roofline_bytes": round(gbs, 1),
                         "frac_of_roofline": round(gbs / peak, 4),
                         "hbm_GBs_with_scratch": round((roof + extra) * n / (ms * 1e-3) / 1e9, 1),
                         "path": "psd1024_kernel" if N == 1024 else "psd_kernel" if N <= 4096 else
                                 "psd_long single CTA" if N <= 16384 else "psd_long two-pass"})
            print(json.dumps(rows[-1]), file=sys.stderr)
    rec = {"device": torch.cuda.get_device_name(0), "card": card(), "peak_GBs": peak, "peak_source": peak_src,
           "steps": STEPS, "warmup": WARMUP, "window": "hamming", "logarithmic": True, "rows": rows}
    text = json.dumps(rec, indent=1)
    if out_path:
        with open(out_path, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
