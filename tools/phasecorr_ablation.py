#!/usr/bin/env python3
"""Where BinaryPhaseCorrectorBlock's time goes (luaradio_b200/csrc/phasecorr.cu): one call of 256 Mi complex samples for
(N, I) = (8000, 32), (50, 32) and (4, 1), timed whole with CUDA events and per launch with torch.profiler (reduce, scan,
apply), on this code and on timing-only variants of the kernel file, each built in a temporary copy of the package:

  apply_no_math     the apply pass without the double sincos and the double product (a float32 product with the
                    average itself as the phasor): its outputs are wrong; what is left is the data movement and the scans
  v16               16 samples per thread instead of 8 (4096-sample tiles, twice the registers per thread)

One JSON object on stdout.  Needs a GPU.

    python tools/phasecorr_ablation.py > profiles/h100_400w_phasecorr_ablation.json
"""
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join("luaradio_b200", "csrc", "phasecorr.cu")
HDR = os.path.join("luaradio_b200", "csrc", "blocks.h")

VARIANTS = {
    "this_code": [],
    "apply_no_math": [
        ("""            double sn, cs;
            sincos(-avg, &sn, &cs);
            pr = (double)__double2float_rn(cs);
            pi = (double)__double2float_rn(sn);""",
         """            pr = 1.0;
            pi = avg;"""),
        ("""        xv[i] = make_float2(__double2float_rn(__dsub_rn(__dmul_rn(xr, pr), __dmul_rn(xi, pi))),
                            __double2float_rn(__dadd_rn(__dmul_rn(xr, pi), __dmul_rn(xi, pr))));""",
         """        (void)xr; (void)xi;
        xv[i] = make_float2(xv[i].x * (float)pr - xv[i].y * (float)pi, xv[i].x * (float)pi + xv[i].y * (float)pr);"""),
    ],
    "v16": [("constexpr int PC_V = 8; ", "constexpr int PC_V = 16;"),
            ("constexpr int PC_MAX_TILES = 1 << 17;", "constexpr int PC_MAX_TILES = 1 << 16;")],
}

TIMER = r"""
import ctypes, json, sys
import torch
from luaradio_b200 import _lib
lib = _lib.require_device(0)
stream = torch.cuda.Stream()
torch.cuda.set_stream(stream)
_lib.check(lib.lrb200_set_stream(ctypes.c_void_p(stream.cuda_stream)))
n, steps = 1 << 28, 10
x = torch.empty(n, dtype=torch.complex64, device="cuda")
_lib.check(lib.lrb200_synth_white_iq(ctypes.c_void_p(x.data_ptr()), 0, n, 1))
y = torch.empty(n, dtype=torch.complex64, device="cuda")
no = ctypes.c_size_t(0)
rows = []
for N, I in ((8000, 32), (50, 32), (4, 1)):
    h = _lib.check_handle(lib.lrb200_phasecorrector_create(N, I, _lib.LRB200_DEVICE), "phasecorr")
    step = lambda: _lib.check(lib.lrb200_block_execute(h, ctypes.c_void_p(x.data_ptr()), n, ctypes.c_void_p(y.data_ptr()),
                                                       ctypes.byref(no)), "execute")
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        step()
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            step()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        for k in ("pc_reduce_kernel", "pc_scan_kernel", "pc_apply_kernel"):
            if k in ev.name:
                per.setdefault(k, []).append(ev.time_range.elapsed_us())
    lib.lrb200_block_destroy(h)
    gbs = 16.0 * n / (ms * 1e-3) / 1e9
    rows.append({"N": N, "I": I, "samples": n, "ms": round(ms, 4), "GBs": round(gbs, 1), "frac_of_3350_GBs": round(gbs / 3350.0, 4),
                 "launch_us": {k.replace("_kernel", ""): round(sum(v) / len(v), 1) for k, v in per.items()}})
print(json.dumps(rows))
"""


def run_variant(name, patches, tmp):
    d = os.path.join(tmp, name)
    shutil.copytree(os.path.join(ROOT, "luaradio_b200"), os.path.join(d, "luaradio_b200"),
                    ignore=shutil.ignore_patterns("__pycache__", "*.so"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(d, "include"))
    for rel in (SRC, HDR):
        path = os.path.join(d, rel)
        text = open(path).read()
        for old, new in patches:
            text = text.replace(old, new)
        with open(path, "w") as f:
            f.write(text)
    env = dict(os.environ, PYTHONPATH=d)
    subprocess.run([sys.executable, "-m", "luaradio_b200.build"], cwd=d, env=env, check=True, capture_output=True)
    out = subprocess.run([sys.executable, "-c", TIMER], cwd=d, env=env, check=True, capture_output=True, text=True)
    return json.loads(out.stdout.strip().splitlines()[-1])


def main():
    from tools.aux_bench import card
    result = {"card": card(), "command": "python tools/phasecorr_ablation.py", "variants": {}}
    with tempfile.TemporaryDirectory() as tmp:
        for name, patches in VARIANTS.items():
            result["variants"][name] = run_variant(name, patches, tmp)
    print(json.dumps(result))


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()
