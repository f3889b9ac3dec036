#!/usr/bin/env python3
"""Device time of the ERT receiver's front-end stages (composites/ertreceiver.lua:38-41: ComplexMagnitude ->
Lowpass(128, 4 * 32768) -> Downsampler(6)) on 2^28 samples per call in DEVICE mode, fused and unfused, alternating in
one process, timed with CUDA events around each stage (lrb200_graph_set_timing).

    fused:    one graph, "mag+fir_rrrf[fused x3]": the overlap-save FIR takes |x| at its load
    unfused:  "cmag" then "fir_rrrf[fused x2]" as two graphs, the magnitude stream going through HBM between them

Bytes per input sample are the stages' own traffic, not measured: fused 8 (complex in) + 4/6 (decimated out); unfused
8 + 4 (magnitude out) + 4 (magnitude back in) + 4/6.  GB/s is that model over the measured stage time.

    python tools/ert_bench.py [out.json] [log2_samples]
"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BAUD = 32768.0
RATE = 72 * BAUD
DECIM = 6
STEPS, WARMUP = 10, 2
BYTES = {"fused": 8 + 4 / DECIM, "unfused": 8 + 4 + 4 + 4 / DECIM}


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
    import luaradio_b200 as radio
    from luaradio_b200 import _lib
    from luaradio_b200.types import ComplexFloat32
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    n = 1 << (int(sys.argv[2]) if len(sys.argv) > 2 else 28)
    lib = _lib.require_device(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    _lib.check(lib.lrb200_set_stream(ctypes.c_void_p(stream.cuda_stream)))

    def blocks(*bs):
        rate, t = RATE, ComplexFloat32
        for b in bs:
            b.get_rate = (lambda r: (lambda: r))(rate)
            b.differentiate([t])
            b.initialize()
            t = b.get_output_type()
        return bs

    def graph(*bs):
        g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
        for b in bs:
            _lib.check(lib.lrb200_graph_append(g, b.make_device_handle()), "append")
        _lib.check(lib.lrb200_graph_commit(g, 1), "commit")
        _lib.check(lib.lrb200_graph_set_timing(g, 1), "timing")
        return g

    mag, lp, down = blocks(radio.ComplexMagnitudeBlock(), radio.LowpassFilterBlock(128, 4 * BAUD), radio.DownsamplerBlock(DECIM))
    fused = graph(mag, lp, down)
    g_mag, g_fir = graph(mag), graph(lp, down)
    descs = {"fused": lib.lrb200_graph_describe(fused).decode(),
             "unfused": lib.lrb200_graph_describe(g_mag).decode() + " ; " + lib.lrb200_graph_describe(g_fir).decode()}
    assert descs["fused"] == "mag+fir_rrrf[fused x3]" and descs["unfused"] == "cmag ; fir_rrrf[fused x2]", descs

    x = torch.empty(n, dtype=torch.complex64, device="cuda")
    _lib.check(lib.lrb200_synth_white_iq(ctypes.c_void_p(x.data_ptr()), 0, n, 1))
    m = torch.empty(n, dtype=torch.float32, device="cuda")
    y = {k: torch.empty(n // DECIM + 2, dtype=torch.float32, device="cuda") for k in ("fused", "unfused")}
    no = ctypes.c_size_t(0)

    def run(kind):
        if kind == "fused":
            _lib.check(lib.lrb200_graph_execute_device(fused, ctypes.c_void_p(x.data_ptr()), n, ctypes.c_void_p(y[kind].data_ptr()),
                                                       ctypes.byref(no)), "fused")
        else:
            _lib.check(lib.lrb200_graph_execute_device(g_mag, ctypes.c_void_p(x.data_ptr()), n, ctypes.c_void_p(m.data_ptr()),
                                                       ctypes.byref(no)), "cmag")
            _lib.check(lib.lrb200_graph_execute_device(g_fir, ctypes.c_void_p(m.data_ptr()), n, ctypes.c_void_p(y[kind].data_ptr()),
                                                       ctypes.byref(no)), "fir")
        return no.value

    def stage_ms(*gs):
        ex = ctypes.c_int(0)
        total = 0.0
        for g in gs:
            for s in range(lib.lrb200_graph_num_stages(g)):
                total += lib.lrb200_graph_stage_time_ms(g, s, ctypes.byref(ex))
        return total

    for _ in range(WARMUP):
        for kind in ("fused", "unfused"):
            run(kind)
    stage_ms(fused)
    stage_ms(g_mag, g_fir)
    times = {"fused": [], "unfused": []}
    for _ in range(STEPS):
        for kind in ("fused", "unfused"):
            run(kind)
            times[kind].append(stage_ms(fused) if kind == "fused" else stage_ms(g_mag, g_fir))
    torch.cuda.synchronize()
    # both forms compute the same stream: the FIR's own summation order differs only in where |x| is rounded (nowhere)
    a, b = y["fused"][:no.value].cpu().numpy(), y["unfused"][:no.value].cpu().numpy()
    rows = {}
    for kind in ("fused", "unfused"):
        t = np.array(times[kind])
        med = float(np.median(t))
        rows[kind] = {"graph": descs[kind], "stage_ms_median": med, "stage_ms_min": float(t.min()), "stage_ms_max": float(t.max()),
                      "bytes_per_input_sample_model": BYTES[kind], "GBs_model_over_median": BYTES[kind] * n / (med * 1e-3) / 1e9,
                      "Msamples_per_s": n / (med * 1e-3) / 1e6}
    rec = {"tool": "tools/ert_bench.py", "samples_per_call": n, "steps": STEPS, "warmup": WARMUP, "card": card(),
           "torch_device": torch.cuda.get_device_name(0), "rows": rows,
           "speedup_median": rows["unfused"]["stage_ms_median"] / rows["fused"]["stage_ms_median"],
           "outputs": int(no.value), "max_abs_diff_fused_vs_unfused": float(np.max(np.abs(a.astype(np.float64) - b))),
           "max_abs_output": float(np.max(np.abs(b)))}
    for g in (fused, g_mag, g_fir):
        lib.lrb200_graph_destroy(g)
    s = json.dumps(rec, indent=1)
    print(s)
    if out_path:
        with open(out_path, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
