#!/usr/bin/env python3
"""Device-side throughput of the kernels on the rows next to the hot path (SURVEY.md 8f): file sample-format converters
at the graph boundaries, the resampling family, level control (AGCBlock, PowerSquelchBlock, the rx_am envelope chain) and
BinaryPhaseCorrectorBlock (with the RDS signal path end to end).  One JSON object; achieved GB/s counts ALGORITHMIC bytes (input +
output of the block), against the measured HBM peak (MEASURED_PEAKS.json, see bench.peaks()).

    python tools/aux_bench.py [--samples N] [--steps K] [--only-level | --only-phasecorr] > profiles/rNN_aux_bench.json
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=1 << 28)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--only-resample", action="store_true", help="skip the file-format rows")
    ap.add_argument("--only-level", action="store_true", help="only the level-control rows")
    ap.add_argument("--only-phasecorr", action="store_true", help="only the BinaryPhaseCorrectorBlock and RDS-path rows")
    args = ap.parse_args()
    import torch
    import luaradio_b200 as radio
    from luaradio_b200 import _lib
    import bench
    lib = _lib.require_device(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    _lib.check(lib.lrb200_set_stream(ctypes.c_void_p(stream.cuda_stream)))
    D = _lib.LRB200_DEVICE
    n = args.samples
    peak, src = bench.peaks()
    x = torch.empty(n, dtype=torch.complex64, device="cuda")
    _lib.check(lib.lrb200_synth_white_iq(ctypes.c_void_p(x.data_ptr()), 0, n, 1))
    xs = x * 0.7                                   # inside [-1, 1] for the sink converters
    raw = torch.empty(n * 16, dtype=torch.uint8, device="cuda")
    y = torch.empty(n * 2 + 64, dtype=torch.complex64, device="cuda")
    rows = []

    def timed(name, make, in_ptr, n_in, out_ptr, bytes_per_in, note=""):
        g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
        for h in make():
            _lib.check(lib.lrb200_graph_append(g, _lib.check_handle(h, name)), "append")
        _lib.check(lib.lrb200_graph_commit(g, 1), "commit")
        no = ctypes.c_size_t(0)

        def step():
            _lib.check(lib.lrb200_graph_reset(g), "reset")
            _lib.check(lib.lrb200_graph_execute_device(g, ctypes.c_void_p(in_ptr), n_in, ctypes.c_void_p(out_ptr), ctypes.byref(no)), name)

        for _ in range(3):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            step()
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        gbs = bytes_per_in * n_in / (ms * 1e-3) / 1e9
        rows.append({"kernel": name, "graph": lib.lrb200_graph_describe(g).decode(), "input_samples": n_in, "output_samples": no.value,
                     "ms": round(ms, 4), "msamples_per_s": round(n_in / ms / 1e3, 1), "algorithmic_bytes_per_input_sample": bytes_per_in,
                     "hbm_GBs": round(gbs, 1), "frac_of_peak": round(gbs / peak, 4), "note": note})
        lib.lrb200_graph_destroy(g)

    def timed_calls(name, h, in_ptr, n_in, call, out_ptr, bytes_per_in, note=""):
        """One block handle (DEVICE pointers) fed `call` samples per execute, state carried: the reference's per-vector
        regime.  A step is n_in samples in n_in / call launches."""
        no = ctypes.c_size_t(0)
        h = _lib.check_handle(h, name)
        es = bytes_per_in // 2                       # element size: input and output have the same type

        def step():
            for k in range(0, n_in, call):
                _lib.check(lib.lrb200_block_execute(h, ctypes.c_void_p(in_ptr + k * es), min(call, n_in - k),
                                                    ctypes.c_void_p(out_ptr + k * es), ctypes.byref(no)), name)

        step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            step()
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        gbs = bytes_per_in * n_in / (ms * 1e-3) / 1e9
        rows.append({"kernel": name, "graph": lib.lrb200_block_name(h).decode(), "input_samples": n_in, "samples_per_call": call,
                     "ms": round(ms, 4), "msamples_per_s": round(n_in / ms / 1e3, 1), "algorithmic_bytes_per_input_sample": bytes_per_in,
                     "hbm_GBs": round(gbs, 1), "frac_of_peak": round(gbs / peak, 4), "note": note})
        lib.lrb200_block_destroy(h)

    if args.only_level:
        level_rows(lib, _lib, radio, timed, timed_calls, x, y, n)
        print(json.dumps({"peak_GBs": peak, "peak_source": src, "samples": n, "steps": args.steps, "rows": rows}))
        return
    if args.only_phasecorr:
        phasecorr_rows(lib, timed, timed_calls, x, y, n, rows, args.steps)
        print(json.dumps({"card": card(), "peak_GBs": peak, "peak_source": src, "samples": n, "steps": args.steps, "rows": rows}))
        return

    # ---- file formats: fill `raw` with the sink's own output so the source converters read realistic bytes
    for fmt, b in (() if args.only_resample else (("u8", 1), ("s16le", 2), ("f32be", 4))):
        timed("iqsink(%s)" % fmt, lambda: [lib.lrb200_iqsink_create(fmt.encode(), D)], xs.data_ptr(), n, raw.data_ptr(), 8 + 2 * b)
        timed("iqconv(%s)" % fmt, lambda: [lib.lrb200_iqconv_create(fmt.encode(), D)], raw.data_ptr(), n, y.data_ptr(), 2 * b + 8)
    if not args.only_resample:
        timed("realsink(s16le)", lambda: [lib.lrb200_realsink_create(b"s16le", D)], xs.data_ptr(), 2 * n, raw.data_ptr(), 4 + 2,
              "WAVFileSink, 16 bits per sample")
    # ---- resampling family (LowpassFilterBlock(128, 1/L or min(1/L, 1/D), nyquist 1.0) taps)
    for L, Dn in ((2, 1), (3, 1), (4, 1), (8, 1), (2, 3), (3, 2), (5, 4), (2, 5), (160, 147)):
        m = n // (2 * L) if Dn == 1 else n // 2
        taps = np.array(radio.filter_utils.firwin_lowpass(128, min(1.0 / L, 1.0 / Dn)), np.float32)

        def make():
            hs = [lib.lrb200_mulconst_create(float(L), 0.0, 1, 0, D), lib.lrb200_upsample_create(L, 8, D),
                  lib.lrb200_fir_create_crcf(taps.ctypes.data, 128, 1, D)]
            if Dn > 1:
                hs.append(lib.lrb200_downsample_create(Dn, 8, D))
            return hs
        timed("interpolator x%d" % L if Dn == 1 else "rational resampler %d/%d" % (L, Dn), make, x.data_ptr(), m, y.data_ptr(),
              8 + 8.0 * L / Dn, "128 taps, complex")
    level_rows(lib, _lib, radio, timed, timed_calls, x, y, n)
    phasecorr_rows(lib, timed, timed_calls, x, y, n, rows, args.steps)
    print(json.dumps({"peak_GBs": peak, "peak_source": src, "samples": n, "steps": args.steps, "rows": rows}))


def level_rows(lib, _lib, radio, timed, timed_calls, x, y, n):
    """AGCBlock('slow') and PowerSquelchBlock(-40) at 1 MS/s on white noise (the gate open throughout: the costly case), the
    AGC once more with the gate closed throughout (the copy), each as one call of n samples and as 8192-sample calls, and
    the rx_am envelope chain (rx_am.lua:51-55) at 1.1025 MS/s.  Real rows read the I/Q words as n Float32 samples."""
    from luaradio_b200.types import ComplexFloat32
    D = _lib.LRB200_DEVICE
    for cplx, bpi in ((0, 8), (1, 16)):
        kind = "complex" if cplx else "real"
        for label, mk in (("agc(slow) %s" % kind, lambda: lib.lrb200_agc_create(-35.0, -75.0, 3.0, 1.0, 1e6, cplx, D)),
                          ("agc(slow) %s, gate closed" % kind, lambda: lib.lrb200_agc_create(-35.0, 30.0, 3.0, 1.0, 1e6, cplx, D)),
                          ("powersquelch(-40) %s" % kind, lambda: lib.lrb200_powersquelch_create(-40.0, 0.001, 1e6, cplx, D))):
            timed(label, lambda: [mk()], x.data_ptr(), n, y.data_ptr(), bpi, "one call")
            timed_calls(label + ", 8192-sample calls", mk(), x.data_ptr(), n // 16, 8192, y.data_ptr(), bpi,
                        "the reference's vector size, one launch per call")
    rate = 1102500.0

    def dev(blk, in_type, r):
        blk.get_rate = lambda: r
        blk.differentiate([in_type])
        blk.initialize()
        h = blk.make_device_handle()
        blk.cleanup()
        return h

    def envelope_chain():
        from luaradio_b200.types import Float32
        af = rate / 25
        return [dev(radio.FrequencyTranslatorBlock(-50e3), ComplexFloat32, rate), dev(radio.LowpassFilterBlock(128, 5e3), ComplexFloat32, rate),
                dev(radio.DownsamplerBlock(25), ComplexFloat32, rate), dev(radio.ComplexMagnitudeBlock(), ComplexFloat32, af),
                dev(radio.SinglepoleHighpassFilterBlock(100), Float32, af), dev(radio.LowpassFilterBlock(128, 5e3), Float32, af),
                dev(radio.AGCBlock("slow"), Float32, af)]
    timed("rx_am envelope chain", envelope_chain, x.data_ptr(), n, y.data_ptr(), 8 + 4.0 / 25,
          "Tuner(-50e3, 10e3, 25) -> AMEnvelopeDemodulator(5e3) -> AGCBlock('slow'); bytes = chain input + output")


def card():
    """The card the rows ran on: name, power limit and SM clocks, read (not set) through nvidia-smi."""
    import subprocess
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:                       # the rows stand without it; say why it is missing
        return {"error": str(e)}
    return dict(zip(("name", "power_limit", "clocks_max_sm", "clocks_sm"), (v.strip() for v in out.split(","))))


def phasecorr_rows(lib, timed, timed_calls, x, y, n, rows, steps):
    """BinaryPhaseCorrectorBlock on white noise, 16 algorithmic bytes per sample (x read once, y written once), for
    (N, I) = (8000, 32) (the RDS example), (50, 32) (BPSK31) and (4, 1) (a measurement every sample): one call of n samples,
    and n / 16 samples in 8192- and 131072-sample calls.  Then the RDS signal path (examples/rtlsdr_rds.lua, TunerBlock to
    ComplexToRealBlock) end to end through CompositeBlock.run from host memory, with the PLL serial and chunk-parallel."""
    import time
    import numpy as np
    import luaradio_b200 as radio
    from luaradio_b200 import _lib
    D = _lib.LRB200_DEVICE
    for N, I in ((8000, 32), (50, 32), (4, 1)):
        label = "phasecorr(%d, %d)" % (N, I)
        mk = lambda: lib.lrb200_phasecorrector_create(N, I, D)
        timed(label, lambda: [mk()], x.data_ptr(), n, y.data_ptr(), 16, "one call")
        for call in (8192, 131072):
            timed_calls(label + ", %d-sample calls" % call, mk(), x.data_ptr(), n // 16, call, y.data_ptr(), 16,
                        "one block, three launches per call")
    rate, m = 1102500.0, 1 << 24
    rng = np.random.default_rng(1)
    t = np.arange(m) / rate
    mpx = 0.4 * np.sin(2 * np.pi * 700 * t) + 0.1 * np.sin(2 * np.pi * 19e3 * t) + 0.05 * np.sin(2 * np.pi * 57e3 * t)
    xs = (np.exp(1j * (2 * np.pi * 75e3 * np.cumsum(mpx) / rate + 2 * np.pi * 250e3 * t))
          + 0.01 * (rng.standard_normal(m) + 1j * rng.standard_normal(m))).astype(np.complex64)
    for parallel in (False, True):
        def run():
            src = radio.ArraySource(xs, rate, 1 << 22)
            hil, dly = radio.HilbertTransformBlock(129), radio.DelayBlock(129)
            pll, mix = radio.PLLBlock(1500.0, 19e3 - 100, 19e3 + 100, 3.0), radio.MultiplyConjugateBlock()
            pll.parallel = parallel
            rrc, bpc = radio.RootRaisedCosineFilterBlock(101, 1, 1187.5), radio.BinaryPhaseCorrectorBlock(8000)
            top = radio.CompositeBlock()
            top.connect(src, radio.TunerBlock(-250e3, 200e3, 5), radio.FrequencyDiscriminatorBlock(1.25), hil, dly)
            top.connect(hil, radio.ComplexBandpassFilterBlock(129, [18e3, 20e3]), pll)
            top.connect(dly, "out", mix, "in1")
            top.connect(pll, "out", mix, "in2")
            top.connect(mix, radio.LowpassFilterBlock(128, 4e3), rrc, bpc)
            top.connect(bpc, radio.ComplexToRealBlock(), radio.ArraySink())
            top.connect(bpc, radio.ArraySink())
            top.connect(rrc, radio.ArraySink())
            t0 = time.perf_counter()
            top.run()
            return time.perf_counter() - t0, top.describe_gpu_graph()
        run()
        secs = [run() for _ in range(max(1, steps // 5))]
        s, desc = min(secs)
        rows.append({"kernel": "rds path, PLL %s" % ("chunk-parallel" if parallel else "serial"), "graph": desc,
                     "input_samples": m, "ms": round(s * 1e3, 2), "msamples_per_s": round(m / s / 1e6, 2),
                     "note": "CompositeBlock.run wall time from host memory (pageable), best of %d; PLL-bound" % len(secs)})


if __name__ == "__main__":
    main()
