#!/usr/bin/env python3
"""Throughput of the device DAG at its host boundary, on 1.1025 MS/s-shaped input.

DAGs:
  stereo  TunerBlock(-250 kHz, 200 kHz, /5) -> WBFMStereoDemodulator, both de-emphasis outputs (examples/rtlsdr_wbfm_stereo.lua)
  rds     TunerBlock -> discriminator -> Hilbert -> pilot PLL x3 / delay -> mixer -> lowpass -> RRC -> phase corrector
          -> ComplexToReal, three outputs (examples/rtlsdr_rds.lua up to the clock recovery)
  fanout  complex input fanned out to two LowpassFilterBlocks joined in AddBlock: no serial block caps the rate

Configurations:
  (a) 8192-sample process() vectors (the reference's source vectors), no super-chunk
  (b) the same vectors with superchunk = 2^20
  (c) fanout only: a u8 IQFileSource of the same samples, absorbed into the DAG, with super-chunks
  (d) lrb200_dag_execute_device on 2^26 device-resident samples in one call, timed with CUDA events
and stereo and rds (b) once more with PLLBlock.parallel = True.  Host configurations are timed with a wall clock around run(),
which ends after the flush; each is warmed up on 2^20 samples first.  Every configuration's outputs are compared with a
baseline: (b) with (a) and (c) with an ArraySource of the host-converted samples, at the tolerances of
tests/test_gpu_dag_boundary.py; (d) bit for bit with lrb200_dag_execute of the same call.

    python tools/dag_bench.py --out profiles/h100_<W>w_dag_bench.json
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import luaradio_b200 as radio                                   # noqa: E402
from luaradio_b200 import _lib                                  # noqa: E402
from luaradio_b200.composite import GPUDagBlock                 # noqa: E402
from oracle import lr_oracle as O                               # noqa: E402

RATE = 1102500.0
VECTOR = 8192
SUPERCHUNK = 1 << 20


def fm_multiplex(n, seed):
    """FM stereo multiplex (L+R, 19 kHz pilot, L-R on 38 kHz) at 1.1025 MS/s, 250 kHz above the tuner's centre."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / RATE
    left, right = 0.5 * np.sin(2 * np.pi * 700 * t), 0.4 * np.sin(2 * np.pi * 2300 * t)
    mpx = 0.45 * (left + right) + 0.1 * np.sin(2 * np.pi * 19e3 * t) + 0.45 * (left - right) * np.sin(2 * np.pi * 38e3 * t)
    phase = 2 * np.pi * 75e3 * np.cumsum(mpx) / RATE + 2 * np.pi * 250e3 * t
    noise = rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n)
    return (np.exp(1j * phase) + 0.001 * noise).astype(np.complex64)


def noise(n, seed):
    rng = np.random.default_rng(seed)
    return (rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n)).astype(np.complex64)


def stereo(src, parallel=False):
    demod, sinks = radio.WBFMStereoDemodulator(), [radio.ArraySink(), radio.ArraySink()]
    for b in demod._blocks:
        if isinstance(b, radio.PLLBlock):
            b.parallel = parallel
    top = radio.CompositeBlock()
    top.connect(src, radio.TunerBlock(-250e3, 200e3, 5), demod)
    top.connect(demod, "left", sinks[0], "in")
    top.connect(demod, "right", sinks[1], "in")
    return top, sinks


def rds(src, parallel=False):
    hilbert, delay = radio.HilbertTransformBlock(129), radio.DelayBlock(129)
    pll, mixer = radio.PLLBlock(1500.0, 19e3 - 100, 19e3 + 100, 3.0), radio.MultiplyConjugateBlock()
    pll.parallel = parallel
    rrc, corr, c2r = radio.RootRaisedCosineFilterBlock(101, 1, 1187.5), radio.BinaryPhaseCorrectorBlock(8000), radio.ComplexToRealBlock()
    sinks = [radio.ArraySink() for _ in range(3)]
    top = radio.CompositeBlock()
    top.connect(src, radio.TunerBlock(-250e3, 200e3, 5), radio.FrequencyDiscriminatorBlock(1.25), hilbert, delay)
    top.connect(hilbert, radio.ComplexBandpassFilterBlock(129, [18e3, 20e3]), pll)
    top.connect(delay, "out", mixer, "in1")
    top.connect(pll, "out", mixer, "in2")
    top.connect(mixer, radio.LowpassFilterBlock(128, 4e3), rrc, corr)
    top.connect(corr, c2r, sinks[2])
    top.connect(corr, sinks[1])
    top.connect(rrc, sinks[0])
    return top, sinks


def fanout(src, parallel=False):
    first, second, add, snk = radio.LowpassFilterBlock(128, 200e3), radio.LowpassFilterBlock(65, 100e3), radio.AddBlock(), radio.ArraySink()
    top = radio.CompositeBlock()
    top.connect(src, "out", first, "in")
    top.connect(src, "out", second, "in")
    top.connect(first, "out", add, "in1")
    top.connect(second, "out", add, "in2")
    top.connect(add, snk)
    return top, [snk]


DAGS = {"stereo": (stereo, fm_multiplex), "rds": (rds, fm_multiplex), "fanout": (fanout, noise)}


def max_err(got, ref):
    if len(got) != len(ref):
        return float("inf")
    return float(np.max(np.abs(got.astype(np.complex128) - ref), initial=0.0))


def equal_within(name, got, ref):
    """The tolerances of tests/test_gpu_dag_boundary.py: fanout 1e-5 of max(1, |ref|); behind a PLL 5e-3 (the FIR kernels
    depend on the call length, and the PLL's multiplied phase keeps the sum of every past rounding difference)."""
    ok, errs = True, []
    for g, r in zip(got, ref):
        if len(g) != len(r):
            return False, None
        e = max_err(g, r)
        ok = ok and e <= (1e-5 * max(1.0, float(np.max(np.abs(r), initial=0.0))) if name == "fanout" else 5e-3)
        errs.append(e)
    return ok, errs


def timed_run(make, src_fn, superchunk, parallel=False):
    make(src_fn(1 << 20))[0].run(superchunk=superchunk)      # warm-up: modules, FIR plans, pinned slots
    src = src_fn(None)
    top, sinks = make(src, parallel)
    t0 = time.perf_counter()
    top.run(superchunk=superchunk)
    t = time.perf_counter() - t0
    return t, [s.result() for s in sinks], top.describe_gpu_graph()


def host_configs(name, n, rows):
    make, gen = DAGS[name]
    x = gen(n, 1)

    def array_src(m, chunk=VECTOR):
        return radio.ArraySource(x if m is None else x[:m], RATE, chunk)

    base = None
    configs = [("a", 0, False), ("b", SUPERCHUNK, False)] + ([("b_parallel_pll", SUPERCHUNK, True)] if name in ("stereo", "rds") else [])
    for cfg, sc, par in configs:
        t, outs, desc = timed_run(make, array_src, sc, par)
        row = {"dag": name, "config": cfg, "superchunk": sc, "pll_parallel": par, "samples": n, "seconds": t, "msps": n / t / 1e6,
               "describe": desc}
        if base is None:
            base = outs
            row["outputs_equal"], row["max_err"] = True, [0.0] * len(outs)
        else:
            row["outputs_equal"], row["max_err"] = equal_within(name, outs, base)
            if par:
                row["outputs_equal_note"] = ("the chunk-parallel PLL re-runs every chunk whose lead-in missed the carried loop "
                                             "state, so it equals the serial one on any input")
        rows.append(row)
        print(json.dumps({k: v for k, v in row.items() if k != "describe"}), flush=True)
    if name == "fanout":
        # (c) the same samples as u8 bytes in a file, absorbed: compared with (b) on the host-converted samples
        raw = np.clip(np.round(np.stack([x.real, x.imag], 1).reshape(-1) * 127.5 + 127.5), 0, 255).astype(np.uint8)
        conv = O.iq_file_convert(raw, "u8")

        def file_src(m):
            return radio.IQFileSource((raw if m is None else raw[:2 * m]).tobytes(), "u8", RATE)
        t, outs, desc = timed_run(make, file_src, SUPERCHUNK)
        top, sinks = make(radio.ArraySource(conv, RATE, GPUDagBlock.RAW_READ))
        top.run(superchunk=SUPERCHUNK)
        ok, errs = equal_within(name, outs, [s.result() for s in sinks])
        row = {"dag": name, "config": "c", "superchunk": SUPERCHUNK, "samples": n, "seconds": t, "msps": n / t / 1e6,
               "describe": desc, "absorbed": desc.startswith("dag{iqconv(u8)"), "outputs_equal": ok, "max_err": errs}
        rows.append(row)
        print(json.dumps({k: v for k, v in row.items() if k != "describe"}), flush=True)


def planned(name, n):
    make, _ = DAGS[name]
    top, _ = make(radio.ArraySource(np.zeros(16, np.complex64), RATE))
    top._prepare_to_run()
    top._collapse_gpu_runs(True, 0)
    return top, next(c for c in top._chains if isinstance(c, GPUDagBlock))


def device_config(name, n_log2, reps, rows):
    import torch
    lib = _lib.require_device()
    n = 1 << n_log2
    x = torch.from_numpy(DAGS[name][1](n, 2))
    top_h, dag_h = planned(name, n)
    top_d, dag_d = planned(name, n)
    k_out = len(dag_d.ext_out)
    dts = [torch.complex64 if p.data_type.dtype == np.complex64 else torch.float32 for p in dag_d.ext_out]
    # host mode, one call: the baseline outputs
    outs_h = [torch.empty(lib.lrb200_dag_max_output(dag_h.dag, k, n), dtype=dts[k]) for k in range(k_out)]
    n_out = (ctypes.c_size_t * k_out)()
    _lib.check(lib.lrb200_dag_execute(dag_h.dag, x.data_ptr(), n, (ctypes.c_void_p * k_out)(*[o.data_ptr() for o in outs_h]), n_out), "dag_execute")
    want = [outs_h[k][:n_out[k]].clone() for k in range(k_out)]
    for c in top_h._chains:
        c.cleanup()
    dx = x.cuda()
    dys = [torch.empty(lib.lrb200_dag_max_output(dag_d.dag, k, n), dtype=dts[k], device="cuda") for k in range(k_out)]
    ptrs = (ctypes.c_void_p * k_out)(*[d.data_ptr() for d in dys])
    stream = torch.cuda.ExternalStream(lib.lrb200_get_stream())
    times, equal = [], None
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        _lib.check(lib.lrb200_dag_execute_device(dag_d.dag, dx.data_ptr(), n, ptrs, n_out), "dag_execute_device")
        e1.record(stream)
        e1.synchronize()
        if r == 0:                                           # the first call from a fresh DAG: compare with host mode
            equal = all(n_out[k] == len(want[k]) and
                        np.array_equal(dys[k][:n_out[k]].cpu().numpy().view(np.uint8), want[k].numpy().view(np.uint8))
                        for k in range(k_out))
        else:
            times.append(e0.elapsed_time(e1) * 1e-3)
    for c in top_d._chains:
        c.cleanup()
    t = float(np.median(times))
    row = {"dag": name, "config": "d", "samples": n, "seconds": t, "all_s": times, "msps": n / t / 1e6, "outputs_equal": bool(equal),
           "outputs_equal_note": "bit for bit against lrb200_dag_execute of the same call"}
    rows.append(row)
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=23, help="log2 of the samples of the host configurations")
    ap.add_argument("--device-n", type=int, default=26, help="log2 of the samples of the DEVICE-mode call")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dags", default="stereo,rds,fanout")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    _lib.require_device()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    rows = []
    for name in args.dags.split(","):
        host_configs(name, 1 << args.n, rows)
        device_config(name, args.device_n, args.reps, rows)
    rec = {"gpu": smi, "input_rate": RATE, "vector": VECTOR, "results": rows}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
