#!/usr/bin/env python3
"""The POCSAG receiver's mark/space detector (composites/pocsagreceiver.lua:28-45) fused and unfused, and both FSK
receivers' signal paths end to end (examples/rtlsdr_pocsag.lua, rtlsdr_ax25.lua up to the data filter).

  * detector: the device DAG of the detector alone, lrb200_dag_execute_device on 2^26-sample DEVICE calls, timed with CUDA
    events per call, fused (`fsk_detect(129)[fused x5]`) and unfused (fuse=False: two `fir_cccf | cmag` graphs and a
    Subtract) alternated in one process after a warm-up.  Model traffic per input sample: fused 8 B in + 4 B out = 12 B;
    unfused 2 x (8 in + 8 out + 8 in + 4 out) + 2 x 4 in + 4 out = 68 B.
  * the same two DAGs on 13 107-sample DEVICE calls (one 2^20-sample super-chunk after the ÷80 tuner), 256 calls per
    timed batch, five batches each.
  * receivers: a 2^24-sample capture at 1 MS/s, 8192-sample source vectors and super-chunks of 2^20, seven rounds
    alternated: POCSAG with the DAG rewrite and without it (linear graphs fused in both), AX.25.  Wall clock of the set-up
    (planning, block creation, DAG commit) and of the stream (the scheduler loop to the last output, then a device
    synchronise) separately.

    python tools/fsk_bench.py [out.json] [log2_detector_samples]
"""
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from ert_bench import card  # noqa: E402

STEPS, WARMUP = 10, 2
ROUNDS = 7
BYTES = {"fused": 12.0, "unfused": 68.0}
HBM_TBS = 3.35


def main():
    import numpy as np
    import torch
    from luaradio_b200 import _lib
    from tests import fsk_ref as K
    from tests import test_gpu_fsk as T
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    n = 1 << (int(sys.argv[2]) if len(sys.argv) > 2 else 26)
    lib = _lib.require_device(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    _lib.check(lib.lrb200_set_stream(ctypes.c_void_p(stream.cuda_stream)))
    rec = {"card": card(), "device": torch.cuda.get_device_name(0), "samples_per_call": n, "steps": STEPS,
           "warmup": WARMUP}

    # ---- detector stage, DEVICE mode
    x = torch.from_numpy(K.fsk_iq(n, 1, offset=0.0, rate=K.RATE).view(np.float32)).cuda()
    y = torch.empty(n, dtype=torch.float32, device="cuda")
    small = K.fsk_iq(1 << 16, 2, offset=0.0, rate=K.RATE)
    dags, tops = {}, []
    for mode in ("fused", "unfused"):
        top, dag = T.dag_of(T.detector_top, small, mode == "fused")
        tops.append(top)
        dags[mode] = dag
        rec["describe_" + mode] = dag.desc
    times = {m: [] for m in dags}
    outs = {}
    n_out = (ctypes.c_size_t * 1)()
    for it in range(WARMUP + STEPS):
        for mode, dag in dags.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            _lib.check(lib.lrb200_dag_execute_device(dag.dag, ctypes.c_void_p(x.data_ptr()), n,
                                                     (ctypes.c_void_p * 1)(y.data_ptr()), n_out), "execute_device")
            e1.record(stream)
            e1.synchronize()
            if it >= WARMUP:
                times[mode].append(e0.elapsed_time(e1))
            if it == WARMUP + STEPS - 1:
                outs[mode] = y.cpu().numpy().copy()
            _lib.check(lib.lrb200_dag_reset(dag.dag), "reset")
    det = {}
    for mode, t in times.items():
        med = float(np.median(t))
        det[mode] = {"ms_median": med, "ms_min": float(min(t)), "ms_max": float(max(t)),
                     "model_bytes_per_sample": BYTES[mode], "model_GBps": BYTES[mode] * n / (med * 1e-3) / 1e9,
                     "share_of_3.35TBps": BYTES[mode] * n / (med * 1e-3) / (HBM_TBS * 1e12)}
    det["speedup_median"] = det["unfused"]["ms_median"] / det["fused"]["ms_median"]
    det["bit_identical"] = bool(np.array_equal(outs["fused"].view(np.uint32), outs["unfused"].view(np.uint32)))
    rec["detector"] = det
    for t in tops:
        for c in t._chains:
            c.cleanup()
    del x, y
    torch.cuda.empty_cache()

    # ---- the detector at the receiver's per-call length: one super-chunk of 2^20 capture samples is 13 107 detector inputs
    calls = 256
    m = (1 << 20) // K.DECIM
    xs = torch.from_numpy(K.fsk_iq(m, 5, offset=0.0, rate=K.RATE).view(np.float32)).cuda()
    ys = torch.empty(m, dtype=torch.float32, device="cuda")
    dags, tops = {}, []
    for mode in ("fused", "unfused"):
        top, dag = T.dag_of(T.detector_top, small, mode == "fused")
        tops.append(top)
        dags[mode] = dag
    per = {mode: [] for mode in dags}
    for it in range(WARMUP + 5):
        for mode, dag in dags.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(calls):
                _lib.check(lib.lrb200_dag_execute_device(dag.dag, ctypes.c_void_p(xs.data_ptr()), m,
                                                         (ctypes.c_void_p * 1)(ys.data_ptr()), n_out), "execute_device")
            e1.record(stream)
            e1.synchronize()
            if it >= WARMUP:
                per[mode].append(e0.elapsed_time(e1) * 1e3 / calls)
    rec["detector_13107_sample_calls_us"] = {mode: {"median": float(np.median(t)), "min": float(min(t)), "max": float(max(t))}
                                             for mode, t in per.items()}
    for t in tops:
        for c in t._chains:
            c.cleanup()

    # ---- receivers: wall clock of the set-up (planning, block creation, DAG commit) and of the stream, rounds alternated
    cap = K.fsk_iq(1 << 24, 3)
    afsk = K.afsk_nbfm_iq(1 << 24, 4)
    e2e = {}
    for rep in range(ROUNDS):
        for name, make, xx, rewrite in (("pocsag", T.pocsag_top, cap, True), ("pocsag_no_dag_rewrite", T.pocsag_top, cap, False),
                                        ("ax25", T.ax25_top, afsk, True)):
            for sc in (0, 1 << 20):
                top, sinks = make(xx)
                with T.dag_rewrites(rewrite):
                    t0 = time.perf_counter()
                    top._prepare_to_run()
                    top._stop_requested = False
                    top._collapse_gpu_runs(True, sc)
                    t1 = time.perf_counter()
                    try:
                        top._schedule()
                        torch.cuda.synchronize()
                        t2 = time.perf_counter()
                    finally:
                        for c in top._chains:
                            c.cleanup()
                key = "%s_%s" % (name, "superchunk_2^20" if sc else "vectors_8192")
                e2e.setdefault(key, {"setup_s": [], "stream_s": [], "describe": top.describe_gpu_graph(),
                                     "outputs": len(sinks[0].result())})
                e2e[key]["setup_s"].append(t1 - t0)
                e2e[key]["stream_s"].append(t2 - t1)
    for v in e2e.values():
        tot = [a + b for a, b in zip(v["setup_s"], v["stream_s"])]
        v["MSps_median"] = (1 << 24) / float(np.median(tot)) / 1e6
        v["stream_MSps_median"] = (1 << 24) / float(np.median(v["stream_s"])) / 1e6
    rec["receivers_2^24_capture"] = e2e
    txt = json.dumps(rec, indent=1)
    print(txt)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
