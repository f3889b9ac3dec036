#!/usr/bin/env python3
"""Sharded WBFM-stereo DAG throughput (lrb200_dag_shard_*, luaradio_b200.sharding.dag_shard_step).

    torchrun --nproc_per_node N tools/dag_shard_bench.py [--samples 2**28] [--reps 3] [--out FILE]

Each rank runs 2^28 input samples (1.1025 MS/s FM stereo multiplex, PLL in mode 1, chunk-parallel) as one shard of a
stream and reports its MS/s, the begin -> end exchange time and its re-runs.  With one process it reports, on one GPU,
the plain lrb200_dag_execute_device of the same samples against (a) the world-1 shard (rank 0: the plain run plus the
PLL probe), (b) begin + end of a non-first shard whose start is accepted (halo overhead plus the split around the
exchange), and (c) the same shard with a miss (its loop run again).  Writes one JSON line with the card and its power
limit."""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from luaradio_b200 import _lib, sharding  # noqa: E402
from tests.test_gpu_dag_boundary import planned_dag, release, stereo_input, stereo_top  # noqa: E402


def gpu_name():
    import torch
    return torch.cuda.get_device_name() if torch.cuda.is_available() else None


def power_limit():
    """The card's power limit in W (a number belongs with it), read with nvidia-smi; None when it cannot be read."""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            os.environ.get("LOCAL_RANK", "0")], capture_output=True, text=True, timeout=20)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=1 << 28)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    dist = None
    if world > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        dist.init_process_group("nccl")
    lib = _lib.require_device(int(os.environ.get("LOCAL_RANK", rank)) if world > 1 else None)
    n = a.samples
    base = stereo_input(1 << 22, 31)
    top, dag = planned_dag(lambda y: stereo_top(y, parallel_pll=True), base)
    d = dag.dag
    halo = lib.lrb200_dag_halo(d)
    nb = lib.lrb200_dag_shard_record_bytes(d)
    n = n // halo * halo
    dx = lib.lrb200_malloc((halo + n) * 8)
    # the input: the 2^22-sample multiplex repeated (the pilot stays locked across the seams: its phase is continuous
    # to within the tuner's tolerance only, which the re-run count reports)
    for off in range(0, halo + n, len(base)):
        m = min(len(base), halo + n - off)
        _lib.check(lib.lrb200_memcpy_h2d(dx + off * 8, base[:m].ctypes.data, m * 8), "h2d")
    ys = [lib.lrb200_malloc(lib.lrb200_dag_max_output(d, k, halo + n) * 4) for k in range(2)]
    yp = (ctypes.c_void_p * 2)(*ys)
    n_out = (ctypes.c_size_t * 2)()

    def timed(fn):
        best = None
        for _ in range(a.reps + 1):                    # the first is the warm-up
            _lib.check(lib.lrb200_sync(), "sync")
            t0 = time.perf_counter()
            extra = fn()
            _lib.check(lib.lrb200_sync(), "sync")
            dt = time.perf_counter() - t0
            best = (dt, extra) if best is None or dt < best[0] else best
        return best

    res = {"tool": "dag_shard_bench", "gpu": gpu_name(), "power_limit_w": power_limit(), "graph": "wbfm_stereo dag (pll mode 1)",
           "samples_per_rank": n, "halo": halo, "record_bytes": nb, "world": world}
    if world == 1:
        res["multi_gpu"] = "not measured: one device"
    if world == 1:
        def plain():
            _lib.check(lib.lrb200_dag_reset(d), "reset")
            _lib.check(lib.lrb200_dag_execute_device(d, dx + halo * 8, n, yp, n_out), "execute_device")
        t_plain, _ = timed(plain)
        rec = (ctypes.c_double * (nb // 8))()
        rp = ctypes.cast(rec, ctypes.c_void_p)

        def shard(start, lead, miss=False):
            """begin, then end against a left record: for a non-first shard one whose end state is this shard's own
            speculated start (accepted: the no-miss cost), or with miss=True its own record (a re-run)."""
            def go():
                t0 = time.perf_counter()
                _lib.check(lib.lrb200_dag_shard_begin(d, dx + (halo - lead) * 8, lead, n, start, yp, n_out, rp, nb), "begin")
                t1 = time.perf_counter()
                own = list(rec)
                left = own if miss else [0.0, 0.0, own[0], 0.0, own[1], 0.0]
                la = (ctypes.c_double * len(left))(*left)
                rc = lib.lrb200_dag_shard_end(d, ctypes.cast(la, ctypes.c_void_p), 0 if start == 0 else 1, yp, n_out, rp, nb)
                assert rc in (0, 1), _lib.last_error()
                _lib.check(lib.lrb200_sync(), "sync")
                return rc, t1 - t0, time.perf_counter() - t1
            return go
        t_first, _ = timed(shard(0, 0))
        t_next, (rr, tb, te) = timed(shard(halo * 1000, halo))
        t_miss, (rm, _, _) = timed(shard(halo * 1000, halo, miss=True))
        assert rr == 0 and rm == 1
        res.update({"plain_ms": t_plain * 1e3, "plain_msps": n / t_plain / 1e6,
                    "world1_shard_ms": t_first * 1e3, "world1_shard_msps": n / t_first / 1e6,
                    "nonfirst_shard_ms": t_next * 1e3, "nonfirst_shard_msps": n / t_next / 1e6,
                    "nonfirst_begin_ms": tb * 1e3, "nonfirst_end_ms": te * 1e3,
                    "nonfirst_over_plain": t_next / t_plain,
                    "nonfirst_miss_ms": t_miss * 1e3, "nonfirst_miss_over_plain": t_miss / t_plain})
    else:
        start = rank * n
        lead = halo if rank else 0
        times = {}
        t0 = time.perf_counter()
        rr = sharding.dag_shard_step(dist, lib, d, dx + (halo - lead) * 8, lead, n, start, yp, n_out, rank, world,
                                     device="cuda", times=times)
        _lib.check(lib.lrb200_sync(), "sync")
        dt = time.perf_counter() - t0
        res.update({"rank": rank, "msps": n / dt / 1e6, "ms": dt * 1e3, "exchange_ms": times["exchange"] * 1e3,
                    "begin_ms": times["begin"] * 1e3, "end_ms": times["end"] * 1e3, "reruns": rr})
        dist.destroy_process_group()
    for y in ys:
        lib.lrb200_free(y)
    lib.lrb200_free(dx)
    release(top)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
