"""The device DAG's host boundary: super-chunk mode, DEVICE-mode execute and an absorbed raw file source.

  * super-chunk equals streaming: the WBFM-stereo, AM-synchronous and RDS receivers and a fan-out DAG with no PLL, fed in
    the reference's 8192-sample vectors, give the same stream with `run(superchunk=S)` as with `run()`, for slots of whole
    vectors, of 2^20 samples, of a size no decimation divides, and smaller than one vector; the flush at end of stream
    drains a partial and an empty last slot, and a second run() of the same top block starts clean;
  * the WBFM-stereo DAG in super-chunks with the chunk-parallel PLL equals the one with the serial PLL once locked;
  * lrb200_dag_execute_device returns bit for bit what lrb200_dag_execute returns for the same call lengths;
  * DEVICE-mode bounds: guard-banded, poisoned buffers at aligned and unaligned offsets (the harness of
    tests/test_gpu_bounds.py);
  * a u8 IQFileSource / f32 RealFileSource read by a DAG alone is absorbed: the converter is the DAG's first node, and the
    file's chunks reach the DAG with no conversion call of their own;
  * API errors leave the DAG usable, and a reset in the middle of a super-chunk gives a fresh DAG.

A super-chunked run makes exactly the DAG calls that streaming in vectors of the slot size makes, so those two runs are
compared bit for bit.  Against the reference's 8192-sample vectors the FIR kernels differ (FirBlock::path chooses them by
call length), so the outputs agree to float32 rounding: for the fan-out DAG within the stream tolerance of the other
tests, 1e-5 of max(1, |ref|).  Behind a PLL the rounding differences are amplified while it acquires, and the multiplied
phase keeps the sum of every past phase error (pll.lua:155-157), so what they leave grows with the stream: those DAGs are
held to 5e-3, the acquisition bound of tests/test_gpu_dag.py, over streams of 2^22 input samples."""
import ctypes

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from luaradio_b200.composite import GPUDagBlock
from oracle import lr_oracle as O
from tests.test_gpu_bounds import GUARD, POISON_A, SENTINELS, Guarded
from tests.test_gpu_dag import rnd_c, stereo_mpx
from tests.test_gpu_rds import rds_input, rds_top

pytestmark = pytest.mark.gpu

RATE = 1102500.0
VECTOR = 8192                        # the reference's source vectors (iqfile.lua:52, zero.lua:30)
N = 1 << 22
SUPERCHUNKS = (VECTOR * 128, 1 << 20, 100003, 4096)


def stereo_input(n, seed):
    """An FM stereo multiplex at 1.1025 MS/s, 250 kHz above the tuner's centre."""
    x, _, _ = stereo_mpx(n, RATE, np.random.default_rng(seed))
    return (x * np.exp(2j * np.pi * 250e3 / RATE * np.arange(n))).astype(np.complex64)


def stereo_top(x, chunk=VECTOR, src=None, parallel_pll=False):
    src = src if src is not None else radio.ArraySource(x, RATE, chunk)
    demod, sinks = radio.WBFMStereoDemodulator(), [radio.ArraySink(), radio.ArraySink()]
    for b in demod._blocks:
        if isinstance(b, radio.PLLBlock):
            b.parallel = parallel_pll
    top = radio.CompositeBlock()
    top.connect(src, radio.TunerBlock(-250e3, 200e3, 5), demod)
    top.connect(demod, "left", sinks[0], "in")
    top.connect(demod, "right", sinks[1], "in")
    return top, sinks


def am_top(x, chunk=VECTOR):
    snk = radio.ArraySink()
    top = radio.CompositeBlock()
    top.connect(radio.ArraySource(x, 48000.0, chunk), radio.AMSynchronousDemodulator(5000.0, 5e3), snk)
    return top, [snk]


def am_input(n, seed):
    rate, rng = 48000.0, np.random.default_rng(seed)
    t = np.arange(n) / rate
    env = 0.5 * (1 + 0.5 * np.sin(2 * np.pi * 440 * t))
    return (env * np.exp(2j * np.pi * 5003.0 * t + 0.7j) + 0.002 * rnd_c(rng, n)).astype(np.complex64)


def fanout_top(x, chunk=VECTOR, src=None, real=False):
    """Input fanned out to two filters that join in AddBlock: no serial block caps the rate."""
    src = src if src is not None else radio.ArraySource(x, RATE, chunk)
    first = radio.LowpassFilterBlock(128, 200e3)
    second = radio.HighpassFilterBlock(65, 100e3) if real else radio.LowpassFilterBlock(65, 100e3)
    add, snk = radio.AddBlock(), radio.ArraySink()
    top = radio.CompositeBlock()
    top.connect(src, "out", first, "in")
    top.connect(src, "out", second, "in")
    top.connect(first, "out", add, "in1")
    top.connect(second, "out", add, "in2")
    top.connect(add, snk)
    return top, [snk]


def cmp_stereo(got, ref, what):
    # tests/test_gpu_dag.py::test_wbfm_stereo_demodulator_dag: 5e-3 while the PLL acquires, 5e-4 once it is locked
    lock = 60000
    d = np.abs(got.astype(np.float64) - ref)
    assert float(d[:lock].max(initial=0)) <= 5e-3, "%s: acquisition: max err %.3g" % (what, float(d[:lock].max()))
    assert float(d[lock:].max(initial=0)) <= 5e-4, "%s: locked: max err %.3g" % (what, float(d[lock:].max(initial=0)))


def cmp_rel(rel):
    def cmp(got, ref, what):
        tol = rel * max(1.0, float(np.max(np.abs(ref), initial=0)))
        err = float(np.max(np.abs(got.astype(np.complex128) - ref), initial=0))
        assert err <= tol, "%s: max abs err %.3g > %.3g" % (what, err, tol)
    return cmp


def cmp_abs(tol):
    def cmp(got, ref, what):
        err = float(np.max(np.abs(got.astype(np.complex128) - ref), initial=0))
        assert err <= tol, "%s: max abs err %.3g > %.3g" % (what, err, tol)
    return cmp


CASES = {
    # name: (top builder, input, comparison with 8192-sample streaming, comparison for equal call lengths)
    "stereo": (stereo_top, lambda: stereo_input(N, 31), cmp_abs(5e-3), cmp_stereo),
    "am_synchronous": (am_top, lambda: am_input(N, 32), cmp_abs(5e-3), cmp_abs(5e-5)),
    "rds": (lambda x, chunk=VECTOR: rds_top(x, RATE, chunk, tuner=True), lambda: rds_input(N, RATE, 33), cmp_abs(5e-3), cmp_rel(5e-5)),
    "fanout": (fanout_top, lambda: rnd_c(np.random.default_rng(34), N), cmp_rel(1e-5), cmp_rel(1e-5)),
}


def run_top(make, x, superchunk):
    top, sinks = make(x)
    top.run(superchunk=superchunk)
    dags = [c for c in top._chains if isinstance(c, GPUDagBlock)]
    assert len(dags) == 1 and dags[0].superchunk == superchunk, top.describe_gpu_graph()
    return top, [s.result() for s in sinks]


@pytest.mark.parametrize("name", list(CASES))
def test_superchunk_equals_streaming(name):
    make, gen, cmp, _ = CASES[name]
    x = gen()
    _, ref = run_top(make, x, 0)
    assert all(len(r) > 0 for r in ref)
    for S in SUPERCHUNKS:
        _, got = run_top(make, x, S)
        _, same = run_top(lambda y: make(y, chunk=S), x, 0)        # streaming in vectors of S: the same DAG calls
        for k, (g, r, e) in enumerate(zip(got, ref, same)):
            assert len(g) == len(r) == len(e), "S=%d port %d: %d samples, streaming gave %d" % (S, k, len(g), len(r))
            assert np.array_equal(g.view(np.uint8), e.view(np.uint8)), "S=%d port %d differs from streaming in S-sample vectors" % (S, k)
            cmp(g, r, "S=%d port %d" % (S, k))


@pytest.mark.parametrize("S", [1 << 20, 5 * (2 * 50536 + 1)])         # PLL calls of 5 chunks; of 2 L + 1 (a 1-sample chunk)
def test_stereo_superchunk_with_the_chunk_parallel_pll(S):
    """The WBFM-stereo DAG in super-chunks with PLLBlock.parallel = True against the same DAG with the serial PLL.  A
    slot hands the PLL S / 5 samples, more than 2 L = 101072, so every call but the partial last one runs the
    chunk-parallel form; its first chunk is exact and the loop has locked before the second chunk's lead-in starts.
    Once locked (the lock index of cmp_stereo) the parallel PLL's output is within out_tol of tests/pll_ref.py of the
    serial one, and the mixer, the two low-pass filters, Add / Subtract and the de-emphasis keep that
    below 10 out_tol of the audio; before, both are held to the acquisition bound."""
    from tests import pll_ref as P
    x = stereo_input(N, 39)
    _, serial = run_top(stereo_top, x, S)
    top, par = run_top(lambda y: stereo_top(y, parallel_pll=True), x, S)
    assert "pll" in top.describe_gpu_graph()
    lock = 60000
    for k, (g, r) in enumerate(zip(par, serial)):
        assert len(g) == len(r) > lock
        d = np.abs(g.astype(np.float64) - r)
        print("port %d: parallel vs serial PLL %.3g before lock, %.3g after" % (k, float(d[:lock].max()), float(d[lock:].max())))
        assert float(d[:lock].max()) <= 5e-3
        assert float(d[lock:].max()) <= 10 * P.out_tol(-(-(N // 5) // 50536)), "port %d: locked: %.3g" % (k, float(d[lock:].max()))


def test_superchunk_second_run_and_partial_last_slot():
    """A second run() of the same top block starts from a clean DAG; a stream that ends inside a slot and one that ends on
    a slot boundary both drain completely."""
    x = rnd_c(np.random.default_rng(35), 3 * (1 << 20) + 12345)
    _, ref = run_top(fanout_top, x, 0)
    src = radio.ArraySource(x, RATE, VECTOR)
    top, sinks = fanout_top(x, src=src)
    for S in (1 << 20, 1 << 20, 100003):                 # the same size twice, then another; every stream ends mid-slot
        src.pos, sinks[0].chunks = 0, []
        top.run(superchunk=S)
        got = sinks[0].result()
        assert len(got) == len(ref[0])
        cmp_rel(1e-5)(got, ref[0], "S=%d" % S)
    # a stream of whole slots: the last one is full and the partial slot empty at the flush
    y = x[:2 * (1 << 20)]
    _, ref = run_top(fanout_top, y, 0)
    _, got = run_top(fanout_top, y, 1 << 19)
    assert len(got[0]) == len(ref[0])
    cmp_rel(1e-5)(got[0], ref[0], "whole slots")


# ---- the C ABI on a DAG the scheduler builds --------------------------------------------------------------------------
def planned_dag(make, x):
    """The GPUDagBlock the scheduler makes of `make`'s graph, initialised (a live lrb200_dag_t in .dag)."""
    top, _ = make(x)
    top._prepare_to_run()
    top._collapse_gpu_runs(True, 0)
    dags = [c for c in top._chains if isinstance(c, GPUDagBlock)]
    assert len(dags) == 1
    return top, dags[0]


def release(top):
    for c in top._chains:
        c.cleanup()


def host_execute(lib, dag, x):
    outs = [np.zeros(max(1, lib.lrb200_dag_max_output(dag.dag, k, len(x))), p.data_type.dtype) for k, p in enumerate(dag.ext_out)]
    ptrs = (ctypes.c_void_p * len(outs))(*[o.ctypes.data for o in outs])
    n_out = (ctypes.c_size_t * len(outs))()
    _lib.check(lib.lrb200_dag_execute(dag.dag, x.ctypes.data if len(x) else None, len(x), ptrs, n_out), "dag_execute")
    return [o[:n_out[k]] for k, o in enumerate(outs)]


RAGGED = (0, 1, 8192, 100003, 5, 3 * 65536 + 7, 0, 333333, 2)


@pytest.mark.parametrize("name", ["stereo", "rds", "fanout"])
def test_execute_device_equals_execute(name):
    make, gen = CASES[name][:2]
    x = gen()[:sum(RAGGED)]
    lib = _lib.require_device()
    top_h, dag_h = planned_dag(make, x)
    top_d, dag_d = planned_dag(make, x)
    maxn = max(RAGGED)
    sizes = [p.data_type.dtype.itemsize for p in dag_d.ext_out]
    dx = lib.lrb200_malloc(maxn * 8)
    dys = [lib.lrb200_malloc(max(1, lib.lrb200_dag_max_output(dag_d.dag, k, maxn)) * s) for k, s in enumerate(sizes)]
    try:
        pos = 0
        for n in RAGGED:
            xs = np.ascontiguousarray(x[pos:pos + n])
            pos += n
            want = host_execute(lib, dag_h, xs)
            if n:
                _lib.check(lib.lrb200_memcpy_h2d(dx, xs.ctypes.data, n * 8), "h2d")
            n_out = (ctypes.c_size_t * len(dys))()
            launches = lib.lrb200_launch_count()
            _lib.check(lib.lrb200_dag_execute_device(dag_d.dag, dx, n, (ctypes.c_void_p * len(dys))(*dys), n_out), "execute_device")
            assert n == 0 or lib.lrb200_launch_count() > launches
            for k, w in enumerate(want):
                assert n_out[k] == len(w), "n=%d port %d: %d outputs, host mode %d" % (n, k, n_out[k], len(w))
                got = np.zeros(len(w), w.dtype)
                if len(w):
                    _lib.check(lib.lrb200_memcpy_d2h(got.ctypes.data, dys[k], len(w) * sizes[k]), "d2h")
                _lib.check(lib.lrb200_sync(), "sync")
                assert np.array_equal(got.view(np.uint8), w.view(np.uint8)), "n=%d port %d differs from host mode" % (n, k)
    finally:
        lib.lrb200_free(dx)
        for d in dys:
            lib.lrb200_free(d)
        release(top_h)
        release(top_d)


BOUNDS_CALLS = (0, 1, 2, 4095, 8193, 100003, 262147)


@pytest.mark.parametrize("name", ["stereo", "rds"])
def test_execute_device_bounds(name):
    """Input and outputs in guard-banded allocations, everything around the input poisoned with a NaN pattern, every output
    allocation filled with a sentinel: nothing outside [dx, dx + n) may reach an output, nothing outside [dy[k], dy[k] +
    n_out[k]) may be written.  The input and outputs move between 16-byte aligned and merely 8- / 4-byte aligned places."""
    make, gen, _, cmp = CASES[name]
    x = gen()[:sum(BOUNDS_CALLS) * 4]
    lib = _lib.require_device()
    top_r, dag_r = planned_dag(make, x)                   # host-mode reference, same call lengths
    outs_ref = [[] for _ in dag_r.ext_out]
    pos = 0
    for aligned in (True, False):
        for n in BOUNDS_CALLS:
            for k, o in enumerate(host_execute(lib, dag_r, np.ascontiguousarray(x[pos:pos + n]))):
                outs_ref[k].append(o)
            pos += n
    release(top_r)
    top, dag = planned_dag(make, x)
    sizes = [p.data_type.dtype.itemsize for p in dag.ext_out]
    maxn = max(BOUNDS_CALLS)
    maxo = [lib.lrb200_dag_max_output(dag.dag, k, maxn) for k in range(len(sizes))]
    ib = Guarded(lib, maxn * 8 + 32)
    obs = [Guarded(lib, m * s + 32) for m, s in zip(maxo, sizes)]
    poison = np.resize(np.array([POISON_A], "<u4").view(np.uint8), ib.size)
    sentinel = np.array([SENTINELS[0]], "<u4").view(np.uint8)
    outs = [[] for _ in sizes]
    try:
        pos, call = 0, 0
        for aligned in (True, False):
            for n in BOUNDS_CALLS:
                xoff = 16 * (call % 2) if aligned else (8 if call % 2 == 0 else 16 - 8)
                img = poison.copy()
                img[GUARD + xoff:GUARD + xoff + n * 8] = np.ascontiguousarray(x[pos:pos + n]).view(np.uint8)
                ib.load(img)
                ys, yoffs, oimgs = [], [], []
                for k, (b, s) in enumerate(zip(obs, sizes)):
                    off = 16 * (call % 2) if aligned else (s if call % 2 == 0 else 16 - s)
                    oimgs.append(np.resize(sentinel, b.size))
                    b.load(oimgs[-1])
                    ys.append(b.ptr + GUARD + off)
                    yoffs.append(off)
                n_out = (ctypes.c_size_t * len(ys))()
                _lib.check(lib.lrb200_dag_execute_device(dag.dag, ib.ptr + GUARD + xoff, n, (ctypes.c_void_p * len(ys))(*ys), n_out), "execute_device")
                for k, (b, s) in enumerate(zip(obs, sizes)):
                    host = b.read()
                    lo, hi = GUARD + yoffs[k], GUARD + yoffs[k] + n_out[k] * s
                    where = "call %d (n=%d, aligned %s, output %d)" % (call, n, aligned, k)
                    assert np.array_equal(host[:lo], oimgs[k][:lo]), "%s: written before y" % where
                    assert np.array_equal(host[hi:], oimgs[k][hi:]), "%s: written past y + n_out" % where
                    outs[k].append(host[lo:hi].view(dag.ext_out[k].data_type.dtype))
                pos += n
                call += 1
    finally:
        ib.free()
        for b in obs:
            b.free()
        release(top)
    for k in range(len(sizes)):
        got, ref = np.concatenate(outs[k]), np.concatenate(outs_ref[k])
        assert not np.isnan(got.view(np.float32)).any(), "output %d: NaN (a stray read of the poison)" % k
        assert got.shape == ref.shape
        cmp(got, ref, "output %d" % k)


# ---- raw file source absorption ---------------------------------------------------------------------------------------
def counting(src):
    calls = []
    orig = src.read_raw

    def read_raw(samples=None):
        calls.append(samples)
        return orig(samples)
    src.read_raw = read_raw
    return calls


def test_u8_iq_file_absorbed_into_the_stereo_dag():
    x = stereo_input(N // 2, 36)
    raw = np.clip(np.round(np.stack([x.real, x.imag], 1).reshape(-1) * 127.5 + 127.5), 0, 255).astype(np.uint8)
    conv = O.iq_file_convert(raw, "u8")
    src = radio.IQFileSource(raw.tobytes(), "u8", RATE)
    calls = counting(src)
    top, sinks = stereo_top(None, src=src)
    launches0 = _lib.require_device().lrb200_launch_count()
    top.run(superchunk=1 << 20)
    desc = top.describe_gpu_graph()
    assert desc.startswith("dag{iqconv(u8) ; ") and desc.count("dag{") == 1 and len(top._chains) == 1, desc
    # the DAG pulls the file's bytes itself, in reads of 2^19 samples, and no conversion handle of the source's own runs
    read = GPUDagBlock.RAW_READ
    assert calls == [read] * (-(-len(conv) // read) + 1) and src._handle is None
    assert _lib.load().lrb200_launch_count() > launches0
    top2, sinks2 = stereo_top(conv, chunk=read)
    top2.run(superchunk=1 << 20)
    assert "iqconv" not in top2.describe_gpu_graph()
    for k in range(2):
        a, b = sinks[k].result(), sinks2[k].result()
        assert len(a) == len(b) == -(-len(conv) // 5)        # outputs at input index 0 mod 5
        cmp_stereo(a, b, "port %d" % k)


def test_real_file_absorbed_into_a_fanout_dag_and_not_when_shared():
    rng = np.random.default_rng(37)
    y = rng.uniform(-1, 1, 1 << 21).astype(np.float32)
    src = radio.RealFileSource(y.astype("<f4").tobytes(), "f32le", RATE)
    calls = counting(src)
    top, sinks = fanout_top(None, src=src, real=True)
    top.run(superchunk=1 << 20)
    desc = top.describe_gpu_graph()
    assert desc.startswith("dag{realconv(f32le) ; "), desc
    assert len(calls) == len(y) // GPUDagBlock.RAW_READ + 1 and src._handle is None
    top2, sinks2 = fanout_top(y, chunk=GPUDagBlock.RAW_READ, real=True)
    top2.run(superchunk=1 << 20)
    assert len(sinks[0].result()) == len(y)
    cmp_rel(1e-5)(sinks[0].result(), sinks2[0].result(), "absorbed source")
    # a second reader of the source's output: the source stays a block of its own
    src3 = radio.RealFileSource(y.astype("<f4").tobytes(), "f32le", RATE)
    top3, sinks3 = fanout_top(None, src=src3, real=True)
    extra = radio.ArraySink()
    top3.connect(src3, extra)
    top3.run(superchunk=1 << 20)
    assert "realconv" not in top3.describe_gpu_graph()
    assert np.array_equal(extra.result(), y)
    cmp_rel(1e-5)(sinks3[0].result(), sinks2[0].result(), "source with a second reader")


# ---- API errors -------------------------------------------------------------------------------------------------------
def stream_through(lib, dag, x, S, vec=VECTOR):
    """x in `vec`-sample host vectors through a DAG in super-chunk mode, then the flush: the whole output stream."""
    outs = [[] for _ in dag.ext_out]
    for i in range(0, len(x), vec):
        for k, o in enumerate(host_execute(lib, dag, np.ascontiguousarray(x[i:i + vec]))):
            outs[k].append(o)
    bufs = [np.zeros(lib.lrb200_dag_max_output(dag.dag, k, 0), p.data_type.dtype) for k, p in enumerate(dag.ext_out)]
    n_out = (ctypes.c_size_t * len(bufs))()
    _lib.check(lib.lrb200_dag_flush(dag.dag, (ctypes.c_void_p * len(bufs))(*[b.ctypes.data for b in bufs]), n_out), "flush")
    return [np.concatenate(o + [b[:n_out[k]]]) for k, (o, b) in enumerate(zip(outs, bufs))]


def test_api_errors_leave_the_dag_usable():
    lib = _lib.require_device()
    x = rnd_c(np.random.default_rng(38), 1 << 20)
    top, dag = planned_dag(fanout_top, x)
    fresh_top, fresh = planned_dag(fanout_top, x)
    d = dag.dag
    S = 1 << 16

    def fails(rc, words):
        assert rc != 0
        assert words in _lib.last_error(), _lib.last_error()

    bufs = [np.zeros(lib.lrb200_dag_max_output(d, 0, 1 << 20), np.complex64)]
    ptrs = (ctypes.c_void_p * 1)(bufs[0].ctypes.data)
    n_out = (ctypes.c_size_t * 1)()
    try:
        _lib.check(lib.lrb200_dag_set_superchunk(d, S), "set_superchunk")
        # flush before any execute
        fails(lib.lrb200_dag_flush(d, ptrs, n_out), "nothing to flush")
        # changing the size with a slot pending
        host_execute(lib, dag, np.ascontiguousarray(x[:S + 100]))
        fails(lib.lrb200_dag_set_superchunk(d, 2 * S), "flush before changing the super-chunk size")
        # DEVICE-mode execute is refused in super-chunk mode
        dx = lib.lrb200_malloc(1 << 16)
        dy = (ctypes.c_void_p * 1)(lib.lrb200_malloc(1 << 16))
        fails(lib.lrb200_dag_execute_device(d, dx, 16, dy, n_out), "super-chunk")
        # reset in the middle of a super-chunk: the DAG then computes what a fresh one with the same slot size does
        _lib.check(lib.lrb200_dag_reset(d), "reset")
        _lib.check(lib.lrb200_dag_set_superchunk(fresh.dag, S), "set_superchunk")
        a, b = stream_through(lib, dag, x, S), stream_through(lib, fresh, x, S)
        assert len(a[0]) == len(x) and np.array_equal(a[0], b[0])
        # after the flush, DEVICE mode works once super-chunk mode is off
        _lib.check(lib.lrb200_dag_set_superchunk(d, 0), "set_superchunk(0)")
        _lib.check(lib.lrb200_dag_execute_device(d, dx, 16, dy, n_out), "execute_device")
        _lib.check(lib.lrb200_sync(), "sync")
        assert n_out[0] == 16
        lib.lrb200_free(dx)
        lib.lrb200_free(dy[0])
    finally:
        release(top)
        release(fresh_top)
