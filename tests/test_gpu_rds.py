"""BinaryPhaseCorrectorBlock on the GPU (luaradio_b200/csrc/phasecorr.cu) against the reference model tests/rds_oracle.py:
the reference's spec and executed vectors through a block and a graph, long streams in every calling pattern, reset,
sharding, and the RDS and BPSK31 signal paths as device flow graphs."""
import ctypes
import os

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from oracle import lr_oracle as O
from tests import pll_ref as P
from tests import rds_oracle as R
from tests.blocks_util import create_block, run_sample_by_sample, run_whole
from tests.golden.make_rds_golden import BPC_CASES, chunks
from tests.golden_util import GOLDEN_DIR, epsilon_ok, load_spec

pytestmark = pytest.mark.gpu

TILE = 2048                   # samples per CTA tile of phasecorr.cu
N_LONG = 1 << 26
SHAPES = [(8000, 32), (50, 32), (17, 15), (4, 1)]


def graph_run(blk, x):
    """One-stage lrb200 graph made from the block's device handle, HOST in/out."""
    lib = _lib.require_device()
    g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
    _lib.check(lib.lrb200_graph_append(g, blk.make_device_handle()), "append")
    _lib.check(lib.lrb200_graph_commit(g, 1), "commit")
    x = np.ascontiguousarray(x)
    y = np.zeros(len(x), x.dtype)
    no = ctypes.c_size_t()
    _lib.check(lib.lrb200_graph_execute(g, x.ctypes.data, len(x), y.ctypes.data, ctypes.byref(no)), "execute")
    desc = lib.lrb200_graph_describe(g).decode()
    lib.lrb200_graph_destroy(g)
    assert no.value == len(x)
    return y, desc


def bpc(N, I):
    return create_block("BinaryPhaseCorrectorBlock", [N, I], [np.zeros(1, np.complex64)])


def close(got, ref, rel=1e-5, what=""):
    """The project's stream tolerance, 1e-5 * max(1, |ref|_inf); returns the largest difference in float32 ulps of the
    sample's magnitude."""
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, "%s: length %s != %s" % (what, got.shape, ref.shape)
    scale = max(1.0, float(np.max(np.abs(ref)))) if ref.size else 1.0
    err = float(np.max(np.abs(got.astype(np.complex128) - ref.astype(np.complex128)))) if ref.size else 0.0
    assert err <= rel * scale, "%s: max abs err %.3g > %.3g" % (what, err, rel * scale)
    if not ref.size:
        return 0.0
    d = np.abs(got.astype(np.complex128) - ref.astype(np.complex128))
    return float(np.max(d / np.spacing(np.maximum(np.abs(ref).astype(np.float32), np.float32(1e-30))).astype(np.float64)))


def test_spec_vectors_through_a_block_and_a_graph():
    block, vectors, eps = load_spec("rds/binaryphasecorrector_spec")
    for v in vectors:
        x, want = v["inputs"][0], v["outputs"][0]
        ok, msg = epsilon_ok(run_whole(create_block(block, v["args"], v["inputs"]), x), want, eps)
        assert ok, "%s (whole): %s" % (v["desc"], msg)
        ok, msg = epsilon_ok(run_sample_by_sample(create_block(block, v["args"], v["inputs"]), x, want.dtype), want, eps)
        assert ok, "%s (sample by sample): %s" % (v["desc"], msg)
        got, desc = graph_run(create_block(block, v["args"], v["inputs"]), x)
        ok, msg = epsilon_ok(got, want, eps)
        assert ok, "%s (graph %s): %s" % (v["desc"], desc, msg)
        assert desc.startswith("phasecorr"), desc


@pytest.mark.parametrize("N,I", [c[:2] for c in BPC_CASES])
def test_executed_vectors_through_a_block_and_a_graph(N, I):
    """binaryphasecorrector.lua executed over ragged calls: the same calls through a block, sample by sample, and through a
    one-stage graph, against the executed output."""
    g = np.load(os.path.join(GOLDEN_DIR, "rds", "bpc_reference_executed.npz"))
    name = "n%d_i%d" % (N, I)
    x, want = g[name + "_x"], g[name + "_y"]
    blk = bpc(N, I)
    ulps = close(np.concatenate([run_whole(blk, x[a:b]) for a, b in chunks(len(x))]), want, what="ragged")
    close(run_sample_by_sample(bpc(N, I), x, want.dtype), want, what="sample by sample")
    got, desc = graph_run(bpc(N, I), x)
    close(got, want, what="graph")
    assert desc.startswith("phasecorr"), desc
    print("%s: executed vector, largest difference %.1f ulp" % (name, ulps))


def test_create_rejects_empty_window_and_interval():
    lib = _lib.require_device()
    for args, msg in (((0, 32), b"num_samples must be >= 1"), ((8000, 0), b"sample_interval must be >= 1")):
        assert not lib.lrb200_phasecorrector_create(*args, _lib.LRB200_DEVICE)
        assert msg in lib.lrb200_last_error()


def drifting_bpsk(n, seed):
    """BPSK symbols of 16 samples whose carrier phase wanders (a slow random walk through every quadrant), with noise."""
    rng = np.random.default_rng(seed)
    sym = np.repeat(rng.choice(np.array([-1.0, 1.0], np.float32), n // 16 + 1), 16)[:n]
    phase = 0.3 + np.cumsum(rng.normal(0.0, 2e-4, n)) + 2 * np.pi * 1e-7 * np.arange(n)
    x = sym * np.exp(1j * phase) + 0.1 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return x.astype(np.complex64)


@pytest.fixture(scope="module", params=SHAPES, ids=["n%d_i%d" % s for s in SHAPES])
def long_case(request):
    N, I = request.param
    x = drifting_bpsk(N_LONG, N + I)
    return N, I, x, R.BinaryPhaseCorrector(N, I).process(x)


def stream(blk, x, cuts):
    return np.concatenate([run_whole(blk, x[a:b]) for a, b in cuts])


def test_long_stream_one_call(long_case):
    N, I, x, y = long_case
    print("n%d_i%d one call: %.1f ulp" % (N, I, close(run_whole(bpc(N, I), x), y, what="one call")))


def test_long_stream_ragged_calls(long_case):
    N, I, x, y = long_case
    rng = np.random.default_rng(4)
    sizes = [0, 1, I - 1 if I > 1 else 1, TILE - 1, TILE, TILE + 1, 0, 1, 3 * TILE + 5, 8192, 7, N * I + 3]
    while sum(sizes) < N_LONG:
        sizes.append(int(rng.integers(1, 1 << 22)))
    edges = np.minimum(np.cumsum([0] + sizes), N_LONG)
    cuts = [(int(a), int(b)) for a, b in zip(edges, edges[1:])]
    print("n%d_i%d ragged calls: %.1f ulp" % (N, I, close(stream(bpc(N, I), x, cuts), y, what="ragged calls")))


def test_long_stream_8192_sample_calls(long_case):
    N, I, x, y = long_case
    n = N_LONG
    got = stream(bpc(N, I), x[:n], [(a, min(n, a + 8192)) for a in range(0, n, 8192)])
    print("n%d_i%d 8192-sample calls: %.1f ulp" % (N, I, close(got, y[:n], what="8192-sample calls")))


def test_long_stream_superchunk(long_case):
    N, I, x, y = long_case
    n = N_LONG
    src, snk = radio.ArraySource(x[:n], 1e6, 8192), radio.ArraySink()
    top = radio.CompositeBlock()
    top.connect(src, radio.BinaryPhaseCorrectorBlock(N, I), radio.MultiplyConstantBlock(1.0), snk)    # two stages: a device chain
    top.run(superchunk=1 << 20)
    assert "phasecorr" in top.describe_gpu_graph()
    print("n%d_i%d super-chunk: %.1f ulp" % (N, I, close(snk.result(), y[:n], what="super-chunk")))


@pytest.mark.parametrize("N,I", SHAPES)
def test_reset_matches_a_fresh_block(N, I):
    x = drifting_bpsk(1 << 20, 3)
    blk = bpc(N, I)
    first = run_whole(blk, x)
    run_whole(blk, x[:12345])
    blk.reset()
    assert np.array_equal(run_whole(blk, x).view(np.uint32), first.view(np.uint32))
    assert np.array_equal(run_whole(bpc(N, I), x).view(np.uint32), first.view(np.uint32))


def test_halo_includes_the_window_and_shards_match_the_stream():
    """Lowpass(128, 100) -> RRC(101, 1, 31.25) -> BinaryPhaseCorrector(50, 32) at 8 kHz: the halo covers the corrector's
    N * I samples on top of the filters' memory, and each of four shards equals a cold start of the model N * I samples
    before it.  The single stream differs from that cold start only by the reference average's float32 drift term
    sum((phi - float32(phi)) / N) over the measurements before the cold start, which grows with the stream position."""
    lib = _lib.require_device()
    rate, N, I = 8000.0, 50, 32

    def blocks():
        out = []
        for cls, args in (("LowpassFilterBlock", [128, 100]), ("RootRaisedCosineFilterBlock", [101, 1, 31.25]),
                          ("BinaryPhaseCorrectorBlock", [N, I])):
            out.append(create_block(cls, args, [np.zeros(1, np.complex64)], rate))
        return out

    def graph():
        g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
        for b in blocks():
            _lib.check(lib.lrb200_graph_append(g, b.make_device_handle()))
        _lib.check(lib.lrb200_graph_commit(g, 1))
        return g
    g, gh = graph(), graph()
    halo = lib.lrb200_graph_halo(g)
    assert N * I <= halo <= N * I + 128 + 101 + 8, halo
    total, world = 1 << 22, 4
    # a carrier of constant magnitude whose phase wanders: no sample near zero, where atan2f would turn the float32
    # differences of two FIR implementations into large phase differences
    rng = np.random.default_rng(9)
    x = (np.exp(1j * (0.3 + np.cumsum(rng.normal(0.0, 2e-3, total)))) * (1 + 0.02 * rng.standard_normal(total))).astype(np.complex64)
    whole = x
    for b in blocks():
        whole = run_whole(b, whole)
    per = total // world
    d_in = lib.lrb200_malloc((per + halo) * 8)
    d_out = lib.lrb200_malloc(per * 8)
    no = ctypes.c_size_t()
    parts = []
    for r in range(world):
        start = r * per
        lead = halo if r > 0 else 0
        seg = np.ascontiguousarray(x[start - lead:start + per])
        _lib.check(lib.lrb200_memcpy_h2d(ctypes.c_void_p(d_in + (halo - lead) * 8), seg.ctypes.data, seg.nbytes))
        _lib.check(lib.lrb200_graph_execute_shard(g, gh, ctypes.c_void_p(d_in), halo, per, start, ctypes.c_void_p(d_out),
                                                  ctypes.byref(no), None))
        out = np.zeros(no.value, np.complex64)
        _lib.check(lib.lrb200_memcpy_d2h(out.ctypes.data, ctypes.c_void_p(d_out), out.nbytes))
        _lib.check(lib.lrb200_sync())
        parts.append(out)
    filtered = x
    for b in blocks()[:2]:
        filtered = run_whole(b, filtered)
    model = O.Chain(O.lowpass_filter(128, 100, rate, True), R.rrc_filter(101, 1, 31.25, rate, True)).process(x)
    close(filtered, model, what="filters")
    drift = 0.0
    for r, got in enumerate(parts):
        start = r * per
        ref = R.BinaryPhaseCorrector(N, I).process(filtered[:per]) if r == 0 else None
        if r > 0:
            cold = R.BinaryPhaseCorrector(N, I)
            cold.consumed, cold.measurements = start - N * I, (start - N * I + I - 1) // I
            ref = cold.process(filtered[start - N * I:start + per])[N * I:]
            drift = max(drift, float(np.max(np.abs(ref - whole[start:start + per]))))
        close(got, ref, what="shard %d" % r)
    close(np.concatenate(parts), whole, rel=1e-5 + drift, what="shards against the stream")
    print("shards: the stream's drift term reaches %.3g" % drift)
    lib.lrb200_free(d_in)
    lib.lrb200_free(d_out)
    lib.lrb200_graph_destroy(g)
    lib.lrb200_graph_destroy(gh)


def rds_top(x, rate, chunk, tuner, parallel_pll=False):
    """examples/rtlsdr_rds.lua:13-24,38-43,48 up to ComplexToRealBlock, with sinks on the RRC, the corrector and
    ComplexToReal.  tuner=False starts at the FrequencyDiscriminatorBlock (the source is then at 220.5 kHz)."""
    src = radio.ArraySource(x, rate, chunk)
    hilbert, delay = radio.HilbertTransformBlock(129), radio.DelayBlock(129)
    pll, mixer = radio.PLLBlock(1500.0, 19e3 - 100, 19e3 + 100, 3.0), radio.MultiplyConjugateBlock()
    pll.parallel = parallel_pll
    rrc, corr, c2r = radio.RootRaisedCosineFilterBlock(101, 1, 1187.5), radio.BinaryPhaseCorrectorBlock(8000), radio.ComplexToRealBlock()
    sinks = [radio.ArraySink() for _ in range(3)]
    top = radio.CompositeBlock()
    front = [src, radio.TunerBlock(-250e3, 200e3, 5)] if tuner else [src]
    top.connect(*front, radio.FrequencyDiscriminatorBlock(1.25), hilbert, delay)
    top.connect(hilbert, radio.ComplexBandpassFilterBlock(129, [18e3, 20e3]), pll)
    top.connect(delay, "out", mixer, "in1")
    top.connect(pll, "out", mixer, "in2")
    top.connect(mixer, radio.LowpassFilterBlock(128, 4e3), rrc, corr)
    top.connect(corr, c2r, sinks[2])
    top.connect(corr, sinks[1])
    top.connect(rrc, sinks[0])
    return top, sinks


def assert_one_dag(top):
    desc = top.describe_gpu_graph()
    assert desc.startswith("dag{") and desc.count("dag{") == 1 and "phasecorr" in desc and "pll" in desc, desc
    assert len(top._chains) == 1, desc


def test_rds_path_matches_the_reference_executed_golden():
    g = np.load(os.path.join(GOLDEN_DIR, "rds", "rds_reference_executed.npz"))
    x, rate = g["x"], float(g["rate"])
    top, sinks = rds_top(x, rate, 1500, tuner=False)
    top.run()
    assert_one_dag(top)
    # the PLL's float32 path of two libraries: the DAG tolerance of tests/test_gpu_dag.py
    for snk, key in zip(sinks, ("rrc", "bpc", "real")):
        close(snk.result(), g[key], 5e-5, key)


def rds_input(n, rate, seed):
    """The golden's multiplex at 1.1025 MS/s, 250 kHz above the tuner's centre."""
    from tests.golden.make_rds_golden import rds_mpx
    x = rds_mpx(n, rate, np.random.default_rng(seed))
    return (x * np.exp(2j * np.pi * 250e3 / rate * np.arange(n))).astype(np.complex64)


def test_rds_path_from_the_source_against_the_oracle():
    """TunerBlock onward at 1.1025 MS/s, 2^22 samples: one device DAG, against the oracle chain (the PLL serial), and the
    same graph with the chunk-parallel PLL against the serial one once the loop is locked.  Every DAG call hands the
    PLL 2^20 / 5 samples, more than 2 L = 32768, so the parallel form runs from the first call; its chunk 0 is exact and
    the loop locks within its first chunk.  From 2^16 PLL samples (0.3 s) on, the parallel PLL's output is within out_tol
    of tests/pll_ref.py of the serial one.  The mixer scales that by the delayed multiplex (the discriminator's output
    peaks at 0.4 here), the low-pass and the RRC have an L1 gain of 1.2 together, and the phase corrector only rotates:
    the sinks are held to 10 out_tol max(1, |serial|)."""
    rate, n = 1102500.0, 1 << 22
    x = rds_input(n, rate, 2)
    top, sinks = rds_top(x, rate, 1 << 20, tuner=True)
    top.run()
    assert_one_dag(top)
    d = O.tuner(-250e3, 200e3, 5, rate).process(x)
    rrc, corr, real = R.RDSPath(rate / 5).process(d)
    for snk, ref, what in zip(sinks, (rrc, corr, real), ("rrc", "bpc", "real")):
        close(snk.result(), ref, 5e-5, what)
    assert np.max(np.abs(rrc)) > 1e-3
    serial = [snk.result() for snk in sinks]
    top, sinks = rds_top(x, rate, 1 << 20, tuner=True, parallel_pll=True)
    top.run()
    assert_one_dag(top)
    for snk, ref, what in zip(sinks, serial, ("rrc", "bpc", "real")):
        got = snk.result()
        assert len(got) == len(ref), what
        lock = len(ref) * (1 << 16) // (n // 5)                # 2^16 samples at the PLL's rate
        d = float(np.max(np.abs(got[lock:].astype(np.complex128) - ref[lock:])))
        scale = max(1.0, float(np.max(np.abs(ref))))
        print("%s: parallel vs serial PLL, locked: %.3g" % (what, d))
        assert d <= 10 * P.out_tol(-(-(n // 5) // P.MIN_CHUNK)) * scale, "%s: parallel PLL differs from the serial one by %.3g once locked" % (what, d)


def test_bpsk31_front_end_against_the_oracle():
    """composites/bpsk31receiver.lua:27-37 up to the clock recoverer, at 8 kHz: every signal block on the device."""
    rate, n = 8000.0, 1 << 21
    rng = np.random.default_rng(6)
    t = np.arange(n) / rate
    sym = np.repeat(rng.choice([-1.0, 1.0], int(n / 256) + 1), 256)[:n]           # 31.25 baud
    x = (sym * np.exp(1j * (2 * np.pi * 3.0 * t + 0.5)) + 0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))).astype(np.complex64)
    front = R.BPSK31FrontEnd(rate)
    src, s_corr, s_real = radio.ArraySource(x, rate, 1 << 18), radio.ArraySink(), radio.ArraySink()
    corr = radio.BinaryPhaseCorrectorBlock(50)
    top = radio.CompositeBlock()
    top.connect(src, radio.LowpassFilterBlock(128, 100), radio.RootRaisedCosineFilterBlock(101, 1, 31.25), corr)
    top.connect(corr, radio.ComplexToRealBlock(), s_real)
    top.connect(corr, s_corr)
    top.run()
    desc = top.describe_gpu_graph()
    assert "phasecorr" in desc and len(top._chains) == 1, desc
    # the same two filters as a chain of their own: the corrector's input as the device computed it
    src, s_rrc = radio.ArraySource(x, rate, 1 << 18), radio.ArraySink()
    top = radio.CompositeBlock()
    top.connect(src, radio.LowpassFilterBlock(128, 100), radio.RootRaisedCosineFilterBlock(101, 1, 31.25), s_rrc)
    top.run()
    filt = s_rrc.result()
    close(filt, front.rrc.process(front.lowpass.process(x)), what="filters")
    # The filtered BPSK passes through zero at every symbol change, where atan2f turns float32 differences of two FIR
    # implementations into phase differences of any size; so the corrector is checked on the device's own filter output.
    ref_corr = front.bpc.process(filt)
    close(s_corr.result(), ref_corr, what="corrector")
    close(s_real.result(), O.complex_to_real(ref_corr), what="complex to real")


def test_call_longer_than_one_launch_set():
    """A call of more than 256 Mi samples (on device pointers, as a graph stage may pass it) is split into launch sets that
    carry the consumed count, the window and the average between them: bit for bit two calls of the same lengths (the
    ragged-call tests hold such calls to the model)."""
    import torch
    lib = _lib.require_device()
    n = (1 << 28) + 12345
    x = torch.empty(n, dtype=torch.complex64, device="cuda")
    # the library stream is non-blocking: neither it nor torch's stream waits for the other, so each hand-over is a sync
    _lib.check(lib.lrb200_synth_white_iq(ctypes.c_void_p(x.data_ptr()), 0, n, 7))
    _lib.check(lib.lrb200_sync())
    x = x + 0.8                                         # a carrier with noise: the average moves away from zero
    y1, y2 = torch.empty_like(x), torch.empty_like(x)
    torch.cuda.synchronize()
    no = ctypes.c_size_t()
    for N, I in ((8000, 32), (17, 15)):
        one = _lib.check_handle(lib.lrb200_phasecorrector_create(N, I, _lib.LRB200_DEVICE), "phasecorr")
        two = _lib.check_handle(lib.lrb200_phasecorrector_create(N, I, _lib.LRB200_DEVICE), "phasecorr")
        _lib.check(lib.lrb200_block_execute(one, ctypes.c_void_p(x.data_ptr()), n, ctypes.c_void_p(y1.data_ptr()), ctypes.byref(no)))
        assert no.value == n
        k = 1 << 28
        _lib.check(lib.lrb200_block_execute(two, ctypes.c_void_p(x.data_ptr()), k, ctypes.c_void_p(y2.data_ptr()), ctypes.byref(no)))
        _lib.check(lib.lrb200_block_execute(two, ctypes.c_void_p(x.data_ptr() + 8 * k), n - k, ctypes.c_void_p(y2.data_ptr() + 8 * k),
                                            ctypes.byref(no)))
        torch.cuda.synchronize()
        assert torch.equal(y1.view(torch.int64), y2.view(torch.int64))
        assert not torch.equal(y1[k:].view(torch.int64), x[k:].view(torch.int64))     # the second set was rotated
        lib.lrb200_block_destroy(one)
        lib.lrb200_block_destroy(two)
