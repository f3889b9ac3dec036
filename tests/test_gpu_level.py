"""AGCBlock and PowerSquelchBlock on the GPU (luaradio_b200/csrc/level.cu) against the reference model tests/level_oracle.py:
the reference's spec vectors through a block and through a graph, long bursty streams in every calling pattern, sharding,
and the two rx_am flow graphs."""
import ctypes

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from luaradio_b200.types import ComplexFloat32, Float32, Vector
from oracle import lr_oracle as O
from tests import level_oracle as L
from tests.blocks_util import create_block, run_sample_by_sample, run_whole
from tests.golden_util import epsilon_ok, load_spec

pytestmark = pytest.mark.gpu

TILE = 2048                   # samples per CTA tile of level.cu: flips are placed on and around its boundaries
RATE = 1e6
N_LONG = 1 << 26


def make(cls, args, cplx, rate=RATE):
    return create_block(cls, args, [np.zeros(1, np.complex64 if cplx else np.float32)], rate)


def oracle(cls, args, rate=RATE):
    return (L.AGC if cls == "AGCBlock" else L.PowerSquelch)(*args, rate=rate)


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


@pytest.mark.parametrize("spec", ["agc_spec", "powersquelch_spec"])
def test_spec_vectors_through_a_block_and_a_graph(spec):
    block, vectors, eps = load_spec("level/" + spec)
    for v in vectors:
        x, want = v["inputs"][0], v["outputs"][0]
        blk = create_block(block, v["args"], v["inputs"])
        for got, how in ((run_whole(blk, x), "whole"),):
            ok, msg = epsilon_ok(got, want, eps)
            assert ok, "%s / %s (%s): %s" % (block, v["desc"], how, msg)
        blk = create_block(block, v["args"], v["inputs"])
        ok, msg = epsilon_ok(run_sample_by_sample(blk, x, want.dtype), want, eps)
        assert ok, "%s / %s (sample by sample): %s" % (block, v["desc"], msg)
        got, desc = graph_run(create_block(block, v["args"], v["inputs"]), x)
        ok, msg = epsilon_ok(got, want, eps)
        assert ok, "%s / %s (graph %s): %s" % (block, v["desc"], desc, msg)
        assert desc.startswith("agc" if block == "AGCBlock" else "powersquelch"), desc


def bursty_stream(n, cplx, seed):
    """Loud spans (|x|^2 = 0.01, -20 dBFS) in a -80 dBFS noise floor.  Span starts and lengths are random; every third loud
    span starts exactly on a tile boundary, and the quiet gaps range from a few hundred samples (the gate closes and
    reopens inside a tile) to several tiles (whole tiles with the gate closed)."""
    rng = np.random.default_rng(seed)
    loud = np.zeros(n, bool)
    i, k = 0, 0
    while i < n:
        gap = int(rng.integers(300, 1500)) if rng.random() < 0.6 else int(rng.integers(3 * TILE, 12 * TILE))
        start = i + gap
        if k % 3 == 0:
            start = (start // TILE + 1) * TILE
        length = int(rng.integers(50, 4 * TILE))
        loud[start:start + length] = True
        i, k = start + length, k + 1
    sign = np.where(rng.random(n) < 0.5, -0.1, 0.1)
    if cplx:
        ph = np.exp(2j * np.pi * rng.random(n))
        x = np.where(loud, 0.1 * ph, 1e-4 * (rng.standard_normal(n) + 1j * rng.standard_normal(n)) / np.sqrt(2))
        return x.astype(np.complex64)
    return np.where(loud, sign, 1e-4 * rng.standard_normal(n)).astype(np.float32)


# AGC: power estimator ~50 samples, gain filter ~1000 samples at 1 MHz; threshold -40 dBFS.  Squelch: tau = 1 ms.
AGC_ARGS = ("custom", -20, -40, {"gain_tau": 1e-3, "power_tau": 5e-5})
SQ_ARGS = (-45,)
SQ_RATE = 1e5                 # alpha = 1/101: the squelch's pole also flips within a tile


def check_close(got, want, what):
    """Within 4 float32 ulps per component (closed samples pass through bit for bit)."""
    g = got.view(np.float32).astype(np.float64)
    w = want.view(np.float32)
    ulp = np.spacing(np.abs(w)).astype(np.float64)
    d = np.abs(g - w.astype(np.float64))
    bad = d > 4 * ulp
    assert not bad.any(), "%s: %d components beyond 4 ulps, first at %d: got %r want %r" % (
        what, int(bad.sum()), int(np.argmax(bad)) // (2 if np.iscomplexobj(want) else 1), g[np.argmax(bad)], w[np.argmax(bad)])


def reference(cls, args, rate, x):
    o = oracle(cls, args, rate)
    P, gate = o.gate(x)
    theta = o.threshold
    # the test is meaningful only when no sample's power sits within double-precision reach of the threshold
    assert np.min(np.abs(P - theta)) >= 1e-9 * theta, "stimulus too close to the threshold"
    y = o.process(x)
    flips = np.flatnonzero(np.diff(gate.astype(np.int8))) + 1
    return y, gate, flips


@pytest.fixture(scope="module", params=[("AGCBlock", False), ("AGCBlock", True), ("PowerSquelchBlock", False), ("PowerSquelchBlock", True)],
                ids=["agc_real", "agc_complex", "squelch_real", "squelch_complex"])
def long_case(request):
    cls, cplx = request.param
    args, rate = (AGC_ARGS, RATE) if cls == "AGCBlock" else (SQ_ARGS, SQ_RATE)
    x = bursty_stream(N_LONG, cplx, 11 if cplx else 12)
    y, gate, flips = reference(cls, args, rate, x)
    # flips inside tiles, exactly on tile boundaries, and whole tiles with the gate closed
    assert len(flips) > 5000 and (flips % TILE == 0).sum() >= 10 and ((flips % TILE) != 0).sum() > 1000
    closed_tiles = ~gate[:N_LONG // TILE * TILE].reshape(-1, TILE).any(axis=1)
    assert closed_tiles.sum() > 100
    return cls, args, rate, cplx, x, y


def stream(blk, x, cuts):
    return np.concatenate([run_whole(blk, x[a:b]) for a, b in cuts])


def test_long_stream_one_call(long_case):
    cls, args, rate, cplx, x, y = long_case
    blk = make(cls, args, cplx, rate)
    check_close(run_whole(blk, x), y, "one call")


def test_long_stream_ragged_calls(long_case):
    cls, args, rate, cplx, x, y = long_case
    rng = np.random.default_rng(4)
    sizes = [1, TILE - 1, TILE, TILE + 1, 1, 1, 3 * TILE + 5, 8192, 7]
    while sum(sizes) < N_LONG:
        sizes.append(int(rng.integers(1, 1 << 22)))
    edges = np.minimum(np.cumsum([0] + sizes), N_LONG)
    cuts = [(int(a), int(b)) for a, b in zip(edges, edges[1:]) if b > a]
    blk = make(cls, args, cplx, rate)
    check_close(stream(blk, x, cuts), y, "ragged calls")


def test_long_stream_8192_sample_calls(long_case):
    cls, args, rate, cplx, x, y = long_case
    n = N_LONG // 8
    blk = make(cls, args, cplx, rate)
    check_close(stream(blk, x[:n], [(a, min(n, a + 8192)) for a in range(0, n, 8192)]), y[:n], "8192-sample calls")


def test_long_stream_superchunk(long_case):
    cls, args, rate, cplx, x, y = long_case
    n = N_LONG // 8
    src, snk = radio.ArraySource(x[:n], rate, 8192), radio.ArraySink()
    top = radio.CompositeBlock()
    blk = getattr(radio, cls)(*args)
    top.connect(src, blk, radio.MultiplyConstantBlock(1.0), snk)     # two stages: a device chain
    top.run(superchunk=1 << 20)
    assert ("agc" if cls == "AGCBlock" else "powersquelch") in top.describe_gpu_graph()
    check_close(snk.result(), y[:n], "super-chunk")


def test_halo_refuses_agc_and_shards_powersquelch():
    lib = _lib.require_device()
    agc = make("AGCBlock", AGC_ARGS, True)
    g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
    _lib.check(lib.lrb200_graph_append(g, agc.make_device_handle()))
    _lib.check(lib.lrb200_graph_commit(g, 1))
    assert lib.lrb200_graph_halo(g) < 0
    assert "unbounded memory" in _lib.last_error() and "agc" in _lib.last_error()
    lib.lrb200_graph_destroy(g)

    total, world = 1 << 22, 4
    x = bursty_stream(total, True, 8)
    want, _, _ = reference("PowerSquelchBlock", SQ_ARGS, SQ_RATE, x)

    def graph():
        gg = _lib.check_handle(lib.lrb200_graph_create(), "graph")
        _lib.check(lib.lrb200_graph_append(gg, make("PowerSquelchBlock", SQ_ARGS, True, SQ_RATE).make_device_handle()))
        _lib.check(lib.lrb200_graph_commit(gg, 1))
        return gg
    g, gh = graph(), graph()
    halo = lib.lrb200_graph_halo(g)
    assert 2000 < halo < 4000, halo
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
    got = np.concatenate(parts)
    whole = run_whole(make("PowerSquelchBlock", SQ_ARGS, True, SQ_RATE), x)
    assert np.array_equal(whole.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(got.view(np.uint32), whole.view(np.uint32))
    lib.lrb200_free(d_in)
    lib.lrb200_free(d_out)
    lib.lrb200_graph_destroy(g)
    lib.lrb200_graph_destroy(gh)


def close(got, ref, rel=1e-5):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, "length %s != %s" % (got.shape, ref.shape)
    scale = max(1.0, float(np.max(np.abs(ref))))
    err = float(np.max(np.abs(got.astype(np.complex128) - ref.astype(np.complex128))))
    assert err <= rel * scale, "max abs err %.3g > %.3g" % (err, rel * scale)


def am_input(n, rate, carrier, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / rate
    env = 0.5 * (1 + 0.5 * np.sin(2 * np.pi * 440 * t) + 0.2 * np.sin(2 * np.pi * 1250 * t))
    x = env * np.exp(2j * np.pi * carrier * t + 0.7j) + 0.002 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return x.astype(np.complex64)


@pytest.mark.parametrize("chunk", [1 << 22, 8192])
def test_rx_am_envelope_graph(chunk):
    """rx_am.lua:51-55 at 1.1025 MS/s: Tuner(-50 kHz, 10 kHz, /25) -> AMEnvelopeDemodulator(5 kHz) -> AGCBlock('slow'), one
    device chain, against the oracle chain."""
    rate, n = 1102500.0, 1 << 22
    x = am_input(n, rate, -50e3 + 3.0, 1)
    src, snk = radio.ArraySource(x, rate, chunk), radio.ArraySink()
    top = radio.CompositeBlock()
    top.connect(src, radio.TunerBlock(-50e3, 10e3, 25), radio.AMEnvelopeDemodulator(5e3), radio.AGCBlock("slow"), snk)
    top.run()
    desc = top.describe_gpu_graph()
    assert "agc_rr" in desc and len(top._chains) == 1, desc
    af = rate / 25
    b, a = O.singlepole_highpass_taps(100, af)
    ref = O.Chain(O.tuner(-50e3, 10e3, 25, rate), O.complex_magnitude, O.IIRFilterFast(b, a, False),
                  O.lowpass_filter(128, 5e3, af, False), L.AGC("slow", rate=af)).process(x)
    close(snk.result(), ref)
    assert np.max(np.abs(ref[-10000:])) > 1e-3


def test_rx_am_synchronous_graph():
    """rx_am.lua:66-71: DecimatorBlock(5) -> AMSynchronousDemodulator(50 kHz, 5 kHz) -> DownsamplerBlock(5) -> AGCBlock('slow'),
    one device DAG.  Its AGC stage is checked against the oracle AGC applied to the same DAG's output without the AGC, and
    that output against the oracle chain.  (The AGC turns the float32 differences of the PLL path into gain differences at
    its first threshold crossing -- one sample more or less at P = threshold adds ga * T / threshold to g -- so the whole
    chain is not held to 1e-5 against the oracle chain.)"""
    rate, n = 1102500.0, 1 << 21
    x = am_input(n, rate, 50e3 + 3.0, 2)

    def run(with_agc):
        src, snk = radio.ArraySource(x, rate, 1 << 20), radio.ArraySink()
        top = radio.CompositeBlock()
        tail = [radio.AGCBlock("slow")] if with_agc else []
        top.connect(src, radio.DecimatorBlock(5), radio.AMSynchronousDemodulator(50e3, 5e3), radio.DownsamplerBlock(5), *tail, snk)
        top.run()
        return snk.result(), top
    got, top = run(True)
    desc = top.describe_gpu_graph()
    assert desc.startswith("dag{") and "agc_rr" in desc and len(top._chains) == 1, desc
    demod, _ = run(False)
    close(got, L.AGC("slow", rate=rate / 25).process(demod))
    ifr = rate / 5
    rf = O.complex_bandpass_filter(129, [50e3 - 5e3, 50e3 + 5e3], ifr).process(O.decimator(5, True).process(x))
    pll_out, _ = O.PLL(1000, 50e3 - 100, 50e3 + 100, None, ifr).process(rf)
    b, a = O.singlepole_highpass_taps(100, ifr)
    ref = O.Chain(O.complex_to_real, O.IIRFilterFast(b, a, False), O.lowpass_filter(128, 5e3, ifr, False), O.Downsampler(5)).process(
        O.binary_op("multiplyconjugate", rf, pll_out))
    close(demod, ref, 5e-5)                          # the AM-synchronous DAG's own tolerance (tests/test_gpu_dag.py)
    assert np.max(np.abs(got[-10000:])) > 1e-3
