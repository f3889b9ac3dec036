"""The ERT receiver's signal path on the GPU (composites/ertreceiver.lua:38-43):

    ComplexMagnitude -> LowpassFilter(128, 4 * 32768) -> Downsampler(6) -> ManchesterMatchedFilter(32768)

  * ManchesterMatchedFilterBlock on the reference's vectors, as a host-mode block and as a one-block graph;
  * 2^24 samples of on-off keyed Manchester bursts through the front end as a linear graph -- in one call, in ragged calls,
    in 8192-sample calls, in super-chunk mode and from an absorbed u8 IQFileSource -- against the float64 oracle chain,
    every output held to its own bound;
  * the magnitude folded into the decimating low-pass (graph.cu fuse_magnitude_fir) against the same graph with a
    MultiplyConstantBlock(1.0) between the two, which keeps the rule from matching: both meet the bound, and only the
    first one's description names the fused stage; the rule leaves undecimated, direct-form and polyphase FIRs alone;
  * the receiver's fan-out, the matched filter feeding one branch per protocol, as one device DAG: equal to the linear
    graph bit for bit for calls of equal length, and in DEVICE mode in guard-banded buffers;
  * the fused-magnitude overlap-save mode in poisoned guard bands at unaligned offsets and tile-boundary lengths.

Bound of a stage output o of an FIR h (M taps) over an input v (u = 2^-24), for either kernel FirBlock::path may run:

    C u ||v_W(o)||_2 ||H||_inf + 4 u |ref_o| + gamma_M sum_k |h_k| |v_(o-k)|    (+ MAG_REL sum_k |h_k| |x_(o-k)| after |x|)

The first two terms are the overlap-save bound of tests/fft_fir_ref.py over W(o) = [o - per - (M - 1), o + per), which
holds every block that can contain o, whatever the call cuts; the third is the direct form's (Higham, Thm 3.5 style dot
product bound); the last is the float32 magnitude's own rounding (tests/ert_ref.py MAG_REL).  The matched filter's output
adds its own bound over the low-pass output to sum_k |h_k| times the low-pass outputs' bounds."""
import ctypes

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from luaradio_b200.composite import GPUChainBlock, GPUDagBlock
from luaradio_b200.types import ComplexFloat32, Float32, Vector
from oracle import lr_oracle as O
from tests import ert_ref as E
from tests import fft_fir_ref as F
from tests.golden_util import JIG_RATE, epsilon_ok, load_spec
from tests.test_gpu_bounds import GUARD, POISON_A, SENTINELS, Guarded
from tests.test_gpu_dag_boundary import host_execute, planned_dag, release

pytestmark = pytest.mark.gpu

BAUD = 32768.0
RATE = 72 * BAUD                     # 2.359296 MS/s: 12 samples per symbol after the decimation by 6
DECIM = 6
N = 1 << 24
VECTOR = 8192
DEV = _lib.LRB200_DEVICE


# ---- signal and reference -----------------------------------------------------------------------------------------------
def ook_bursts(n, seed, scale=0.5):
    """On-off keyed Manchester bursts at 32768 baud on a 150 kHz carrier, 50 dB above the noise, with silent gaps: bursts
    of 40-400 symbols, gaps of 5-50 ms."""
    rng = np.random.default_rng(seed)
    chip = np.zeros(n)
    spc = RATE / BAUD
    pos = int(rng.integers(0, 20000))
    while pos < n:
        nsym = int(rng.integers(40, 400))
        bits = rng.integers(0, 2, nsym)
        chips = np.stack([bits, 1 - bits], 1).reshape(-1).astype(np.float64)      # 1 -> on/off, 0 -> off/on
        idx = pos + np.arange(int(nsym * spc))
        idx = idx[idx < n]
        chip[idx] = chips[((idx - pos) * 2 / spc).astype(np.int64)]
        pos += int(nsym * spc) + int(rng.integers(int(0.005 * RATE), int(0.05 * RATE)))
    t = np.arange(n)
    noise = 10 ** (-50 / 20) / np.sqrt(2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    x = scale * (chip * np.exp(2j * np.pi * 150e3 / RATE * t + 0.3j) + noise)
    return x.astype(np.complex64)


def lowpass_taps():
    return O.lowpass_filter(128, 4 * BAUD, RATE, False).taps


def mf_taps():
    return E.manchester_taps(BAUD, RATE / DECIM)


def _window_norm(v, M, per):
    """||v_W(o)||_2 over W(o) = [o - per - (M - 1), o + per) for every o."""
    c = np.concatenate([[0.0], np.cumsum(np.asarray(v, np.float64) ** 2)])
    o = np.arange(len(v))
    lo, hi = np.clip(o - per - (M - 1), 0, len(v)), np.clip(o + per, 0, len(v))
    return np.sqrt(np.maximum(c[hi] - c[lo], 0.0))


def stage_bound(h, v, ref, mag=False):
    """The module docstring's bound of every full-rate output of FIR h over the non-negative input magnitudes v."""
    M = len(h)
    per = 2 * (1024 - (M - 1))
    hn = F.spectrum_norms("rrrf", h, 1)[0]
    ah = np.abs(np.asarray(h, np.float64))
    S = F.fir_ref(ah, v, wide=True)
    b = F.c_factor(1) * F.U * _window_norm(v, M, per) * hn + 4 * F.U * np.abs(ref) + F.gamma(M) * S
    if mag:
        b += E.MAG_REL * S
    return b


def front_end_reference(x):
    """float64 oracle chain and the bound of every matched-filter output."""
    ax = np.abs(x.astype(np.complex128))
    hl, hm = lowpass_taps(), mf_taps()
    y1_full = F.fir_ref(hl, ax, wide=True)
    b1_full = stage_bound(hl, ax, y1_full, mag=True)
    y1, b1 = y1_full[::DECIM], b1_full[::DECIM]
    y2 = F.fir_ref(hm, y1, wide=True)
    b2 = stage_bound(hm, np.abs(y1) + b1, y2) + F.fir_ref(np.abs(hm.astype(np.float64)), b1, wide=True)
    return y2, b2


def check(got, ref, bound, what):
    got = np.asarray(got)
    assert got.shape == ref.shape, "%s: %d outputs, expected %d" % (what, len(got), len(ref))
    assert not np.isnan(got).any(), "%s: NaN" % what
    d = np.abs(got.astype(np.float64) - ref)
    ratio = d / bound
    i = int(np.argmax(ratio))
    assert ratio[i] <= 1.0, "%s: output %d off by %.3g, bound %.3g (%.2fx)" % (what, i, d[i], bound[i], ratio[i])
    return float(ratio[i])


@pytest.fixture(scope="module")
def stream():
    x = ook_bursts(N, 11)
    ref, bound = front_end_reference(x)
    return x, ref, bound


# ---- graphs through the C ABI -------------------------------------------------------------------------------------------
def front_end_blocks(stand_in=False):
    blocks = [radio.ComplexMagnitudeBlock()]
    if stand_in:
        blocks.append(radio.MultiplyConstantBlock(1.0))
    blocks += [radio.LowpassFilterBlock(128, 4 * BAUD), radio.DownsamplerBlock(DECIM), radio.ManchesterMatchedFilterBlock(BAUD)]
    rate, t = RATE, ComplexFloat32
    for b in blocks:
        b.get_rate = (lambda r: (lambda: r))(rate)
        b.differentiate([t])
        b.initialize()                   # (the filters design their taps from get_rate() here)
        t = b.get_output_type()
        if isinstance(b, radio.DownsamplerBlock):
            rate /= DECIM
    return blocks


def make_graph(lib, blocks):
    g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
    for b in blocks:
        _lib.check(lib.lrb200_graph_append(g, b.make_device_handle()), "append %s" % b.name)
    _lib.check(lib.lrb200_graph_commit(g, 1), "commit")
    return g, lib.lrb200_graph_describe(g).decode()


def run_host(lib, g, x, calls, superchunk=0):
    if superchunk:
        _lib.check(lib.lrb200_graph_set_superchunk(g, superchunk), "superchunk")
    outs, pos, no = [], 0, ctypes.c_size_t()
    for n in list(calls) + ([None] if superchunk else []):
        if n is None:
            y = np.zeros(max(1, lib.lrb200_graph_max_output(g, 0)), np.float32)
            _lib.check(lib.lrb200_graph_flush(g, y.ctypes.data, ctypes.byref(no)), "flush")
        else:
            xs = np.ascontiguousarray(x[pos:pos + n])
            pos += n
            y = np.zeros(max(1, lib.lrb200_graph_max_output(g, n)), np.float32)
            _lib.check(lib.lrb200_graph_execute(g, xs.ctypes.data if n else None, n, y.ctypes.data, ctypes.byref(no)), "execute")
        outs.append(y[:no.value].copy())
    assert pos == len(x)
    return np.concatenate(outs)


def ragged(n, seed):
    rng = np.random.default_rng(seed)
    calls, left = [0, 1, 2, 127, 1793, 1794, 1795, 8 * 897 - 1, 8 * 897, 8 * 897 + 1, 100003, 0, 5], n
    left -= sum(calls)
    while left > 0:
        c = min(left, int(rng.integers(1, 3 << 20)))
        calls.append(c)
        left -= c
    return calls


MODES = {
    "one_call": lambda n: [n],
    "ragged": lambda n: ragged(n, 3),
    "vectors_8192": lambda n: [VECTOR] * (n // VECTOR) + ([n % VECTOR] if n % VECTOR else []),
}


@pytest.mark.parametrize("mode", list(MODES) + ["superchunk"])
@pytest.mark.parametrize("fused", [True, False])
def test_front_end_stream(stream, mode, fused):
    x, ref, bound = stream
    lib = _lib.require_device()
    g, desc = make_graph(lib, front_end_blocks(stand_in=not fused))
    try:
        if fused:
            assert desc.startswith("mag+fir_rrrf[fused x3] | fir_rrrf"), desc
        else:
            assert "mag+" not in desc and desc.startswith("cmag | mulconst"), desc
        if mode == "superchunk":
            got = run_host(lib, g, x, [VECTOR] * (N // VECTOR), superchunk=1 << 20)
        else:
            got = run_host(lib, g, x, MODES[mode](N))
        ex = check(got, ref, bound, "%s %s" % (desc, mode))
        print("\n%s %s: largest |got - ref| / bound %.3g" % (mode, "fused" if fused else "unfused", ex))
    finally:
        lib.lrb200_graph_destroy(g)


def test_composite_run_and_the_absorbed_u8_file_source(stream):
    """The front end built with CompositeBlock and run by its scheduler: from an ArraySource in the reference's 8192-sample
    vectors, and from a u8 IQFileSource, RTL-SDR's format, whose bytes the chain converts as its first stage."""
    x, _, _ = stream
    x = x[:N // 2]
    raw = np.clip(np.round(np.stack([x.real, x.imag], 1).reshape(-1) * 127.5 + 127.5), 0, 255).astype(np.uint8)
    conv = O.iq_file_convert(raw, "u8")
    ref, bound = front_end_reference(conv)

    def top_of(src):
        top, snk = radio.CompositeBlock(), radio.ArraySink()
        top.connect(src, radio.ComplexMagnitudeBlock(), radio.LowpassFilterBlock(128, 4 * BAUD), radio.DownsamplerBlock(DECIM),
                    radio.ManchesterMatchedFilterBlock(BAUD), snk)
        return top, snk

    top, snk = top_of(radio.IQFileSource(raw.tobytes(), "u8", RATE))
    top.run()
    desc = top.describe_gpu_graph()
    assert desc.startswith("iqconv(u8) | mag+fir_rrrf[fused x3] | fir_rrrf") and len(top._chains) == 1, desc
    assert isinstance(top._chains[0], GPUChainBlock)
    check(snk.result(), ref, bound, "u8 file")
    top, snk = top_of(radio.ArraySource(conv, RATE, VECTOR))
    top.run()
    assert top.describe_gpu_graph().startswith("mag+fir_rrrf[fused x3] | fir_rrrf"), top.describe_gpu_graph()
    check(snk.result(), ref, bound, "ArraySource")


def test_rule_leaves_other_shapes_alone():
    """No fusion for an undecimated FIR, a forced direct form, or a shape the real polyphase kernel covers (131 taps at
    D = 5: the decimator keeps its own kernel); an FFT forced on a short filter fuses."""
    lib = _lib.require_device()
    rng = np.random.default_rng(4)

    def desc(M, D, algo=None):
        h = rng.uniform(-1, 1, M).astype(np.float32)
        f = _lib.check_handle(lib.lrb200_fir_create_rrrf(h.ctypes.data, M, 1, DEV), "fir")
        if algo is not None:
            _lib.check(lib.lrb200_fir_set_algorithm(f, algo), "algo")
        hs = [lib.lrb200_cmag_create(DEV), f] + ([lib.lrb200_downsample_create(D, 4, DEV)] if D > 1 else [])
        g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
        for b in hs:
            _lib.check(lib.lrb200_graph_append(g, _lib.check_handle(b, "block")), "append")
        _lib.check(lib.lrb200_graph_commit(g, 1), "commit")
        s = lib.lrb200_graph_describe(g).decode()
        lib.lrb200_graph_destroy(g)
        return s

    assert desc(128, 1) == "cmag | fir_rrrf"
    assert desc(128, 6, _lib.FIR_DIRECT) == "cmag | fir_rrrf[fused x2]"
    assert desc(131, 5) == "cmag | fir_rrrf[fused x2]"
    assert desc(128, 6) == "mag+fir_rrrf[fused x3]"
    assert desc(8, 3, _lib.FIR_FFT) == "mag+fir_rrrf[fused x3]"
    assert desc(600, 6, _lib.FIR_FFT) == "cmag | fir_rrrf[fused x2]"


# ---- the receiver's fan-out as one device DAG ---------------------------------------------------------------------------
def ert_dag_top(x, chunk=VECTOR):
    """The matched filter feeds one branch per protocol (ertreceiver.lua:46-84, idm / scm / scm+).  Each branch's
    PreambleSampler, Slicer and framer stay on the host; a MultiplyConstantBlock(1.0), exact in float32, stands in for the
    branch's first block here so that the fan-out is inside the device set."""
    src = radio.ArraySource(x, RATE, chunk)
    mf = radio.ManchesterMatchedFilterBlock(BAUD)
    top = radio.CompositeBlock()
    top.connect(src, radio.ComplexMagnitudeBlock(), radio.LowpassFilterBlock(128, 4 * BAUD), radio.DownsamplerBlock(DECIM), mf)
    sinks = []
    for _ in ("idm", "scm", "scm+"):
        sinks.append(radio.ArraySink())
        top.connect(mf, radio.MultiplyConstantBlock(1.0), sinks[-1])
    return top, sinks


def test_fanout_dag_equals_the_linear_graph(stream):
    x = stream[0][:N // 4]
    lib = _lib.require_device()
    top, sinks = ert_dag_top(x)
    top.run()
    desc = top.describe_gpu_graph()
    assert desc.startswith("dag{mag+fir_rrrf[fused x3] | fir_rrrf ; ") and desc.count("dag{") == 1, desc
    assert len(top._chains) == 1 and isinstance(top._chains[0], GPUDagBlock)
    g, _ = make_graph(lib, front_end_blocks())
    try:
        want = run_host(lib, g, x, [VECTOR] * (len(x) // VECTOR))
    finally:
        lib.lrb200_graph_destroy(g)
    for k, s in enumerate(sinks):
        got = s.result()
        assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), "branch %d" % k


def test_fanout_dag_device_mode_in_guard_bands(stream):
    """lrb200_dag_execute_device in guard-banded buffers, input and outputs at 16-byte aligned and merely 8- / 4-byte aligned
    places, poison around the input and sentinels around the outputs: nothing outside the input may reach an output and
    nothing outside [dy[k], dy[k] + n_out[k]) may be written; the outputs equal host-mode calls of the same lengths."""
    calls = (0, 1, 2, 1793, 1795, 8191, 8 * 897 + 1, 100003, 262147)
    x = stream[0][:2 * sum(calls)]
    lib = _lib.require_device()
    top_r, dag_r = planned_dag(lambda y: ert_dag_top(y), x)
    want, pos = [[] for _ in dag_r.ext_out], 0
    for _ in range(2):
        for n in calls:
            for k, o in enumerate(host_execute(lib, dag_r, np.ascontiguousarray(x[pos:pos + n]))):
                want[k].append(o)
            pos += n
    release(top_r)
    top, dag = planned_dag(lambda y: ert_dag_top(y), x)
    assert "mag+fir_rrrf" in dag.desc, dag.desc
    maxn = max(calls)
    nk = len(dag.ext_out)
    maxo = [lib.lrb200_dag_max_output(dag.dag, k, maxn) for k in range(nk)]
    ib, obs = Guarded(lib, maxn * 8 + 32), [Guarded(lib, m * 4 + 32) for m in maxo]
    poison = np.resize(np.array([POISON_A], "<u4").view(np.uint8), ib.size)
    sentinel = np.array([SENTINELS[0]], "<u4").view(np.uint8)
    got, pos, call = [[] for _ in range(nk)], 0, 0
    try:
        for aligned in (True, False):
            for n in calls:
                xoff = 16 * (call % 2) if aligned else 8
                img = poison.copy()
                img[GUARD + xoff:GUARD + xoff + n * 8] = np.ascontiguousarray(x[pos:pos + n]).view(np.uint8)
                ib.load(img)
                ys, offs, imgs = [], [], []
                for k, b in enumerate(obs):
                    off = 16 * (call % 2) if aligned else (4 if (call + k) % 2 == 0 else 12)
                    imgs.append(np.resize(sentinel, b.size))
                    b.load(imgs[-1])
                    ys.append(b.ptr + GUARD + off)
                    offs.append(off)
                n_out = (ctypes.c_size_t * nk)()
                _lib.check(lib.lrb200_dag_execute_device(dag.dag, ib.ptr + GUARD + xoff, n, (ctypes.c_void_p * nk)(*ys), n_out),
                           "execute_device")
                for k, b in enumerate(obs):
                    host = b.read()
                    lo, hi = GUARD + offs[k], GUARD + offs[k] + n_out[k] * 4
                    where = "call %d (n=%d, aligned %s, output %d)" % (call, n, aligned, k)
                    assert np.array_equal(host[:lo], imgs[k][:lo]), "%s: written before y" % where
                    assert np.array_equal(host[hi:], imgs[k][hi:]), "%s: written past y + n_out" % where
                    got[k].append(host[lo:hi].view(np.float32))
                pos += n
                call += 1
    finally:
        ib.free()
        for b in obs:
            b.free()
        release(top)
    for k in range(nk):
        a, b = np.concatenate(got[k]), np.concatenate(want[k])
        assert not np.isnan(a).any(), "output %d: NaN (a stray read of the poison)" % k
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "output %d differs from host mode" % k


# ---- the kernel mode in poisoned guard bands ------------------------------------------------------------------------------
SHAPES = ((128, 6), (1, 5), (33, 33), (513, 2), (257, 7))


@pytest.mark.parametrize("M,D", SHAPES)
def test_magnitude_mode_bounds(M, D):
    """The fused stage alone (FFT forced, so that short filters fuse too), fed from poisoned guard bands at aligned and
    unaligned offsets with call lengths around its block (2 L per transform) and the AUTO switch; every output against the
    float64 bound of tests/ert_ref.py MagCase for the kernel's own geometry, and bit for bit the same as aligned buffers."""
    lib = _lib.require_device()
    h = F.G.asym_taps(M, 900 + M)
    model = E.MagFirModel(M, D)
    per, L = model.per, model.L
    calls = [1, 2, M, per - 1, per, per + 1, 3, 2 * per + 1, 8 * L - 1, 8 * L + 1, 5 * per - 3, 4099, 777]
    x = F.signal("bursty", sum(calls), 950 + M, True, F.burst_length(model))
    case = E.MagCase("", h, D, streams=[(0, calls)])
    ref, bound, _, _ = case.expect(x, 0, calls)

    def graph():
        f = _lib.check_handle(lib.lrb200_fir_create_rrrf(np.ascontiguousarray(h).ctypes.data, M, 1, DEV), "fir")
        _lib.check(lib.lrb200_fir_set_algorithm(f, _lib.FIR_FFT), "algo")
        g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
        for b in (lib.lrb200_cmag_create(DEV), f, lib.lrb200_downsample_create(D, 4, DEV)):
            _lib.check(lib.lrb200_graph_append(g, _lib.check_handle(b, "block")), "append")
        _lib.check(lib.lrb200_graph_commit(g, 1), "commit")
        assert lib.lrb200_graph_describe(g).decode() == "mag+fir_rrrf[fused x3]"
        return g

    maxn = max(calls)
    maxo = lib.lrb200_graph_max_output(graph_probe := graph(), maxn)
    lib.lrb200_graph_destroy(graph_probe)
    ib, ob = Guarded(lib, maxn * 8 + 32), Guarded(lib, maxo * 4 + 32)
    poison = np.resize(np.array([POISON_A], "<u4").view(np.uint8), ib.size)
    sentinel = np.resize(np.array([SENTINELS[1]], "<u4").view(np.uint8), ob.size)
    runs = {}
    try:
        for aligned in (True, False):
            g = graph()
            outs, pos = [], 0
            for c, n in enumerate(calls):
                xoff = 16 * (c % 2) if aligned else (8 if c % 2 == 0 else 24)
                yoff = 16 * (c % 2) if aligned else (4 if c % 2 == 0 else 12)
                img = poison.copy()
                img[GUARD + xoff:GUARD + xoff + n * 8] = np.ascontiguousarray(x[pos:pos + n]).view(np.uint8)
                ib.load(img)
                ob.load(sentinel)
                no = ctypes.c_size_t()
                launches = lib.lrb200_launch_count()
                _lib.check(lib.lrb200_graph_execute_device(g, ib.ptr + GUARD + xoff, n, ob.ptr + GUARD + yoff, ctypes.byref(no)),
                           "execute_device")
                assert lib.lrb200_launch_count() - launches == model.plan(n, pos)[1], "call %d (n=%d)" % (c, n)
                host = ob.read()
                lo, hi = GUARD + yoff, GUARD + yoff + no.value * 4
                assert np.array_equal(host[:lo], sentinel[:lo]) and np.array_equal(host[hi:], sentinel[hi:]), \
                    "call %d (n=%d, aligned %s): written outside y" % (c, n, aligned)
                outs.append(host[lo:hi].view(np.float32))
                pos += n
            lib.lrb200_graph_destroy(g)
            runs[aligned] = np.concatenate(outs)
    finally:
        ib.free()
        ob.free()
    assert not np.isnan(runs[False]).any()
    assert np.array_equal(runs[True].view(np.uint32), runs[False].view(np.uint32))
    check(runs[True], ref, bound, "M=%d D=%d" % (M, D))


# ---- the block on the reference's vectors ---------------------------------------------------------------------------------
def test_golden_vectors_host_block_and_one_block_graph():
    block, vectors, eps = load_spec("ert/manchestermatchedfilter_spec")
    lib = _lib.require_device()
    for v in vectors:
        x, want = v["inputs"][0], v["outputs"][0]
        b = radio.ManchesterMatchedFilterBlock(*v["args"])
        b.get_rate = lambda: JIG_RATE
        b.differentiate([Float32])
        b.initialize()
        got = np.array(b.process(Vector.cast(x)).data, copy=True)
        ok, msg = epsilon_ok(got, want, eps)
        assert ok, "%s: %s" % (v["desc"], msg)
        b.reset()
        split = np.concatenate([np.array(b.process(Vector.cast(x[i:i + 3])).data, copy=True) for i in range(0, len(x), 3)])
        ok, msg = epsilon_ok(split, want, eps)
        assert ok, "%s, in calls of 3: %s" % (v["desc"], msg)
        g, desc = make_graph(lib, [b])
        try:
            assert desc == "fir_rrrf", desc
            ok, msg = epsilon_ok(run_host(lib, g, x, [len(x)]), want, eps)
            assert ok, "%s, one-block graph: %s" % (v["desc"], msg)
        finally:
            lib.lrb200_graph_destroy(g)
        b.cleanup()
