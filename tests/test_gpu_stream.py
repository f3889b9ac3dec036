"""GPU parity against the oracle on seeded streams beyond the golden-vector sizes: long inputs,
ragged chunking (streaming state), decimation phases, large sample indices, the fused WBFM chain.

Tolerance (north_star: float32 match within 1e-5 relative): |got - ref| <= 1e-5 * max(1, ||ref||_inf)."""
import ctypes

import os

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from luaradio_b200.types import ComplexFloat32, Float32, Vector
from oracle import lr_oracle as O
from tests import iir_small_ref as S

pytestmark = pytest.mark.gpu

REL = 1e-5


def close(got, ref, rel=REL):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, "length %s != %s" % (got.shape, ref.shape)
    if ref.size == 0:
        return
    scale = max(1.0, float(np.max(np.abs(ref))))
    err = float(np.max(np.abs(got.astype(np.complex128) - ref.astype(np.complex128))))
    assert err <= rel * scale, "max abs err %.3g > %.3g" % (err, rel * scale)


def ragged(rng, n, lo=0, hi=5000):
    cuts, i = [], 0
    while i < n:
        k = int(rng.integers(lo, hi))
        cuts.append((i, min(n, i + k)))
        i += k
    return cuts


def stream(blk, x, cuts):
    outs = [np.array(blk.process(Vector.cast(x[a:b])).data, copy=True) for a, b in cuts]
    return np.concatenate(outs)


def mk(cls, args, in_type, rate=2.0):
    b = cls(*args)
    b.get_rate = lambda: rate
    b.differentiate([in_type])
    b.initialize()
    return b


def rnd_c(rng, n):
    return (rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n)).astype(np.complex64)


@pytest.mark.parametrize("M", [1, 2, 16, 33, 128, 129, 500, 2048])
@pytest.mark.parametrize("kind", ["crcf", "cccf", "rrrf"])
def test_fir_stream(M, kind):
    rng = np.random.default_rng(M * 7 + len(kind))
    n = 60000
    taps = rng.uniform(-1, 1, M)
    if kind == "cccf":
        taps = taps + 1j * rng.uniform(-1, 1, M)
    taps = taps / np.sum(np.abs(taps))
    taps = taps.astype(np.complex64 if kind == "cccf" else np.float32)
    x = rng.uniform(-1, 1, n).astype(np.float32) if kind == "rrrf" else rnd_c(rng, n)
    in_t = Float32 if kind == "rrrf" else ComplexFloat32
    for use_fft in (None, False, True):
        blk = mk(radio.FIRFilterBlock, [(ComplexFloat32 if kind == "cccf" else Float32).vector_from_array(taps), use_fft], in_t)
        got = stream(blk, x, ragged(rng, n))
        ref = O.FIRFilter(taps, kind != "rrrf").process(x)
        close(got, ref)
        blk.cleanup()


@pytest.mark.parametrize("D", [2, 3, 4, 5, 7, 8, 10, 25])
@pytest.mark.parametrize("M", [16, 64, 128, 200])
def test_decimating_fir_matches_fir_then_downsample(D, M):
    """FIR with fused decimation (C ABI `decim`) == FIRFilter -> Downsampler of the oracle, any chunking."""
    rng = np.random.default_rng(D * 100 + M)
    n = 50000
    taps = O.f32_taps(O.firwin_lowpass(M, 1.0 / D))
    x = rnd_c(rng, n)
    lib = _lib.require_device()
    h = _lib.check_handle(lib.lrb200_fir_create_crcf(taps.ctypes.data, M, D, _lib.LRB200_HOST), "fir")
    outs = []
    for a, b in ragged(rng, n, 0, 3000):
        seg = np.ascontiguousarray(x[a:b])
        out = np.zeros(lib.lrb200_block_max_output(h, len(seg)), np.complex64)
        no = ctypes.c_size_t()
        _lib.check(lib.lrb200_fir_execute(h, seg.ctypes.data, len(seg), out.ctypes.data, ctypes.byref(no)))
        outs.append(out[:no.value])
    lib.lrb200_fir_destroy(h)
    ref = O.Chain(O.FIRFilter(taps, True), O.Downsampler(D)).process(x)
    close(np.concatenate(outs), ref)


def test_translator_large_index():
    """Phase is the closed form of the global sample index: seek to > 2^33 and compare with the oracle."""
    rng = np.random.default_rng(5)
    n = 20000
    x = rnd_c(rng, n)
    for offset, rate in ((-250e3, 1102500.0), (0.2, 2.0), (123456.789, 2.4e6)):
        blk = mk(radio.FrequencyTranslatorBlock, [offset], ComplexFloat32, rate)
        o = O.FrequencyTranslator(offset, rate)
        for n0 in (0, (1 << 33) + 12345):
            _lib.check(blk._lib.lrb200_block_seek(blk._handle, n0))
            o.n0 = n0
            got = stream(blk, x, ragged(rng, n))
            close(got, o.process(x), 2e-6)
        blk.cleanup()


def test_discriminator_and_downsampler_stream():
    rng = np.random.default_rng(6)
    n = 100001
    x = rnd_c(rng, n)
    blk = mk(radio.FrequencyDiscriminatorBlock, [1.25], ComplexFloat32)
    close(stream(blk, x, ragged(rng, n)), O.FrequencyDiscriminator(1.25).process(x), 2e-6)
    for D in (1, 2, 5, 7, 257):
        for xin, t in ((x, ComplexFloat32), (x.real.copy(), Float32)):
            b = mk(radio.DownsamplerBlock, [D], t)
            got = stream(b, xin, ragged(rng, n))
            assert np.array_equal(got, O.Downsampler(D).process(xin))    # pure gather: bit exact


@pytest.mark.parametrize("cplx", [False, True])
def test_single_pole_iir_long_stream(cplx):
    """Multi-tile decoupled look-back (n >> 2048-sample tiles), slow and fast poles, ragged chunks."""
    rng = np.random.default_rng(8)
    n = 400000
    x = rnd_c(rng, n) if cplx else rng.uniform(-1, 1, n).astype(np.float32)
    t = ComplexFloat32 if cplx else Float32
    for cls, args, rate, taps in (
        (radio.FMDeemphasisFilterBlock, [75e-6], 220500.0, O.fm_deemphasis_taps(75e-6, 220500.0)),
        (radio.SinglepoleLowpassFilterBlock, [10.0], 1e6, O.singlepole_lowpass_taps(10.0, 1e6)),
        (radio.SinglepoleHighpassFilterBlock, [1e3], 48e3, O.singlepole_highpass_taps(1e3, 48e3)),
    ):
        blk = mk(cls, args, t, rate)
        cuts = ragged(rng, n, 0, 90000)
        got = stream(blk, x, cuts)
        # the per-output bound of tests/iir_small_ref.py, over the same calls
        _, ref, bnd, _ = S.scan_bound(taps[0], taps[1], [x[a:b] for a, b in cuts], cplx)
        assert S.excess(got, ref, bnd) <= 1.0
        close(got, O.IIRFilterFast(taps[0], taps[1], cplx).process(x))
        blk.cleanup()


def test_hilbert_cmag_c2r_stream():
    rng = np.random.default_rng(9)
    n = 30000
    xr = rng.uniform(-1, 1, n).astype(np.float32)
    for M in (9, 65, 129, 257):
        blk = mk(radio.HilbertTransformBlock, [M], Float32)
        close(stream(blk, xr, ragged(rng, n)), O.HilbertTransform(M).process(xr))
    x = rnd_c(rng, n)
    close(stream(mk(radio.ComplexMagnitudeBlock, [], ComplexFloat32), x, ragged(rng, n)), O.complex_magnitude(x), 2e-7)
    assert np.array_equal(stream(mk(radio.ComplexToRealBlock, [], ComplexFloat32), x, ragged(rng, n)), O.complex_to_real(x))


def test_synth_sources_match_oracle():
    lib = _lib.require_device()
    n, n0 = 100000, (1 << 34) + 777
    d = lib.lrb200_malloc(n * 8)
    host = np.zeros(n, np.complex64)
    _lib.check(lib.lrb200_synth_white_iq(d, n0, n, 1))
    _lib.check(lib.lrb200_memcpy_d2h(host.ctypes.data, d, n * 8))
    _lib.check(lib.lrb200_sync())
    assert np.array_equal(host, O.synth_white_iq(n0, n, 1))          # integer hash: bit exact
    for start in (0, 268435456 - 50000):
        _lib.check(lib.lrb200_synth_fm_iq(d, start, n, 1, 1102500.0, 250e3, 75e3, 0.5, 0.01))
        _lib.check(lib.lrb200_memcpy_d2h(host.ctypes.data, d, n * 8))
        _lib.check(lib.lrb200_sync())
        close(host, O.synth_fm_iq(start, n), 2e-6)
    lib.lrb200_free(d)


def wbfm_graph(x, rate=1102500.0, fuse=True, chunk=1 << 22):
    src, snk = radio.ArraySource(x, rate, chunk), radio.ArraySink()
    top = radio.CompositeBlock()
    # examples/rtlsdr_wbfm_mono.lua:12-28
    top.connect(src, radio.TunerBlock(-250e3, 200e3, 5), radio.FrequencyDiscriminatorBlock(1.25),
                radio.LowpassFilterBlock(128, 15e3), radio.FMDeemphasisFilterBlock(75e-6),
                radio.DownsamplerBlock(5), snk)
    top.run(False, fuse=fuse)
    return snk.result(), top


@pytest.mark.parametrize("fuse", [True, False])
@pytest.mark.parametrize("chunk", [1 << 22, 100003, 1234])
def test_wbfm_mono_chain(fuse, chunk):
    """The full rtlsdr_wbfm_mono.lua chain as a GPU flow graph vs the oracle chain on synthetic FM."""
    n = 600000
    x = O.synth_fm_iq(0, n)
    got, top = wbfm_graph(x, fuse=fuse, chunk=chunk)
    ref = O.wbfm_mono_chain().process(x)
    close(got, ref)
    if fuse:
        assert "tuner" in top.describe_gpu_graph()
    # the demodulated tone must be there (sanity that the chain does FM demodulation, not just agreement)
    assert np.max(np.abs(ref[2000:])) > 0.05


@pytest.mark.parametrize("kind", ["crcf", "cccf", "rrrf"])
@pytest.mark.parametrize("D,M", [(5, 128), (7, 200), (3, 33), (25, 513), (2, 16)])
@pytest.mark.parametrize("algo", [_lib.FIR_AUTO, _lib.FIR_DIRECT, _lib.FIR_FFT])
def test_decimating_fir_all_kinds_and_algorithms(kind, D, M, algo):
    """C-ABI `decim` for every type combination and both algorithms == FIR -> Downsampler of the oracle."""
    rng = np.random.default_rng(D * 1000 + M + len(kind))
    n = 120000
    taps = O.firwin_lowpass(M, 1.0 / D)
    if kind == "cccf":
        taps = taps * np.exp(1j * 0.3 * np.arange(M))
    taps = O.f32_taps(taps)
    x = rng.uniform(-1, 1, n).astype(np.float32) if kind == "rrrf" else rnd_c(rng, n)
    lib = _lib.require_device()
    create = {"crcf": lib.lrb200_fir_create_crcf, "cccf": lib.lrb200_fir_create_cccf, "rrrf": lib.lrb200_fir_create_rrrf}[kind]
    h = _lib.check_handle(create(taps.ctypes.data, M, D, _lib.LRB200_HOST), "fir")
    _lib.check(lib.lrb200_fir_set_algorithm(h, algo))
    outs = []
    for a, b in ragged(rng, n, 0, 60000):
        seg = np.ascontiguousarray(x[a:b])
        out = np.zeros(lib.lrb200_block_max_output(h, len(seg)), x.dtype)
        no = ctypes.c_size_t()
        _lib.check(lib.lrb200_fir_execute(h, seg.ctypes.data, len(seg), out.ctypes.data, ctypes.byref(no)))
        outs.append(out[:no.value])
    lib.lrb200_fir_destroy(h)
    ref = O.Chain(O.FIRFilter(taps, kind != "rrrf"), O.Downsampler(D)).process(x)
    close(np.concatenate(outs), ref)


@pytest.mark.parametrize("fuse", [True, False])
@pytest.mark.parametrize("D", [1, 5])
def test_translator_complex_fir_decimate_graph(fuse, D):
    """BASELINE config 1 shape: FrequencyTranslator -> 128-tap COMPLEX-tap FIR -> /5, as a flow graph
    (fused: translator folded into the overlap-save kernel) vs the oracle."""
    rate, n = 1102500.0, 700000
    rng = np.random.default_rng(77)
    x = O.synth_white_iq(0, n)
    blocks = [radio.FrequencyTranslatorBlock(-250e3), radio.ComplexBandpassFilterBlock(128, [-100e3, 100e3])]
    if D > 1:
        blocks.append(radio.DownsamplerBlock(D))
    src, snk = radio.ArraySource(x, rate, 250001), radio.ArraySink()
    top = radio.CompositeBlock()
    top.connect(src, *blocks, snk)
    top.run(False, fuse=fuse)
    ochain = [O.FrequencyTranslator(-250e3, rate), O.complex_bandpass_filter(128, [-100e3, 100e3], rate)]
    if D > 1:
        ochain.append(O.Downsampler(D))
    close(snk.result(), O.Chain(*ochain).process(x))
    if fuse:
        assert "rot+fir_cccf" in top.describe_gpu_graph(), top.describe_gpu_graph()


def test_hilbert_long_call_uses_fft_path():
    rng = np.random.default_rng(10)
    n = 200000
    xr = rng.uniform(-1, 1, n).astype(np.float32)
    for M in (65, 129, 257):
        blk = mk(radio.HilbertTransformBlock, [M], Float32)
        got = np.concatenate([np.array(blk.process(Vector.cast(xr[:150000])).data, copy=True),
                              np.array(blk.process(Vector.cast(xr[150000:])).data, copy=True)])
        close(got, O.HilbertTransform(M).process(xr))


def test_c_abi_argument_errors():
    lib = _lib.require_device()
    taps = np.ones(4, np.float32)
    assert not lib.lrb200_fir_create_crcf(None, 4, 1, 0)
    assert not lib.lrb200_fir_create_crcf(taps.ctypes.data, 0, 1, 0)
    assert not lib.lrb200_fir_create_crcf(taps.ctypes.data, 4, 0, 0)
    assert b"decimation" in lib.lrb200_last_error()
    assert not lib.lrb200_hilbert_create(taps.ctypes.data, 4, 0)          # even tap count
    assert not lib.lrb200_downsample_create(0, 8, 0)
    assert not lib.lrb200_downsample_create(2, 3, 0)
    assert not lib.lrb200_discrim_create(0.0, 0)
    assert lib.lrb200_block_execute(None, None, 0, None, None) != 0
    h = lib.lrb200_fir_create_crcf(taps.ctypes.data, 4, 1, 0)
    assert h and lib.lrb200_fir_set_algorithm(h, 7) != 0
    assert lib.lrb200_block_execute(h, None, 5, None, None) != 0          # null buffers with n > 0
    lib.lrb200_fir_destroy(h)
    g = lib.lrb200_graph_create()
    hh = lib.lrb200_cmag_create(_lib.LRB200_HOST)
    assert lib.lrb200_graph_append(g, hh) != 0                            # host-mode block in a device graph
    lib.lrb200_block_destroy(hh)
    a, b = lib.lrb200_cmag_create(_lib.LRB200_DEVICE), lib.lrb200_cmag_create(_lib.LRB200_DEVICE)
    assert lib.lrb200_graph_append(g, a) == 0
    assert lib.lrb200_graph_append(g, b) != 0                             # float output cannot feed a complex input
    lib.lrb200_block_destroy(b)
    lib.lrb200_graph_destroy(g)


@pytest.mark.parametrize("cplx", [False, True])
def test_general_iir_long_stream(cplx):
    """IIRFilterBlock of order 2/4/8 on a long stream: the time-parallel chunks (warm-up restart) must agree with
    the sequential recurrence, for one big call and for ragged streaming."""
    import scipy.signal
    rng = np.random.default_rng(12)
    n = 300000
    x = rnd_c(rng, n) if cplx else rng.uniform(-1, 1, n).astype(np.float32)
    t = ComplexFloat32 if cplx else Float32
    for order, wn in ((2, 0.3), (4, 0.2), (8, 0.45)):
        b, a = scipy.signal.butter(order, wn)
        b, a = b.astype(np.float32), a.astype(np.float32)
        ref32 = O.IIRFilterFast(b, a, cplx).process(x)
        for cuts in ([(0, n)], ragged(rng, n, 0, 70000)):
            blk = mk(radio.IIRFilterBlock, [Float32.vector_from_array(b), Float32.vector_from_array(a)], t)
            got = stream(blk, x, cuts)
            # the per-output bound of tests/iir_small_ref.py over the same calls, and the 1e-5 tolerance, which is
            # tighter than the bound for butter(4, 0.2) and butter(8, 0.45) (their direct form amplifies rounding)
            ref, bnd, _ = S.general_bound(b, a, [x[lo:hi] for lo, hi in cuts], cplx)
            assert S.excess(got, ref, bnd) <= 1.0
            close(got, ref32)
            blk.cleanup()


def test_wbfm_chain_from_u8_iq_file():
    """RTL-SDR style u8 IQ 'file' -> fused WBFM chain in one flow graph (raw bytes over PCIe) == oracle on the
    oracle-converted samples."""
    n = 500000
    x = O.synth_fm_iq(0, n)
    u8 = np.clip(np.round(np.stack([x.real, x.imag], 1).reshape(-1) * 127.5 + 127.5), 0, 255).astype(np.uint8)
    src, snk = radio.IQFileSource(u8.tobytes(), "u8", 1102500.0, chunk=200001), radio.ArraySink()
    top = radio.CompositeBlock()
    top.connect(src, radio.TunerBlock(-250e3, 200e3, 5), radio.FrequencyDiscriminatorBlock(1.25),
                radio.LowpassFilterBlock(128, 15e3), radio.FMDeemphasisFilterBlock(75e-6), radio.DownsamplerBlock(5), snk)
    top.run(False)
    ref = O.wbfm_mono_chain().process(O.iq_file_convert(u8, "u8"))
    close(snk.result(), ref)
    assert top.describe_gpu_graph().startswith("iqconv(u8) | tuner+discrim")


@pytest.mark.parametrize("M", [514, 1025, 1536, 2048, 2049, 4097, 8192])
@pytest.mark.parametrize("kind", ["crcf", "cccf"])
def test_long_fir_partitioned_overlap_save(M, kind):
    """Filters longer than one FFT block allows run the partitioned overlap-save kernel (frequency-domain delay line):
    interior runs across many CTAs, ring wrap-around, head/tail runs against the carried history, accumulate launches
    for more than 4 partitions."""
    rng = np.random.default_rng(M + len(kind))
    n = 700000
    taps = rng.uniform(-1, 1, M)
    if kind == "cccf":
        taps = taps + 1j * rng.uniform(-1, 1, M)
    taps = (taps / np.sum(np.abs(taps))).astype(np.complex64 if kind == "cccf" else np.float32)
    x = rnd_c(rng, n)
    blk = mk(radio.FIRFilterBlock, [(ComplexFloat32 if kind == "cccf" else Float32).vector_from_array(taps), True], ComplexFloat32)
    cuts = [(0, 300001), (300001, 300013), (300013, 304000), (304000, n)]
    got = stream(blk, x, cuts)
    import scipy.signal
    ref = scipy.signal.fftconvolve(x.astype(np.complex128), taps.astype(np.complex128))[:n].astype(np.complex64)
    close(got, ref)
    blk.cleanup()


def test_wbfm_chain_u8_file_to_wav_file():
    """u8 IQ file -> fused WBFM chain -> 16-bit WAV, both file formats converted inside the GPU flow graph (the H2D copy
    carries 2 B/sample, the D2H copy 2 B/sample).  The PCM samples equal the oracle's within one LSB (a 1e-6 float
    difference can cross a truncation boundary)."""
    import io
    n = 400000
    x = O.synth_fm_iq(0, n)
    u8 = np.clip(np.round(np.stack([x.real, x.imag], 1).reshape(-1) * 127.5 + 127.5), 0, 255).astype(np.uint8)
    f = io.BytesIO()
    src, snk = radio.IQFileSource(u8.tobytes(), "u8", 1102500.0, chunk=150001), radio.WAVFileSink(f, 1, 16)
    top = radio.CompositeBlock()
    top.connect(src, radio.TunerBlock(-250e3, 200e3, 5), radio.FrequencyDiscriminatorBlock(1.25),
                radio.LowpassFilterBlock(128, 15e3), radio.FMDeemphasisFilterBlock(75e-6), radio.DownsamplerBlock(5), snk)
    top.run(False)
    desc = top.describe_gpu_graph()
    assert desc.startswith("iqconv(u8) | tuner+discrim") and desc.endswith("realsink(s16le)"), desc
    ref = O.wbfm_mono_chain().process(O.iq_file_convert(u8, "u8"))
    wav = f.getvalue()
    assert wav[:44] == O.wav_header(len(ref), 1, 16, 44100)
    got = np.frombuffer(wav[44:], "<i2").astype(np.int64)
    want = np.frombuffer(O.file_sink_convert(ref, "s16le").tobytes(), "<i2").astype(np.int64)
    assert got.shape == want.shape and np.max(np.abs(got - want)) <= 1


def run_demod(demod, x, rate, chunk):
    src, snk = radio.ArraySource(x, rate, chunk), radio.ArraySink()
    top = radio.CompositeBlock()
    top.connect(src, demod, snk)
    top.run(False)
    return snk.result(), top


@pytest.mark.parametrize("chunk", [1 << 20, 33333])
def test_nbfm_am_ssb_demodulators(chunk):
    """composites/nbfmdemodulator.lua, amenvelopedemodulator.lua, ssbdemodulator.lua (SURVEY 8f row 3, the chains that
    need no new block): each composite runs as one GPU flow graph and equals the oracle chain of the same blocks."""
    n, rate = 400000, 48000.0
    # NBFM: 5 kHz deviation FM at baseband with a little noise
    x = O.synth_fm_iq(0, n, 1, rate, 0.0, 5e3, 0.7, 0.005)
    got, top = run_demod(radio.NBFMDemodulator(), x, rate, chunk)
    ref = O.Chain(O.lowpass_filter(128, 9e3, rate, True), O.FrequencyDiscriminator(5e3 / 4e3),
                  O.lowpass_filter(128, 4e3, rate, False)).process(x)
    close(got, ref)
    assert np.max(np.abs(ref[1000:])) > 0.02
    assert top.describe_gpu_graph().count("|") == 2
    # AM envelope: carrier with 60 % modulation by two tones, plus noise
    t = np.arange(n) / rate
    env = 0.5 * (1 + 0.3 * np.sin(2 * np.pi * 440 * t) + 0.3 * np.sin(2 * np.pi * 1250 * t))
    rng = np.random.default_rng(3)
    xa = (env * np.exp(2j * np.pi * 0.013 * np.arange(n)) + 0.003 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))).astype(np.complex64)
    got, top = run_demod(radio.AMEnvelopeDemodulator(), xa, rate, chunk)
    b, a = O.singlepole_highpass_taps(100, rate)
    ref = O.Chain(O.complex_magnitude, O.IIRFilterFast(b, a, False), O.lowpass_filter(128, 5e3, rate, False)).process(xa)
    close(got, ref)
    assert np.max(np.abs(ref[20000:])) > 0.1
    # SSB, both sidebands
    xs = (rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n)).astype(np.complex64)
    for sb, cut in (("usb", [0, 3e3]), ("lsb", [0, -3e3])):
        got, top = run_demod(radio.SSBDemodulator(sb), xs, rate, chunk)
        ref = O.Chain(O.complex_bandpass_filter(129, cut, rate), O.complex_to_real, O.lowpass_filter(128, 3e3, rate, False)).process(xs)
        close(got, ref)
    with pytest.raises(AssertionError):
        radio.SSBDemodulator("dsb")


@pytest.mark.parametrize("L,D,M", [(2, 1, 128), (3, 1, 128), (7, 5, 128), (2, 3, 128), (3, 2, 128), (8, 4, 100), (5, 4, 64), (4, 25, 200),
                                   (160, 147, 1024), (5, 1, 33),
                                   # the remaining instantiations of the register-tiled kernel (resample.cu: the LRB_RS list) and its
                                   # tap-count limits (M = 255 is the largest the x2 shape takes, 300 falls back to the round-1 kernel)
                                   (4, 1, 128), (6, 1, 128), (7, 1, 100), (8, 1, 128), (2, 5, 128), (3, 4, 128), (3, 5, 90), (4, 3, 128),
                                   (4, 5, 128), (5, 2, 128), (5, 3, 77), (2, 1, 255), (2, 1, 300), (2, 1, 3)])
@pytest.mark.parametrize("cplx", [True, False])
def test_interpolator_and_rational_resampler_stream(L, D, M, cplx):
    """InterpolatorBlock / RationalResamplerBlock as one polyphase kernel (fused) and as four separate kernels (unfused)
    on a long stream in ragged chunks == oracle MultiplyConstant -> Upsampler -> Lowpass -> Downsampler."""
    rng = np.random.default_rng(L * 100 + D)
    n = 120000 if L < 100 else 20000
    x = rnd_c(rng, n) if cplx else rng.uniform(-1, 1, n).astype(np.float32)
    ref = (O.rational_resampler(L, D, cplx, M) if D > 1 else O.interpolator(L, cplx, M)).process(x)
    for fuse, chunk in ((True, 1 << 22), (True, 4099), (False, 30011)):
        src, snk = radio.ArraySource(x, 48000.0, chunk), radio.ArraySink()
        blk = radio.RationalResamplerBlock(L, D, {"num_taps": M}) if D > 1 else radio.InterpolatorBlock(L, {"num_taps": M})
        top = radio.CompositeBlock()
        top.connect(src, blk, snk)
        top.run(False, fuse=fuse)
        close(snk.result(), ref)
        if fuse:
            assert "upsample+fir" in top.describe_gpu_graph() and top.describe_gpu_graph().count("|") == 0, top.describe_gpu_graph()
        else:
            assert top.describe_gpu_graph().count("|") == (3 if D > 1 else 2), top.describe_gpu_graph()


# The CUDA chain against what the stock REFERENCE computed for the whole chain (tests/golden/wbfm_chain_ref_executed.npz, made
# by executing the reference's pure-Lua branches and run loop in the test interpreter; the oracle reproduces that vector to
# 4.5e-8 on the CPU, tests/test_oracle_golden.py).  A 1 650-sample stream: far shorter than anything else the chain is tested on.
@pytest.mark.parametrize("chunk", [1 << 22, 700])
def test_wbfm_mono_chain_reference_executed_golden(chunk):
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wbfm_chain_ref_executed.npz"))
    got, top = wbfm_graph(g["x"], rate=float(g["rate"]), fuse=False, chunk=chunk)
    close(got, g["y"])


# The FUSED graph (tuner+discrim | fir*iir1+pole) on the same vector.  The reference's FIRST discriminator output is atan2f
# of y[0] * conj(0), a product of SIGNED zeros -- pi / gain = 0.4 when both parts of y[0] are negative (one stream in four;
# this vector is one), 0 otherwise -- which the fused epilogue's fast atan2 would return as 0; tuner.cu redoes that one
# sample with IEEE operations in the edge-tile kernel.
@pytest.mark.parametrize("chunk", [1 << 22, 700])
def test_wbfm_mono_chain_reference_executed_golden_fused(chunk):
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wbfm_chain_ref_executed.npz"))
    got, top = wbfm_graph(g["x"], rate=float(g["rate"]), fuse=True, chunk=chunk)
    assert len(got) == len(g["y"]), (len(got), len(g["y"]))
    d = np.abs(got - g["y"])
    assert float(d.max()) <= 1e-5, "max |fused - reference| = %.3g at output %d of %d (graph %s)" % (float(d.max()), int(d.argmax()), len(d), top.describe_gpu_graph())


# ---- reset: every block kind with carried state ------------------------------------------------------------------------
# Each case runs x, then part of x (leaving state behind), resets, runs x again: the second full run must be bit-identical
# to the first.  Blocks go through lrb200_block_reset, graph-only fused stages through lrb200_graph_reset, a device DAG
# through lrb200_dag_reset.
N_RESET, PART = 100003, 12345


def _fir(kind, algo, decim):
    def create(lib):
        taps = np.linspace(-1, 1, 33, dtype=np.float32) * np.hamming(33).astype(np.float32)
        if kind == "cccf":
            taps = (taps + 0.5j * taps[::-1]).astype(np.complex64)
        h = getattr(lib, "lrb200_fir_create_" + kind)(taps.ctypes.data, len(taps), decim, _lib.LRB200_HOST)
        _lib.check(lib.lrb200_fir_set_algorithm(_lib.check_handle(h, "fir"), algo))
        return h
    return create, kind == "rrrf", 1


def _iir(cplx, order):
    def create(lib):
        import scipy.signal
        b, a = scipy.signal.butter(order, 0.1)
        b, a = b.astype(np.float32), a.astype(np.float32)
        return getattr(lib, "lrb200_iir_create_" + ("crcf" if cplx else "rrrf"))(b.ctypes.data, len(b), a.ctypes.data, len(a), _lib.LRB200_HOST)
    return create, not cplx, 1


HILBERT_TAPS = np.hamming(33).astype(np.float32)
BLOCK_RESET_CASES = {
    **{"fir_%s_%s_d%d" % (k, a, d): _fir(k, algo, d) for k in ("crcf", "cccf", "rrrf")
       for a, algo in (("direct", _lib.FIR_DIRECT), ("fft", _lib.FIR_FFT)) for d in (1, 3)},
    "hilbert": (lambda lib: lib.lrb200_hilbert_create(HILBERT_TAPS.ctypes.data, len(HILBERT_TAPS), _lib.LRB200_HOST), True, 1),
    "translator": (lambda lib: lib.lrb200_rotator_create(0.0123, _lib.LRB200_HOST), False, 1),
    "discriminator": (lambda lib: lib.lrb200_discrim_create(1.25, _lib.LRB200_HOST), False, 1),
    "iir_singlepole_rrrf": _iir(False, 1),
    "iir_singlepole_crcf": _iir(True, 1),
    "iir_general_rrrf": _iir(False, 4),
    "iir_general_crcf": _iir(True, 4),
    "delay": (lambda lib: lib.lrb200_delay_create(100, 8, _lib.LRB200_HOST), False, 1),
    "pll": (lambda lib: lib.lrb200_pll_create(1000.0, -2e3, 2e3, 2.0, 1e5, _lib.LRB200_HOST), False, 2),
    # AGCBlock('custom', -20, -40, {gain_tau = 1e-3, power_tau = 5e-5}) and PowerSquelchBlock(-45) at 1 MHz, complex
    "agc": (lambda lib: lib.lrb200_agc_create(-20.0, -40.0, 1e-3, 5e-5, 1e6, 1, _lib.LRB200_HOST), "bursty", 1),
    "powersquelch": (lambda lib: lib.lrb200_powersquelch_create(-45.0, 1e-3, 1e6, 1, _lib.LRB200_HOST), "bursty", 1),
}


def _reset_input(real):
    if real == "bursty":             # the level blocks' gate opens and closes inside tiles, on tile edges and for whole tiles
        from tests.test_gpu_level import bursty_stream
        return bursty_stream(1 << 20, True, 3)
    rng = np.random.default_rng(21)
    t = np.arange(N_RESET)
    x = (np.exp(2j * np.pi * 0.003 * t) * (0.1 + 0.1 * (t % 20000 < 9000)) + 0.01 * rnd_c(rng, N_RESET)).astype(np.complex64)
    return np.ascontiguousarray(x.real) if real else x


def _run_ports(lib, h, x, nout):
    cap = lib.lrb200_block_max_output(h, len(x))
    outs = [np.zeros(cap * 8, np.uint8) for _ in range(nout)]
    ins = (ctypes.c_void_p * 1)(x.ctypes.data)
    ptrs = (ctypes.c_void_p * nout)(*[o.ctypes.data for o in outs])
    no = ctypes.c_size_t()
    _lib.check(lib.lrb200_block_execute_multi(h, ins, 1, len(x), ptrs, nout, ctypes.byref(no)), "execute")
    return [o[:no.value * lib.lrb200_block_out_size(h) if k == 0 else no.value * 4] for k, o in enumerate(outs)]


@pytest.mark.parametrize("case", list(BLOCK_RESET_CASES))
def test_block_reset_restores_the_initial_state(case):
    lib = _lib.require_device()
    create, real, nout = BLOCK_RESET_CASES[case]
    h = _lib.check_handle(create(lib), case)
    try:
        x = _reset_input(real)
        first = _run_ports(lib, h, x, nout)
        _run_ports(lib, h, x[:PART], nout)
        _lib.check(lib.lrb200_block_reset(h), "reset")
        again = _run_ports(lib, h, x, nout)
        assert len(first[0]) > 0
        for a, b in zip(first, again):
            assert np.array_equal(a, b), case
    finally:
        lib.lrb200_block_destroy(h)


def _audio_tail(rate):
    # FIR -> de-emphasis -> /5: one stage with the pole fused when c^5 decays fast enough (low rate), else FIR | pole
    return [mk(radio.LowpassFilterBlock, (128, 15e3), Float32, rate), mk(radio.FMDeemphasisFilterBlock, (75e-6,), Float32, rate),
            mk(radio.DownsamplerBlock, (5,), Float32, rate)]


GRAPH_RESET_CASES = {
    "tuner+discrim": (lambda: [mk(radio.FrequencyTranslatorBlock, (-1e5,), ComplexFloat32, 1e6),
                               mk(radio.LowpassFilterBlock, (128, 1e5), ComplexFloat32, 1e6),
                               mk(radio.DownsamplerBlock, (5,), ComplexFloat32, 1e6),
                               mk(radio.FrequencyDiscriminatorBlock, (1.25,), ComplexFloat32, 1e6)], False, np.float32, "tuner+discrim("),
    "fir*iir1_rrrf+pole": (lambda: _audio_tail(1e5), True, np.float32, ")+pole"),
    "fir*iir1_rrrf|pole_rrrf": (lambda: _audio_tail(1e6), True, np.float32, " | pole_rrrf"),
    "resampler": (lambda: [mk(radio.UpsamplerBlock, (3,), ComplexFloat32, 1e6),
                           mk(radio.LowpassFilterBlock, (64, 1e5), ComplexFloat32, 3e6),
                           mk(radio.DownsamplerBlock, (2,), ComplexFloat32, 3e6)], False, np.complex64, "upsample+fir+down("),
    "interpolator": (lambda: [mk(radio.UpsamplerBlock, (4,), Float32, 1e6),
                              mk(radio.LowpassFilterBlock, (64, 1e5), Float32, 4e6)], True, np.float32, "upsample+fir("),
    "iir/D": (lambda: [mk(radio.SinglepoleLowpassFilterBlock, (1e4,), ComplexFloat32, 1e6),
                       mk(radio.DownsamplerBlock, (4,), ComplexFloat32, 1e6)], False, np.complex64, "iir_crcf[fused x2]"),
}


@pytest.mark.parametrize("case", list(GRAPH_RESET_CASES))
def test_graph_reset_restores_the_initial_state(case):
    lib = _lib.require_device()
    make_blocks, real, out_dtype, fused_name = GRAPH_RESET_CASES[case]
    g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
    try:
        for b in make_blocks():
            _lib.check(lib.lrb200_graph_append(g, b.make_device_handle()), "append")
        _lib.check(lib.lrb200_graph_commit(g, 1), "commit")
        assert fused_name in lib.lrb200_graph_describe(g).decode(), lib.lrb200_graph_describe(g)
        x = _reset_input(real)

        def run(v):
            y = np.zeros(lib.lrb200_graph_max_output(g, len(v)), out_dtype)
            no = ctypes.c_size_t()
            _lib.check(lib.lrb200_graph_execute(g, v.ctypes.data, len(v), y.ctypes.data, ctypes.byref(no)), "execute")
            return y[:no.value]
        first = run(x)
        run(x[:PART])
        _lib.check(lib.lrb200_graph_reset(g), "graph_reset")
        assert len(first) > 0 and np.array_equal(run(x).view(np.uint32), first.view(np.uint32))
    finally:
        lib.lrb200_graph_destroy(g)


def test_dag_reset_restores_the_initial_state():
    """The WBFM-stereo demodulator as one device DAG (PLL, delay, fused FIR runs, binary blocks, de-emphasis)."""
    from luaradio_b200.composite import GPUDagBlock
    lib = _lib.require_device()
    rate, n = 220500.0, 60000
    t = np.arange(n) / rate
    mpx = 0.4 * np.sin(2 * np.pi * 700 * t) + 0.1 * np.sin(2 * np.pi * 19e3 * t) + 0.3 * np.sin(2 * np.pi * 2300 * t) * np.sin(2 * np.pi * 38e3 * t)
    x = np.exp(2j * np.pi * 75e3 * np.cumsum(mpx) / rate).astype(np.complex64)
    top = radio.CompositeBlock()
    demod = radio.WBFMStereoDemodulator()
    top.connect(radio.ArraySource(x, rate, n), demod)
    top.connect(demod, "left", radio.ArraySink(), "in")
    top.connect(demod, "right", radio.ArraySink(), "in")
    top._prepare_to_run()
    top._collapse_gpu_runs(True, 0, True)
    dags = [c for c in top._chains if isinstance(c, GPUDagBlock)]
    try:
        assert len(dags) == 1
        dag = dags[0]

        def run(v):
            return [np.array(o.data, copy=True) for o in dag.process(Vector.cast(v))]
        first = run(x)
        run(x[:PART])
        _lib.check(lib.lrb200_dag_reset(dag.dag), "dag_reset")
        again = run(x)
        assert len(first[0]) == n
        for a, b in zip(first, again):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    finally:
        for c in top._chains:
            c.cleanup()
