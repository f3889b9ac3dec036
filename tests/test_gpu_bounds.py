"""Buffer boundaries of every DEVICE-mode kernel: caller-owned pointers at any natural alignment, nothing read or written
outside [x, x+n) / [y, y+n_out).

In LRB200_DEVICE mode the caller's pointers reach the kernels unchanged (Block::execute_multi, graph run_device), so a
torch slice or a sub-buffer of a larger allocation is 4- or 8-byte aligned and sits between other data.  Each case below
runs one stream of calls through one handle and checks, per call:

  * guarded buffers: every input and output is one lrb200_malloc allocation [guard | payload | guard] with GUARD bytes on
    each side (>= 64 Ki elements of every sample type here, and far more than twice any block's look-back), so a stray
    access lands inside the allocation;
  * poison, run twice: everything in the input allocations outside [x, x+n) holds pattern A (a quiet NaN with a payload;
    bytes 0x00 for raw file formats), the run is repeated from a reset handle with pattern B (a large finite value; bytes
    0xFF for raw formats).  The two runs must be bit-identical and the float outputs NaN-free: a stray read shows up as a
    NaN, or as a difference when a comparison swallows the NaN;
  * output sentinels: the whole output allocation is filled with a sentinel NaN before each call (a different one in
    each run); afterwards everything outside [y, y+n_out) must still hold it byte for byte, and the two runs being
    bit-identical means every slot in [0, n_out) was written (an unwritten slot holds two different sentinels);
  * offsets: the calls cycle x / y between 16-byte aligned and merely naturally aligned placements (4 B for float32,
    8 B for complex, the component width for raw file formats), so both sides of every alignment-selected branch run,
    and successive calls move between them while the carried state crosses every call boundary;
  * lengths: 0, 1, 2 and T-1, T, T+1, 2T-1, 2T+1 for the kernel's tile or launch unit T (read from its source), plus one
    long call, so that tails, whole tiles and grid-stride / persistent loops all run;
  * references: the stream's concatenated output against the project's references at the tolerance the other GPU tests
    use for the block; where the aligned and unaligned paths differ only in how they load and store, the output must
    also be bit-identical to the same call sequence run at 16-byte aligned offsets only (`exact`).
"""
import ctypes

import numpy as np
import pytest

from luaradio_b200 import _lib
from oracle import lr_oracle as O

pytestmark = pytest.mark.gpu

GUARD = 1 << 19                     # bytes on each side of a payload
POISON_A, POISON_B = 0x7FC0DEAD, 0x5A5A5A5A
SENTINELS = (0x7FC5EE1D, 0xFFC0FFEE)


class Port:
    """One input or output stream: bytes per sample, natural alignment, 'c' (complex64) / 'f' (float32) / 'raw'."""

    def __init__(self, size, align, kind):
        self.size, self.align, self.kind = size, align, kind

    def view(self, b):
        return b.view({"c": np.complex64, "f": np.float32, "raw": np.uint8}[self.kind])

    def poison(self, run):
        if self.kind == "raw":
            return np.full(4, (0x00, 0xFF)[run], np.uint8)
        return np.array([(POISON_A, POISON_B)[run]], "<u4").view(np.uint8)


CPX, FLT = Port(8, 8, "c"), Port(4, 4, "f")
RAW_WIDTH = {"u8": 1, "s16le": 2, "s16be": 2, "f32le": 4}


class Case:
    """`create` is the lrb200_*_create entry point the case exercises; `make(lib)` returns a block handle (or, with
    graph=True, a committed graph handle and the describe() prefix / substring it must show); `gen(rng, n)` the input
    streams; `ref(inputs)` the expected output streams of the whole stream (with ref_calls=True, `ref(inputs, ns)`, ns
    the call lengths the stream is run in); `cmp` how they are compared."""

    def __init__(self, create, make, ins, outs, lengths, gen, ref, cmp, exact=False, graph=False, describe=None,
                 repeatable=True, ref_calls=False):
        self.create, self.make, self.ins, self.outs = create, make, ins, outs
        self.lengths, self.gen, self.ref, self.cmp = lengths, gen, ref, cmp
        self.exact, self.graph, self.describe, self.repeatable = exact, graph, describe, repeatable
        self.ref_calls = ref_calls


def around(*units):
    out = []
    for t in units:
        out += [t - 1, t, t + 1, 2 * t - 1, 2 * t + 1]
    return out


def base_lengths(*units, big=300000):
    seen, out = set(), []
    for n in [0, 1, 2] + around(*units) + [big]:
        if callable(n) or n not in seen:
            out.append(n)
            seen.add(n)
    return out


def rnd_c(rng, n):
    return (rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n)).astype(np.complex64)


def rnd_f(rng, n):
    return rng.uniform(-1, 1, n).astype(np.float32)


def fir_ref(taps, x, D=1, wide=False):
    """y[n] = sum_k taps[k] x[n-k] from zero history (oracle FIRFilter), by FFT convolution in float64, every D-th.
    wide: return the float64 / complex128 result instead of rounding it to float32 / complex64."""
    import scipy.signal
    cplx = np.iscomplexobj(x) or np.iscomplexobj(taps)
    if len(x) == 0:
        return np.zeros(0, (np.complex128 if wide else np.complex64) if cplx else (np.float64 if wide else np.float32))
    y = scipy.signal.fftconvolve(x.astype(np.complex128 if cplx else np.float64),
                                 np.asarray(taps).astype(np.complex128 if cplx else np.float64))[:len(x)][::D]
    return y if wide else y.astype(np.complex64 if cplx else np.float32)


# ---- tolerance checks, each the one the block's other GPU tests use ---------------------------------------------------
def cmp_rel(rel):
    def check(got, ref, what):
        scale = max(1.0, float(np.max(np.abs(ref)))) if ref.size else 1.0
        err = float(np.max(np.abs(got.astype(np.complex128) - ref.astype(np.complex128)))) if ref.size else 0.0
        assert err <= rel * scale, "%s: max abs err %.3g > %.3g" % (what, err, rel * scale)
    return check


def cmp_abs(tol):
    def check(got, ref, what):
        err = float(np.max(np.abs(got.astype(np.complex128) - ref.astype(np.complex128)))) if ref.size else 0.0
        assert err <= tol, "%s: max abs err %.3g > %.3g" % (what, err, tol)
    return check


def cmp_exact(got, ref, what):
    assert np.array_equal(np.asarray(got).view(np.uint8), np.asarray(ref).view(np.uint8)), what


def cmp_ulp4(got, ref, what):
    from tests.test_gpu_level import check_close
    check_close(got, ref, what)


# ---- the cases ---------------------------------------------------------------------------------------------------------
# Tiles and launch units, from the kernels:
FFT_HOP33 = 1024 - 33 + 1          # fir_fft.cu: FF_N = 1024, hop L = N - M + 1 (doubled for the paired real blocks)
PG_TO = 128 * 8                    # poly_generic.cu: PG_THREADS * PG_R outputs per tile
PT_TO = 64 * 8                     # tuner.cu: PT_THREADS * PT_R outputs per tile
LV_TILE = 256 * 8                  # level.cu: LV_THREADS * LV_V
PC_TILE = 256 * 8                  # phasecorr.cu: PC_THREADS * PC_V
IIR_TILE, IIR_PAY = 512 * 8, 512 * 8 - 512      # iir.cu: first tile, payload of the later (warm-up restarted) tiles
IT_TILE = 4 * 128                  # resample.cu: IT_R * IT_THREADS inputs per interpolator tile
EW_UNITS = (2, 4)                  # elementwise.cu: samples per 128-bit rotator / discrim, cmag, c2r step


def tuner_exact(k, delta, disc, D=5, Q=26):
    """A call length at which the tuner's last interior tile ends exactly on the call's input (lim / step exact in
    tuner.cu launch_shape), +-1.  Depends on the decimation phase the call starts at, hence a function of `consumed`."""
    TS = PT_TO - 8 if disc else PT_TO                  # TileStride: DISC_OV + DISC_TAIL = 8 slots of overlap
    span = (PT_TO + Q - 1) * D + 1
    loaded = 2 * (((span + 1) // 2 + 63) // 64) * 64   # PolyShape::LOADED for 64 threads

    def n_for(consumed):
        first = (D - consumed % D) % D
        off = first - (4 * D if disc else 0) - (Q * D - 1)
        off -= off % 2
        return k * TS * D + loaded + off + delta
    return n_for


def tuner_lengths(disc):
    TS = PT_TO - 8 if disc else PT_TO
    exact = [tuner_exact(k, d, disc) for k in (1, 40) for d in (-1, 0, 1)]
    return base_lengths(TS * 5, big=2000003) + exact      # 2 M inputs: the persistent interior CTAs loop more than once


def _fir_case(kind, algo, D, M=33, lengths=None, exact=True):
    rng = np.random.default_rng(M * 10 + D)
    taps = rng.uniform(-1, 1, M) + (1j * rng.uniform(-1, 1, M) if kind == "cccf" else 0)
    taps = (taps / np.sum(np.abs(taps))).astype(np.complex64 if kind == "cccf" else np.float32)

    def make(lib):
        h = _lib.check_handle(getattr(lib, "lrb200_fir_create_" + kind)(taps.ctypes.data, M, D, _lib.LRB200_DEVICE), "fir")
        _lib.check(lib.lrb200_fir_set_algorithm(h, algo), "set_algorithm")
        return h
    port = FLT if kind == "rrrf" else CPX
    if lengths is None:
        lengths = base_lengths(FFT_HOP33, 2 * FFT_HOP33, PG_TO * D)
    return Case("lrb200_fir_create_" + kind, make, [port], [port], lengths,
                lambda rng, n: [(rnd_f if kind == "rrrf" else rnd_c)(rng, n)],
                lambda xs: [fir_ref(taps, xs[0], D)], cmp_rel(1e-5), exact=exact)


def _iir_case(cplx, b, a, lengths, look_back=False):
    """look_back: a slow pole runs the decoupled look-back scan, whose carries are summed in whatever order the
    predecessors' aggregates and prefixes become visible, so two runs of the same stream agree to rounding, not bit
    for bit: both runs are compared with the reference instead of with each other."""
    from tests import iir_small_ref as S
    b, a = np.asarray(b, np.float32), np.asarray(a, np.float32)
    port = CPX if cplx else FLT
    bounds = {}

    def ref(xs, ns):
        # the per-output bound of tests/iir_small_ref.py, over the calls the stream is run in
        calls = np.split(xs[0], np.cumsum(ns)[:-1])
        if len(a) <= 2 and len(b) <= 9:
            _, r, bnd, _ = S.scan_bound(b, a, calls, cplx)
        else:
            r, bnd, _ = S.general_bound(b, a, calls, cplx)
        bounds[len(r)] = bnd
        return [r]

    def cmp(got, r, what):
        # the bound, and the tolerance these cases were held to before it (the bound is looser than that for the
        # general-order designs, whose direct form amplifies float32 rounding)
        e = S.excess(np.asarray(got), np.asarray(r, np.complex128 if cplx else np.float64), bounds[len(r)])
        assert e <= 1.0, "%s: error %.3g of the bound" % (what, e)
        cmp_rel(1e-5)(got, np.asarray(r), what)
    return Case("lrb200_iir_create_" + ("crcf" if cplx else "rrrf"),
                lambda lib: getattr(lib, "lrb200_iir_create_" + ("crcf" if cplx else "rrrf"))(b.ctypes.data, len(b), a.ctypes.data, len(a), _lib.LRB200_DEVICE),
                [port], [port], lengths, lambda rng, n: [(rnd_c if cplx else rnd_f)(rng, n)],
                ref, cmp, exact=not look_back, repeatable=not look_back, ref_calls=True)


def _general_iir_taps():
    import scipy.signal
    return scipy.signal.butter(4, 0.2)


HILBERT_TAPS = O.f32_taps(O.fir_hilbert_transform(33))
PSD_FRAMES = (64, 1024)
PLL_ARGS = (100.0, 19e3 - 50, 19e3 + 50, 2.0, 220500.0)
PLL_L = 50536                      # pll.cu PllBlock: max(4 ceil(24 / (zeta bw)), 16384) for PLL_ARGS
PLL_PARALLEL_LENGTHS = [1, 2 * PLL_L - 1, 2 * PLL_L, 2 * PLL_L + 1, 3 * PLL_L + 5]
AGC_ARGS, AGC_RATE = ("custom", -20, -40, {"gain_tau": 1e-3, "power_tau": 5e-5}), 1e6
SQ_ARGS, SQ_RATE = (-45,), 1e5


def _psd_case(N):
    win = np.array(O.window(N, "hamming", True), np.float32)
    rate = 1e6
    scale = rate * float(np.sum(win.astype(np.float64) ** 2))
    return Case("lrb200_psd_create", lambda lib: lib.lrb200_psd_create(N, win.ctypes.data, scale, 0, 1, _lib.LRB200_DEVICE),
                [CPX], [FLT], [0, N, 2 * N, 3 * N, 37 * N, (300000 // N) * N],
                lambda rng, n: [(rnd_c(rng, n) * 0.3 + np.exp(2j * np.pi * 0.123 * np.arange(n))).astype(np.complex64)],
                lambda xs: [np.concatenate([np.zeros(0, np.float32)] + [O.psd(xs[0][i:i + N], "hamming", rate, False)
                                                                       for i in range(0, len(xs[0]), N)])], cmp_rel(2e-5))


def _pll_input(rng, n):
    t = np.arange(n) / PLL_ARGS[4]
    return [(0.8 * np.exp(2j * np.pi * 19000.3 * t + 0.4j) + 0.05 * rnd_c(rng, n)).astype(np.complex64)]


def _pll_parallel(lib):
    h = _lib.check_handle(lib.lrb200_pll_create(*PLL_ARGS, _lib.LRB200_DEVICE), "pll")
    _lib.check(lib.lrb200_pll_set_mode(h, 1), "pll_set_mode")
    return h


def _pll_parallel_cmp():
    from tests import pll_ref as P
    lp = P.Loop(*PLL_ARGS)
    assert lp.L == PLL_L
    calls = PLL_PARALLEL_LENGTHS * len(_placements(1, 2))
    return cmp_abs(2e-5 + max(P.ERR_TOL, P.out_tol(P.lead_ins(calls, lp))))


def _level_case(agc, cplx):
    from tests.test_gpu_level import bursty_stream, reference
    cls, args, rate = ("AGCBlock", AGC_ARGS, AGC_RATE) if agc else ("PowerSquelchBlock", SQ_ARGS, SQ_RATE)
    port = CPX if cplx else FLT
    if agc:
        make = lambda lib: lib.lrb200_agc_create(-20.0, -40.0, 1e-3, 5e-5, AGC_RATE, int(cplx), _lib.LRB200_DEVICE)    # noqa: E731
    else:
        make = lambda lib: lib.lrb200_powersquelch_create(-45.0, 1e-3, SQ_RATE, int(cplx), _lib.LRB200_DEVICE)       # noqa: E731
    return Case("lrb200_agc_create" if agc else "lrb200_powersquelch_create", make, [port], [port],
                base_lengths(LV_TILE), lambda rng, n: [bursty_stream(n, cplx, 3)],
                lambda xs: [reference(cls, args, rate, xs[0])[0]], cmp_ulp4, exact=True)


def _phasecorr_case(N, I):
    from tests import rds_oracle as R
    from tests.test_gpu_rds import drifting_bpsk
    return Case("lrb200_phasecorrector_create", lambda lib: lib.lrb200_phasecorrector_create(N, I, _lib.LRB200_DEVICE),
                [CPX], [CPX], base_lengths(PC_TILE, N * I), lambda rng, n: [drifting_bpsk(n, N + I)],
                lambda xs: [R.BinaryPhaseCorrector(N, I).process(xs[0])], cmp_rel(1e-5), exact=True)


def _raw_input(fmt, rng, n_components):
    if fmt == "f32le":
        return rnd_f(rng, n_components).astype("<f4").view(np.uint8)
    return rng.integers(0, 256, n_components * RAW_WIDTH[fmt], dtype=np.uint8)


def _source_case(fmt, iq):
    w = RAW_WIDTH[fmt]
    fn = "lrb200_iqconv_create" if iq else "lrb200_realconv_create"
    return Case(fn, lambda lib: getattr(lib, fn)(fmt.encode(), _lib.LRB200_DEVICE), [Port(w * (2 if iq else 1), w, "raw")],
                [CPX if iq else FLT], base_lengths(*EW_UNITS, 256),
                lambda rng, n: [_raw_input(fmt, rng, n * (2 if iq else 1))],
                lambda xs: [(O.iq_file_convert if iq else O.real_file_convert)(xs[0], fmt)], cmp_exact, exact=True)


def _sink_case(fmt, iq):
    w = RAW_WIDTH[fmt]
    fn = "lrb200_iqsink_create" if iq else "lrb200_realsink_create"
    return Case(fn, lambda lib: getattr(lib, fn)(fmt.encode(), _lib.LRB200_DEVICE), [CPX if iq else FLT],
                [Port(w * (2 if iq else 1), w, "raw")], base_lengths(*EW_UNITS, 256),
                lambda rng, n: [(rnd_c if iq else rnd_f)(rng, n)],
                lambda xs: [O.file_sink_convert(xs[0], fmt)], cmp_exact, exact=True)


def _binary_case(op, cplx):
    port = CPX if cplx else FLT
    gen = rnd_c if cplx else rnd_f
    return Case("lrb200_binary_create", lambda lib: lib.lrb200_binary_create(op.encode(), int(cplx), _lib.LRB200_DEVICE),
                [port, port], [port], base_lengths(*EW_UNITS), lambda rng, n: [gen(rng, n), gen(rng, n)],
                lambda xs: [O.binary_op(op, xs[0], xs[1])], cmp_rel(1e-5), exact=True)


BLOCK_CASES = {
    # FIRFilterBlock: direct / overlap-save, decimation 1 / 3 (no alignment branch: exact across offsets)
    **{"fir_%s_%s_d%d" % (k, a, d): (lambda k=k, algo=algo, d=d: _fir_case(k, algo, d))
       for k in ("crcf", "cccf", "rrrf") for a, algo in (("direct", _lib.FIR_DIRECT), ("fft", _lib.FIR_FFT)) for d in (1, 3)},
    # register-tiled polyphase shapes (tuner.cu): x not 16-byte (real: 8-byte) aligned sends every tile to the edge kernel
    "fir_crcf_poly_m16": lambda: _fir_case("crcf", _lib.FIR_AUTO, 1, 16, base_lengths(PT_TO), exact=False),
    "fir_crcf_poly_m32": lambda: _fir_case("crcf", _lib.FIR_AUTO, 1, 32, base_lengths(PT_TO), exact=False),
    "fir_crcf_poly_m128_d5": lambda: _fir_case("crcf", _lib.FIR_AUTO, 5, 128, base_lengths(PT_TO * 5), exact=False),
    "fir_rrrf_poly_m133_d5": lambda: _fir_case("rrrf", _lib.FIR_AUTO, 5, 133, base_lengths(2 * PT_TO * 5), exact=False),
    # partitioned overlap-save (hop 512 per partition)
    "fir_cccf_m1025": lambda: _fir_case("cccf", _lib.FIR_FFT, 1, 1025, base_lengths(512)),
    "hilbert": lambda: Case("lrb200_hilbert_create",
                            lambda lib: lib.lrb200_hilbert_create(HILBERT_TAPS.ctypes.data, len(HILBERT_TAPS), _lib.LRB200_DEVICE),
                            [FLT], [CPX], base_lengths(FFT_HOP33, 2 * FFT_HOP33), lambda rng, n: [rnd_f(rng, n)],
                            lambda xs: [O.HilbertTransform(33).process(xs[0])], cmp_rel(1e-5), exact=True),
    "translator": lambda: Case("lrb200_rotator_create", lambda lib: lib.lrb200_rotator_create(0.0123, _lib.LRB200_DEVICE),
                               [CPX], [CPX], base_lengths(*EW_UNITS), lambda rng, n: [rnd_c(rng, n)],
                               lambda xs: [O.FrequencyTranslator(0.0123, 1.0).process(xs[0])], cmp_rel(2e-6), exact=True),
    "discriminator": lambda: Case("lrb200_discrim_create", lambda lib: lib.lrb200_discrim_create(2 * np.pi * 1.25, _lib.LRB200_DEVICE),
                                  [CPX], [FLT], base_lengths(*EW_UNITS), lambda rng, n: [rnd_c(rng, n)],
                                  lambda xs: [O.FrequencyDiscriminator(1.25).process(xs[0])], cmp_rel(2e-6), exact=True),
    **{"downsample_%db" % e: (lambda e=e: Case("lrb200_downsample_create", lambda lib: lib.lrb200_downsample_create(3, e, _lib.LRB200_DEVICE),
                                                [CPX if e == 8 else FLT], [CPX if e == 8 else FLT], base_lengths(3, *EW_UNITS),
                                                lambda rng, n: [(rnd_c if e == 8 else rnd_f)(rng, n)],
                                                lambda xs: [O.Downsampler(3).process(xs[0])], cmp_exact, exact=True)) for e in (4, 8)},
    **{"upsample_%db" % e: (lambda e=e: Case("lrb200_upsample_create", lambda lib: lib.lrb200_upsample_create(3, e, _lib.LRB200_DEVICE),
                                              [CPX if e == 8 else FLT], [CPX if e == 8 else FLT], base_lengths(*EW_UNITS),
                                              lambda rng, n: [(rnd_c if e == 8 else rnd_f)(rng, n)],
                                              lambda xs: [O.Upsampler(3).process(xs[0])], cmp_exact, exact=True)) for e in (4, 8)},
    "cmag": lambda: Case("lrb200_cmag_create", lambda lib: lib.lrb200_cmag_create(_lib.LRB200_DEVICE), [CPX], [FLT],
                         base_lengths(*EW_UNITS), lambda rng, n: [rnd_c(rng, n)],
                         lambda xs: [O.complex_magnitude(xs[0])], cmp_rel(2e-7), exact=True),
    "c2r": lambda: Case("lrb200_c2r_create", lambda lib: lib.lrb200_c2r_create(_lib.LRB200_DEVICE), [CPX], [FLT],
                        base_lengths(*EW_UNITS), lambda rng, n: [rnd_c(rng, n)],
                        lambda xs: [O.complex_to_real(xs[0])], cmp_exact, exact=True),
    **{"mulconst_%s" % name: (lambda c=c, cd=cd: Case(
        "lrb200_mulconst_create", lambda lib: lib.lrb200_mulconst_create(c.real, c.imag, int(cd), int(isinstance(c, complex)), _lib.LRB200_DEVICE),
        [CPX if cd else FLT], [CPX if cd else FLT], base_lengths(*EW_UNITS), lambda rng, n: [(rnd_c if cd else rnd_f)(rng, n)],
        lambda xs: [O.MultiplyConstant(c).process(xs[0])], cmp_rel(1e-5), exact=True))
       for name, c, cd in (("cc", 0.5 - 0.25j, True), ("cr", 1.5, True), ("rr", 1.5, False))},
    # single pole: a fast pole (de-emphasis at 220.5 kHz, warm-up restart) and a slow one (10 Hz at 1 MHz, look-back)
    **{"iir1_%s_%s" % (speed, "crcf" if c else "rrrf"): (lambda c=c, taps=taps, speed=speed: _iir_case(
        c, taps[0], taps[1], base_lengths(IIR_TILE, IIR_TILE + IIR_PAY), look_back=speed == "slow"))
       for speed, taps in (("fast", O.fm_deemphasis_taps(75e-6, 220500.0)), ("slow", O.singlepole_lowpass_taps(10.0, 1e6)))
       for c in (False, True)},
    **{"iir_general_%s" % ("crcf" if c else "rrrf"): (lambda c=c: _iir_case(c, *_general_iir_taps(), base_lengths(IIR_TILE)))
       for c in (False, True)},
    **{"binary_%s_%s" % (op, "cc" if c else "rr"): (lambda op=op, c=c: _binary_case(op, c))
       for op in ("multiply", "multiplyconjugate", "add", "subtract") for c in (False, True) if c or op != "multiplyconjugate"},
    **{"delay_%db" % e: (lambda e=e: Case("lrb200_delay_create", lambda lib: lib.lrb200_delay_create(100, e, _lib.LRB200_DEVICE),
                                           [CPX if e == 8 else FLT], [CPX if e == 8 else FLT], base_lengths(100, *EW_UNITS),
                                           lambda rng, n: [(rnd_c if e == 8 else rnd_f)(rng, n)],
                                           lambda xs: [O.Delay(100).process(xs[0])], cmp_exact, exact=True)) for e in (4, 8)},
    **{"psd_%d" % N: (lambda N=N: _psd_case(N)) for N in PSD_FRAMES},
    # one thread runs the recurrence: short calls (and the oracle is a per-sample loop)
    "pll": lambda: Case("lrb200_pll_create", lambda lib: lib.lrb200_pll_create(*PLL_ARGS, _lib.LRB200_DEVICE), [CPX], [CPX, FLT],
                        base_lengths(*EW_UNITS, big=3000), _pll_input,
                        lambda xs: list(O.PLL(*PLL_ARGS).process(xs[0])), cmp_abs(2e-5)),
    # the chunk-parallel form (calls of 2 L and more; L = 50536 for these loop constants): ragged last chunks, the
    # sequential form below 2 L in between.  Against the oracle at the sequential case's 2e-5 plus the parallel form's
    # tolerance against the sequential one (tests/pll_ref.py)
    "pll_parallel": lambda: Case("lrb200_pll_create", _pll_parallel, [CPX], [CPX, FLT], PLL_PARALLEL_LENGTHS, _pll_input,
                                 lambda xs: list(O.PLL(*PLL_ARGS).process(xs[0])), _pll_parallel_cmp(), exact=True),
    **{"%s_%s" % ("agc" if agc else "powersquelch", "complex" if c else "real"): (lambda agc=agc, c=c: _level_case(agc, c))
       for agc in (True, False) for c in (False, True)},
    "phasecorrector_n50_i32": lambda: _phasecorr_case(50, 32),
    "phasecorrector_n4_i1": lambda: _phasecorr_case(4, 1),
    **{"iqconv_" + f: (lambda f=f: _source_case(f, True)) for f in RAW_WIDTH},
    **{"realconv_" + f: (lambda f=f: _source_case(f, False)) for f in RAW_WIDTH},
    **{"iqsink_" + f: (lambda f=f: _sink_case(f, True)) for f in RAW_WIDTH},
    **{"realsink_" + f: (lambda f=f: _sink_case(f, False)) for f in RAW_WIDTH},
}


# ---- graph-only fused stages through lrb200_graph_execute_device ----------------------------------------------------
WBFM_RATE = 1102500.0


def _graph(blocks_fn, in_port, out_port, lengths, gen, ref, describe, cmp=cmp_rel(1e-5)):
    def make(lib):
        g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
        for b in blocks_fn():
            _lib.check(lib.lrb200_graph_append(g, b.make_device_handle()), "append")
        _lib.check(lib.lrb200_graph_commit(g, 1), "commit")
        return g
    return Case("lrb200_graph_create", make, [in_port], [out_port], lengths, gen, ref, cmp, graph=True, describe=describe)


def _tuner_blocks(disc, rest=()):
    import luaradio_b200 as radio
    from luaradio_b200.types import ComplexFloat32, Float32
    from tests.test_gpu_stream import mk
    r1 = WBFM_RATE / 5
    blocks = [mk(radio.FrequencyTranslatorBlock, (-250e3,), ComplexFloat32, WBFM_RATE),
              mk(radio.LowpassFilterBlock, (128, 100e3), ComplexFloat32, WBFM_RATE),
              mk(radio.DownsamplerBlock, (5,), ComplexFloat32, WBFM_RATE)]
    if disc:
        blocks.append(mk(radio.FrequencyDiscriminatorBlock, (1.25,), ComplexFloat32, r1))
    if rest:
        blocks += [mk(radio.LowpassFilterBlock, (128, 15e3), Float32, r1), mk(radio.FMDeemphasisFilterBlock, (75e-6,), Float32, r1),
                   mk(radio.DownsamplerBlock, (5,), Float32, r1)]
    return blocks


def _fm(rng, n):
    return [O.synth_fm_iq(int(rng.integers(0, 1 << 20)), n)]


def _graph_reset_case(name, ref, lengths, gen):
    def blocks():
        from tests.test_gpu_stream import GRAPH_RESET_CASES
        return GRAPH_RESET_CASES[name][0]()
    in_port = FLT if name.startswith("fir*iir1") or name == "interpolator" else CPX
    out_port = FLT if in_port is FLT else CPX
    from_stream = {"fir*iir1_rrrf+pole": ")+pole", "fir*iir1_rrrf|pole_rrrf": " | pole_rrrf", "resampler": "upsample+fir+down(",
                   "interpolator": "upsample+fir(", "iir/D": "iir_crcf[fused x2]"}[name]
    return _graph(blocks, in_port, out_port, lengths, gen, ref, (None, from_stream))


def _audio_tail_ref(rate):
    return lambda xs: [O.Chain(O.lowpass_filter(128, 15e3, rate, False), O.IIRFilterFast(*O.fm_deemphasis_taps(75e-6, rate), False),
                               O.Downsampler(5)).process(xs[0])]


# the real polyphase stage (5, 27) with the pole: tiles of 2 * (PT_TO - 64) outputs, 5 inputs each
AUDIO_T = 2 * (PT_TO - 64) * 5

GRAPH_CASES = {
    "tuner+discrim": lambda: _graph(lambda: _tuner_blocks(True), CPX, FLT, tuner_lengths(True), _fm,
                                    lambda xs: [O.Chain(O.tuner(-250e3, 200e3, 5, WBFM_RATE), O.FrequencyDiscriminator(1.25)).process(xs[0])],
                                    ("tuner+discrim(128,/5)", None)),
    "tuner": lambda: _graph(lambda: _tuner_blocks(False), CPX, CPX, tuner_lengths(False), _fm,
                            lambda xs: [O.tuner(-250e3, 200e3, 5, WBFM_RATE).process(xs[0])], ("tuner(128,/5)", None)),
    "rot+fir_cccf": lambda: _graph(_rot_fir_blocks, CPX, CPX, base_lengths(1024 - 128 + 1), lambda rng, n: [rnd_c(rng, n)],
                                   lambda xs: [O.Chain(O.FrequencyTranslator(-250e3, WBFM_RATE),
                                                       O.complex_bandpass_filter(128, [-100e3, 100e3], WBFM_RATE),
                                                       O.Downsampler(5)).process(xs[0])], (None, "rot+fir_cccf")),
    "fir*iir1_rrrf+pole": lambda: _graph_reset_case("fir*iir1_rrrf+pole", _audio_tail_ref(1e5), base_lengths(AUDIO_T),
                                                    lambda rng, n: [rnd_f(rng, n)]),
    "fir*iir1_rrrf|pole_rrrf": lambda: _graph_reset_case("fir*iir1_rrrf|pole_rrrf", _audio_tail_ref(1e6), base_lengths(AUDIO_T),
                                                         lambda rng, n: [rnd_f(rng, n)]),
    "interpolator": lambda: _graph_reset_case("interpolator", lambda xs: [O.Chain(O.Upsampler(4), O.lowpass_filter(64, 1e5, 4e6, False)).process(xs[0])],
                                              base_lengths(IT_TILE), lambda rng, n: [rnd_f(rng, n)]),
    # rs_poly_kernel for (L, D) = (3, 2): RB = 4 periods per thread, 128 threads -> 1024 inputs per tile
    "resampler": lambda: _graph_reset_case("resampler", lambda xs: [O.Chain(O.Upsampler(3), O.lowpass_filter(64, 1e5, 3e6, True),
                                                                             O.Downsampler(2)).process(xs[0])],
                                           base_lengths(128 * 4 * 2), lambda rng, n: [rnd_c(rng, n)]),
    "iir/D": lambda: _graph_reset_case("iir/D", lambda xs: [O.Chain(O.IIRFilterFast(*O.singlepole_lowpass_taps(1e4, 1e6), True),
                                                                     O.Downsampler(4)).process(xs[0])],
                                       base_lengths(IIR_TILE, IIR_TILE + IIR_PAY), lambda rng, n: [rnd_c(rng, n)]),
    "wbfm_mono": lambda: _graph(lambda: _tuner_blocks(True, rest=True), CPX, FLT, tuner_lengths(True), _fm,
                                lambda xs: [O.wbfm_mono_chain().process(xs[0])], ("tuner+discrim(128,/5)[fused x4] | fir*iir1_rrrf(133,/5)+pole", None)),
}


def _rot_fir_blocks():
    import luaradio_b200 as radio
    from luaradio_b200.types import ComplexFloat32
    from tests.test_gpu_stream import mk
    return [mk(radio.FrequencyTranslatorBlock, (-250e3,), ComplexFloat32, WBFM_RATE),
            mk(radio.ComplexBandpassFilterBlock, (128, [-100e3, 100e3]), ComplexFloat32, WBFM_RATE),
            mk(radio.DownsamplerBlock, (5,), ComplexFloat32, WBFM_RATE)]


# Create entry points of include/lrb200.h that take no sample pointers of their own in this harness (checked on the CPU by
# tests/test_cpu_host.py::test_every_block_create_function_is_in_the_bounds_harness):
#   lrb200_dag_create -- lrb200_dag_execute is HOST in / HOST out only; its nodes are the blocks above, its edges
#                        library-owned device buffers.
BOUNDS_EXCLUDED_CREATE = {"lrb200_dag_create"}


def covered_create_functions():
    """The create entry points the case tables exercise (building a Case touches no GPU)."""
    return {make().create for table in (BLOCK_CASES, GRAPH_CASES) for make in table.values()}


# ---- the harness -------------------------------------------------------------------------------------------------------
class Guarded:
    """One lrb200_malloc allocation [GUARD | payload | GUARD]."""

    def __init__(self, lib, payload):
        self.lib, self.size = lib, 2 * GUARD + payload
        self.ptr = _lib.check_handle(lib.lrb200_malloc(self.size), "guarded buffer")

    def load(self, image):
        assert image.nbytes == self.size
        _lib.check(self.lib.lrb200_memcpy_h2d(self.ptr, image.ctypes.data, self.size), "h2d")

    def read(self):
        host = np.empty(self.size, np.uint8)
        _lib.check(self.lib.lrb200_memcpy_d2h(host.ctypes.data, self.ptr, self.size), "d2h")
        _lib.check(self.lib.lrb200_sync(), "sync")
        return host

    def free(self):
        self.lib.lrb200_free(self.ptr)


def _offset(port, aligned, k):
    """Byte offset of a stream inside its payload: 0 / 16 when aligned, else the natural alignment a or 16 - a."""
    if aligned:
        return 16 * (k % 2)
    return port.align if k % 2 == 0 else 16 - port.align


def _placements(nin, nout):
    """Aligned flags per port (inputs, then outputs): every input and the output(s) independently."""
    flags = [()]
    for _ in range(nin + 1):
        flags = [f + (a,) for f in flags for a in (True, False)]
    return [f[:nin] + (f[nin],) * nout for f in flags]


class Target:
    def __init__(self, lib, case):
        self.lib, self.case = lib, case
        self.h = _lib.check_handle(case.make(lib), "case")
        if case.graph:
            desc = lib.lrb200_graph_describe(self.h).decode()
            prefix, sub = case.describe
            assert prefix is None or desc.startswith(prefix), desc
            assert sub is None or sub in desc, desc

    def max_output(self, n):
        return (self.lib.lrb200_graph_max_output if self.case.graph else self.lib.lrb200_block_max_output)(self.h, n)

    def execute(self, xs, n, ys):
        no = ctypes.c_size_t()
        if self.case.graph:
            _lib.check(self.lib.lrb200_graph_execute_device(self.h, xs[0], n, ys[0], ctypes.byref(no)), "graph execute")
        else:
            xa = (ctypes.c_void_p * len(xs))(*xs)
            ya = (ctypes.c_void_p * len(ys))(*ys)
            _lib.check(self.lib.lrb200_block_execute_multi(self.h, xa, len(xs), n, ya, len(ys), ctypes.byref(no)), "execute")
        return no.value

    def reset(self):
        _lib.check((self.lib.lrb200_graph_reset if self.case.graph else self.lib.lrb200_block_reset)(self.h), "reset")

    def destroy(self):
        (self.lib.lrb200_graph_destroy if self.case.graph else self.lib.lrb200_block_destroy)(self.h)


def _calls(case, placements):
    """(n, placement) per call: every length in every placement, the placement changing from call to call."""
    calls, consumed = [], 0
    for spec in case.lengths:
        for p in placements:
            n = spec(consumed) if callable(spec) else spec
            calls.append((n, p))
            consumed += n
    return calls


def run_stream(lib, tgt, case, data, calls, run, aligned_only=False):
    """One pass over `calls` with poison / sentinel set `run` (0 = A, 1 = B); returns the output bytes per port."""
    nin = len(case.ins)
    maxn = max(n for n, _ in calls)
    maxo = max(tgt.max_output(n) for n, _ in calls)
    ibufs = [Guarded(lib, maxn * p.size + 32) for p in case.ins]
    obufs = [Guarded(lib, maxo * p.size + 32) for p in case.outs]
    sentinel = np.array([SENTINELS[run]], "<u4").view(np.uint8)
    oimages = [np.resize(sentinel, b.size) for b in obufs]
    iimages = [np.resize(p.poison(run), b.size) for p, b in zip(case.ins, ibufs)]
    outs = [[] for _ in case.outs]
    pos = 0
    try:
        for k, (n, place) in enumerate(calls):
            xs, ys, yoffs = [], [], []
            for i, (p, b) in enumerate(zip(case.ins, ibufs)):
                off = _offset(p, aligned_only or place[i], k)
                img = iimages[i].copy()
                img[GUARD + off:GUARD + off + n * p.size] = data[i][pos * p.size:(pos + n) * p.size]
                b.load(img)
                xs.append(b.ptr + GUARD + off)
            for o, (p, b) in enumerate(zip(case.outs, obufs)):
                off = _offset(p, aligned_only or place[nin + o], k)
                b.load(oimages[o])
                ys.append(b.ptr + GUARD + off)
                yoffs.append(off)
            no = tgt.execute(xs, n, ys)
            assert no <= tgt.max_output(n), "call %d (n=%d): n_out %d > max_output" % (k, n, no)
            for o, (p, b) in enumerate(zip(case.outs, obufs)):
                host = b.read()
                lo, hi = GUARD + yoffs[o], GUARD + yoffs[o] + no * p.size
                where = "call %d (n=%d, placement %s, output %d)" % (k, n, place, o)
                assert np.array_equal(host[:lo], oimages[o][:lo]), "%s: written before y: last stray byte at y%+d" % (
                    where, int(np.flatnonzero(host[:lo] != oimages[o][:lo])[-1]) - lo)
                assert np.array_equal(host[hi:], oimages[o][hi:]), "%s: written past y + n_out: first stray byte at y+n_out%+d" % (
                    where, int(np.flatnonzero(host[hi:] != oimages[o][hi:])[0]))
                outs[o].append(host[lo:hi])
            pos += n
    finally:
        for b in ibufs + obufs:
            b.free()
    return [np.concatenate(o) if o else np.zeros(0, np.uint8) for o in outs]


def check_case(case):
    lib = _lib.require_device()
    placements = _placements(len(case.ins), len(case.outs))
    calls = _calls(case, placements)
    total = sum(n for n, _ in calls)
    rng = np.random.default_rng(len(calls) * 7919 + total)
    inputs = case.gen(rng, total)
    data = [np.ascontiguousarray(x).view(np.uint8).reshape(-1) for x in inputs]
    tgt = Target(lib, case)
    try:
        a = run_stream(lib, tgt, case, data, calls, 0)
        tgt.reset()
        b = run_stream(lib, tgt, case, data, calls, 1)
        if case.exact:
            tgt.reset()
            aligned = run_stream(lib, tgt, case, data, calls, 0, aligned_only=True)
    finally:
        tgt.destroy()
    refs = case.ref(inputs, [n for n, _ in calls]) if case.ref_calls else case.ref(inputs)
    for o, p in enumerate(case.outs):
        got = p.view(a[o])
        if case.repeatable:
            first_diff = np.flatnonzero(a[o] != b[o])
            assert not first_diff.size, "output %d: poison / sentinel A and B runs differ first at byte %d of %d" % (
                o, int(first_diff[0]), a[o].size)
        else:
            # a stray read of pattern A is a NaN, of pattern B a value far off the reference
            assert p.kind != "raw" and len(b[o]) == len(a[o]), "output %d: length differs between runs" % o
            assert not np.isnan(p.view(b[o])).any(), "output %d: NaN in the pattern-B run" % o
            case.cmp(p.view(b[o]), np.asarray(refs[o]), "output %d, pattern-B run" % o)
        if p.kind != "raw":
            assert not np.isnan(got).any(), "output %d: NaN at sample %d" % (o, int(np.flatnonzero(np.isnan(got))[0]))
        if case.exact:
            d = np.flatnonzero(a[o] != aligned[o])
            assert not d.size, "output %d: unaligned placements differ from aligned ones first at sample %d" % (o, int(d[0]) // p.size)
        ref = np.asarray(refs[o])
        assert got.shape == ref.shape, "output %d: length %s != %s" % (o, got.shape, ref.shape)
        case.cmp(got, ref, "output %d" % o)


@pytest.mark.parametrize("name", list(BLOCK_CASES))
def test_block_bounds(name):
    check_case(BLOCK_CASES[name]())


@pytest.mark.parametrize("name", list(GRAPH_CASES))
def test_graph_stage_bounds(name):
    check_case(GRAPH_CASES[name]())
