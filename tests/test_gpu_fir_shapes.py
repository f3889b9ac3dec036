"""The register-tiled and fused FIR stages with asymmetric, impulse and alternating-sign taps over every instantiated
shape, against float64 references with per-output error bounds (tests/fir_shape_ref.py).

A symmetric low-pass cannot show which way a kernel walks its taps, and one tap count cannot show an error in the zero
padding or the spare-tap alignment of the others, so every case here uses taps whose reversal, shift or truncation
changes the output by far more than the bound (tests/test_fir_shape_ref.py checks that on the CPU, case by case).

Graphs are built through the C ABI (*_create(..., LRB200_DEVICE), lrb200_graph_append, commit(1)); describe() must name
the intended stage, so a fallback cannot pass silently.  Each stream runs from lrb200_graph_seek(n0) with ragged calls
through lrb200_graph_execute_device on lrb200_malloc buffers.  The tuner and real (5, 27) streams run twice: with a
16-byte aligned input (interior kernels, the fast-FIR form under the discriminator) and with the input 8 (real: 4)
bytes off (edge kernel only, direct form); the aligned run must have launched more kernels."""
import ctypes
import math

import numpy as np
import pytest

from luaradio_b200 import _lib
from oracle import lr_oracle as O
from tests import fir_shape_ref as R
from tests.test_gpu_bounds import tuner_exact

pytestmark = pytest.mark.gpu

DEV = _lib.LRB200_DEVICE
WBFM_RATE = 1102500.0
TUNER_T = 26 * 5                     # tuner.cu (5, 26): Q*D reversed taps (+1 alignment spare)
REAL_T = 27 * 5                      # tuner.cu real (5, 27)
GAINS = (0.3, 1.25, 7.0)
OFFSETS = (0.0, 0.5, -0.5, 0.2, -0.2, -250e3 / WBFM_RATE, 1e-9, (math.sqrt(5) - 1) / 7)
SEEKS = (0, 1, 2, 3, 4, 2 ** 31 - 3, 2 ** 32 + 1, 2 ** 40 + 2)
SIGNALS = ("fm", "noise", "bursty")
BURST = 64 * 8 * 5                   # one tuner tile of inputs: the bursty stream steps by 60 dB every tile
PG_TO = 128 * 8                      # poly_generic.cu outputs per tile
PG_DS = (2, 3, 4, 5, 6, 7, 8, 10, 12, 16, 20, 25)
RS_PAIRS = ((2, 1), (3, 1), (4, 1), (5, 1), (6, 1), (7, 1), (8, 1), (2, 3), (2, 5), (3, 2), (3, 4), (3, 5), (4, 3),
            (4, 5), (5, 2), (5, 3), (5, 4), (7, 5))


# ---- inputs and taps --------------------------------------------------------------------------------------------------
def signal(kind, n, seed, cplx=True):
    rng = np.random.default_rng(seed)
    if kind == "fm":
        x = O.synth_fm_iq(int(rng.integers(0, 1 << 30)), n, seed=seed % 1000 + 1)
    else:
        x = (rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n)) if cplx else rng.uniform(-1, 1, n)
        if kind == "bursty":
            x = x * np.where((np.arange(n) // BURST) % 2 == 0, 1.0, 1e-3)
    if not cplx:
        x = np.real(x)
    return x.astype(np.complex64 if cplx else np.float32)


def asym_taps(M, seed, cplx=False):
    """Random taps with heavy, unequal end taps, so that dropping or moving either end stands out of the bound (which
    grows with M ||h||_1) at every M."""
    rng = np.random.default_rng(seed)
    h = rng.uniform(-1, 1, M) + (1j * rng.uniform(-1, 1, M) if cplx else 0)
    if M > 1:
        h[-1], h[0] = 0.1 * M + 1, -0.05 * M - 1
    return (h / np.sum(np.abs(h))).astype(np.complex64 if cplx else np.float32)


def impulse(M, k, value=1.0):
    h = np.zeros(M, np.float32)
    h[k] = value
    return h


def alternating(M):
    """Alternating signs with a ramp in magnitude: neither symmetric nor a sign flip of its own reversal."""
    k = np.arange(M)
    return ((-1.0) ** k * (1 + k / M) / M).astype(np.float32)


def impulse_positions(M, seed):
    rng = np.random.default_rng(seed)
    ks = set(range(6)) | set(range(0, M, 5)) | {M - 2, M - 1} | set(int(k) for k in rng.integers(0, M, 3))
    return sorted(ks)


# ---- cases ------------------------------------------------------------------------------------------------------------
class Shape:
    """One graph and the streams run through it.  `blocks(lib)` returns the block handles to append; `describe` the
    (prefix, substring) describe() must show; `streams` a list of (n0, [call lengths]); `expect(x, n0)` the float64
    reference and its per-output bound (and the discriminator gain, or None); `mutants(x, n0)` the wrong references;
    `twice` runs the aligned / misaligned pair; `ulp` checks the outputs to one float32 ulp instead; `info` the taps and
    parameters (taps, turns, D, L, c, b, a) for the CPU emulations."""

    def __init__(self, name, blocks, describe, cplx_in, cplx_out, streams, gen, expect, mutants, twice=False, ulp=False,
                 **info):
        self.__dict__.update(info)
        self.name, self.blocks, self.describe = name, blocks, describe
        self.cplx_in, self.cplx_out, self.streams, self.gen = cplx_in, cplx_out, streams, gen
        self.expect, self.mutants, self.twice, self.ulp = expect, mutants, twice, ulp


def _resolve(calls, n0, disc):
    """Call lengths; ('exact', k, d) is a length at which the k-th interior tile ends on the call's input (+-1)."""
    out, consumed = [], n0
    for c in calls:
        n = tuner_exact(c[1], c[2], disc)(consumed) if isinstance(c, tuple) else c
        out.append(n)
        consumed += n
    return out


# 1-4-sample calls produce no output at D = 5 in most phases: the carried previous sample must survive them
TUNER_CALLS = [1, 2, 3, 4, ("exact", 1, -1), 3, ("exact", 1, 0), 1, 2, 4, ("exact", 1, 1), 4, 30011, 2, 4997]
BIG_CALLS = [3, 2 * 1024 * 1024 + 37, 4, 1001]


def _tuner_case(name, h, turns, gain, n0, sig, seed, calls=TUNER_CALLS, translator=True):
    M = len(h)
    disc = gain is not None
    G = 2 * np.pi * gain if disc else None

    def blocks(lib):
        hs = [lib.lrb200_rotator_create(turns, DEV)] if translator else []
        hs += [lib.lrb200_fir_create_crcf(h.ctypes.data, M, 1, DEV), lib.lrb200_downsample_create(5, 8, DEV)]
        if disc:
            hs.append(lib.lrb200_discrim_create(G, DEV))
        return hs

    tr = turns if translator else None
    if translator:
        desc = ("%s(%d,/5)" % ("tuner+discrim" if disc else "tuner", M), None) if 65 < M <= 128 else (None, "rot+fir_crcf")
    else:
        desc = ("fir_crcf[fused x2]", None)

    resolved = _resolve(calls, n0, disc)

    def expect(x, n0):
        y = R.tuner_ref(h, x, tr, 5, n0)
        if 65 < M <= 128:
            e = R.tuner_bound(h, x, 5, n0, TUNER_T)
        else:       # overlap-save (outside the tuner shape): bounded per block (tests/fft_fir_ref.py)
            from tests import fft_fir_ref
            e = fft_fir_ref.Case("", "crcf", h, 5, tr, "auto", [(n0, resolved)]).expect(x, n0, resolved)[1]
        return (R.discrim(y, G), R.disc_bound(y, e, G), G) if disc else (y, e, None)

    return Shape(name, blocks, desc, True, not disc, [(n0, resolved)],
                 lambda n: signal(sig, n, seed), expect,
                 lambda x, n0: R.tuner_mutants(h, x, tr, 5, n0, G), twice=65 < M <= 128, taps=h, turns=tr, D=5)


def _tuner_cases():
    cases = {}
    for i, M in enumerate(range(66, 129)):
        cases["tuner+discrim_m%d" % M] = lambda i=i, M=M: _tuner_case(
            "", asym_taps(M, M), OFFSETS[i % 8], GAINS[(i // 3) % 3], SEEKS[(i // 8) % 8], SIGNALS[i % 3], 1000 + M)
    for M in (66, 101, 128):
        for j, k in enumerate(impulse_positions(M, M)):
            cases["tuner+discrim_m%d_impulse%d" % (M, k)] = lambda M=M, j=j, k=k: _tuner_case(
                "", impulse(M, k), OFFSETS[(j + M) % 8], GAINS[j % 3], SEEKS[(j * 3) % 8], SIGNALS[j % 2], 2000 + k)
        cases["tuner+discrim_m%d_alternating" % M] = lambda M=M: _tuner_case(
            "", alternating(M), OFFSETS[7], 1.25, SEEKS[M % 8], "noise", 3000 + M)
    cases["tuner+discrim_m97_2Mi"] = lambda: _tuner_case("", asym_taps(97, 97), OFFSETS[5], 1.25, 2 ** 32 + 1, "fm", 4097,
                                                         calls=BIG_CALLS)
    cases["tuner+discrim_m128_2Mi_bursty"] = lambda: _tuner_case("", asym_taps(128, 7), OFFSETS[7], 7.0, 3, "bursty", 4128,
                                                                 calls=BIG_CALLS)
    tuner_offsets = (OFFSETS[5], 0.0, 0.5, 1e-9)
    for i, M in enumerate(range(66, 129)):
        cases["tuner_m%d" % M] = lambda i=i, M=M: _tuner_case(
            "", asym_taps(M, 5000 + M), tuner_offsets[i % 4], None, SEEKS[(i * 5) % 8], SIGNALS[i % 3], 5000 + M)
        cases["decim_crcf_m%d" % M] = lambda i=i, M=M: _tuner_case(
            "", asym_taps(M, 6000 + M), None, None, SEEKS[i % 8], SIGNALS[(i + 1) % 3], 6000 + M, translator=False)
    for M in (66, 101, 128):
        cases["tuner_m%d_impulse_last" % M] = lambda M=M: _tuner_case("", impulse(M, M - 1), OFFSETS[7], None, 2 ** 40 + 2,
                                                                     "noise", 7000 + M)
    # leaving the tuner shape: the overlap-save stage takes over
    for M in (65, 129):
        cases["rot+fir_m%d_discrim" % M] = lambda M=M: _tuner_case("", asym_taps(M, M), OFFSETS[5], 1.25, 2, "fm", 8000 + M)
        cases["rot+fir_m%d" % M] = lambda M=M: _tuner_case("", asym_taps(M, M + 1), OFFSETS[5], None, 2, "noise", 8100 + M)
    return cases


REAL_CALLS = [1, 2, 3, 4, 5119, 5120, 5121, 7, 10241, 30000]
AUDIO_T = 2 * (512 - 64) * 5
POLE_CALLS = [1, 2, 3, 4, AUDIO_T - 1, AUDIO_T, AUDIO_T + 1, 5, 2 * AUDIO_T + 1, 30000]


def _real_case(h, seed):
    M = len(h)

    def blocks(lib):
        return [lib.lrb200_fir_create_rrrf(h.ctypes.data, M, 1, DEV), lib.lrb200_downsample_create(5, 4, DEV)]

    return Shape("", blocks, ("fir_rrrf[fused x2]", None), False, False, [(0, REAL_CALLS)],
                 lambda n: signal("noise", n, seed, cplx=False),
                 lambda x, n0: (R.tuner_ref(h, x, None, 5, n0), R.tuner_bound(h, x, 5, n0, REAL_T), None),
                 lambda x, n0: R.tuner_mutants(h, x, None, 5, n0), twice=True, taps=h, D=5)


def _pole_case(h, taps, fused, seed):
    M = len(h)
    b, a = (np.asarray(t, np.float32) for t in taps)

    def blocks(lib):
        return [lib.lrb200_fir_create_rrrf(h.ctypes.data, M, 1, DEV),
                lib.lrb200_iir_create_rrrf(b.ctypes.data, len(b), a.ctypes.data, len(a), DEV),
                lib.lrb200_downsample_create(5, 4, DEV)]

    def expect(x, n0):
        z = R.pole_ref(h, b, a, x, 5, n0)
        return z, R.pole_bound(h, b, a, x, 5, z, REAL_T, n0), None

    desc = ("fir*iir1_rrrf(%d,/5)%s" % (M + len(b) + 3, "+pole" if fused else ""), None if fused else " | pole_rrrf")
    return Shape("", blocks, desc, False, False, [(0, POLE_CALLS)], lambda n: signal("noise", n, seed, cplx=False),
                 expect, lambda x, n0: R.pole_mutants(h, b, a, x, 5, n0), twice=True, taps=h, b=b, a=a)


def _real_cases():
    cases = {}
    for M in range(131, 136):
        cases["decim_rrrf_m%d" % M] = lambda M=M: _real_case(asym_taps(M, 9000 + M), 9000 + M)
        for k in (0, 1, 5, M // 2, M - 2, M - 1):
            cases["decim_rrrf_m%d_impulse%d" % (M, k)] = lambda M=M, k=k: _real_case(impulse(M, k), 9100 + k)
    for M in range(126, 131):
        for tname, taps_at in (("deemph", lambda r: O.fm_deemphasis_taps(75e-6, r)),
                               ("lowpass", lambda r: O.singlepole_lowpass_taps(3e3, r))):
            for fused, rate in ((True, 1e5), (False, 1e6)):
                cases["fir*%s_m%d_%s" % (tname, M, "pole" if fused else "split")] = (
                    lambda M=M, taps_at=taps_at, fused=fused, rate=rate: _pole_case(asym_taps(M, 9500 + M), taps_at(rate), fused, 9500 + M))
    return cases


def rs_rb(L, D):
    """resample.cu rs_rb: periods per thread of an instantiated (L, D), 0 otherwise."""
    if D == 1:
        return 8 if L == 2 else (4 if L <= 4 else (3 if L == 5 else (2 if L <= 8 else 0)))
    return {(2, 3): 4, (2, 5): 4, (3, 2): 4, (3, 4): 3, (3, 5): 3, (4, 3): 3, (4, 5): 3, (5, 2): 3, (5, 3): 3, (5, 4): 3,
            (7, 5): 2}.get((L, D), 0)


def rs_ok(L, D, M, elem):
    """InterpFirBlock::init: the register-tiled kernel takes (L, D, M) (resample.cu rs_geometry and its limits)."""
    RB = rs_rb(L, D)
    if not RB:
        return False
    RI = RB * D
    Tt = (-(-M // L) + 3) // 4 * 4
    HB = max(1, (Tt - 1 + RI - 1) // RI)
    H = HB * RI
    banks = 16 if elem == 8 else 32
    k = (banks + RI - 1) // RI
    ntp = HB + 128 + 1
    while ntp % banks != k % banks:
        ntp += 1
    smem = max(RI * ntp, 128 * ((RB * L) | 1)) * elem
    return Tt * L <= 896 and smem <= 48 * 1024 and H <= 128 and RI + Tt + 8 <= 168


def rs_max_taps(L, D, elem):
    return max(M for M in range(1, 1200) if rs_ok(L, D, M, elem))


def _rs_case(h, L, D, cplx, c, seed, ulp=False):
    M = len(h)
    elem = 8 if cplx else 4

    def blocks(lib):
        hs = [lib.lrb200_mulconst_create(c, 0.0, int(cplx), 0, DEV)] if c is not None else []
        hs.append(lib.lrb200_upsample_create(L, elem, DEV))
        hs.append(getattr(lib, "lrb200_fir_create_" + ("crcf" if cplx else "rrrf"))(h.ctypes.data, M, 1, DEV))
        if D > 1:
            hs.append(lib.lrb200_downsample_create(D, elem, DEV))
        return hs

    cc = 1.0 if c is None else c
    T = (-(-M // L) + 3) // 4 * 4
    RI = max(1, rs_rb(L, D)) * D
    calls = [1, 2, 3, 128 * RI - 1, 128 * RI, 128 * RI + 1, 5, 2 * 128 * RI + 1, 9000]
    desc = ("%supsample+fir%s(%d,x%d%s)" % ("mulconst+" if c is not None else "", "+down" if D > 1 else "", M, L,
                                             "/%d" % D if D > 1 else ""), None)
    return Shape("", blocks, desc, cplx, cplx, [(0, calls)], lambda n: signal("noise", n, seed, cplx),
                 lambda x, n0: (R.resample_ref(h, x, L, D, cc, direct=ulp), R.resample_bound(h, x, L, D, cc, T), None),
                 lambda x, n0: R.resample_mutants(h, x, L, D, cc), ulp=ulp, taps=h, L=L, D=D, c=cc)


def _rs_cases():
    cases = {}
    for L, D in RS_PAIRS:
        for cplx in (True, False):
            Mx = rs_max_taps(L, D, 8 if cplx else 4)
            for c in (None, -0.37):
                for M in (Mx, Mx + 1):
                    cases["rs_%dx%d_%s%s_m%d" % (L, D, "crcf" if cplx else "rrrf", "_scaled" if c else "", M)] = (
                        lambda L=L, D=D, cplx=cplx, c=c, M=M: _rs_case(asym_taps(M, 100 * L + D + M), L, D, cplx, c, M + L))
        Mx = rs_max_taps(L, D, 8)
        for k in sorted({0, 1, L - 1, L, Mx - 1}):
            cases["rs_%dx%d_impulse%d" % (L, D, k)] = lambda L=L, D=D, k=k, Mx=Mx: _rs_case(impulse(Mx, k), L, D, True, -0.37, k, ulp=True)
        cases["rs_%dx%d_m%d_below_L" % (L, D, L - 1)] = lambda L=L, D=D: _rs_case(asym_taps(L - 1, L * D), L, D, True, -0.37, L)
    cases["rs_160x147"] = lambda: _rs_case(asym_taps(301, 160147), 160, 147, True, -0.37, 147)
    return cases


def pg_supports(kind, M, D):
    """poly_generic.cu poly_generic_supports."""
    Qn = -(-M // D)
    if Qn * D * (2 if kind == "cccf" else 1) > 960:
        return False
    return (PG_TO + Qn + PG_TO // 8 + 4) * D * (4 if kind == "rrrf" else 8) <= 200 * 1024


def _pg_case(kind, D, M, seed):
    h = asym_taps(M, seed, cplx=kind == "cccf")
    cplx = kind != "rrrf"

    def blocks(lib):
        f = getattr(lib, "lrb200_fir_create_" + kind)(h.ctypes.data, M, 1, DEV)
        if f:
            _lib.check(lib.lrb200_fir_set_algorithm(f, _lib.FIR_DIRECT), "set_algorithm")
        return [f, lib.lrb200_downsample_create(D, 8 if cplx else 4, DEV)]

    T = -(-M // D) * D
    calls = [1, 2, PG_TO * D + 1, 3, 5000]
    return Shape("", blocks, ("fir_%s[fused x2]" % kind, None), cplx, cplx, [(n0, calls) for n0 in range(D)],
                 lambda n: signal("noise", n, seed, cplx),
                 lambda x, n0: (R.tuner_ref(h, x, None, D, n0), R.tuner_bound(h, x, D, n0, T), None),
                 lambda x, n0: R.tuner_mutants(h, x, None, D, n0), taps=h, D=D)


def _pg_cases():
    cases = {}
    for kind in ("crcf", "cccf", "rrrf"):
        for D in PG_DS:
            ms = [M for M in range(1, 1000) if pg_supports(kind, M, D)]
            if not ms:
                continue        # (crcf at D = 25: the tile does not fit; fir_generic_kernel runs)
            for M in (ms[-1], ms[-1] + 1):
                cases["pg_%s_d%d_m%d" % (kind, D, M)] = lambda kind=kind, D=D, M=M: _pg_case(kind, D, M, 31 * D + M)
    return cases


CASES = {**_tuner_cases(), **_real_cases(), **_rs_cases(), **_pg_cases()}


# ---- the harness ------------------------------------------------------------------------------------------------------
class Graph:
    def __init__(self, lib, shape):
        self.lib = lib
        self.g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
        for b in shape.blocks(lib):
            _lib.check(lib.lrb200_graph_append(self.g, _lib.check_handle(b, "block")), "append")
        _lib.check(lib.lrb200_graph_commit(self.g, 1), "commit")
        self.desc = lib.lrb200_graph_describe(self.g).decode()

    def run(self, x, n0, calls, in_off, cplx_out):
        """One stream from a reset graph at global index n0; x staged `in_off` bytes into a 256-byte aligned buffer."""
        lib = self.lib
        _lib.check(lib.lrb200_graph_reset(self.g), "reset")
        _lib.check(lib.lrb200_graph_seek(self.g, n0), "seek")
        isz, osz = x.itemsize, 8 if cplx_out else 4
        maxn = max(calls)
        xb = _lib.check_handle(lib.lrb200_malloc(maxn * isz + 64), "x")
        yb = _lib.check_handle(lib.lrb200_malloc(lib.lrb200_graph_max_output(self.g, maxn) * osz + 64), "y")
        outs, pos = [], 0
        self.launches = []             # kernels launched by each call
        try:
            for n in calls:
                chunk = np.ascontiguousarray(x[pos:pos + n])
                if n:
                    _lib.check(lib.lrb200_memcpy_h2d(xb + in_off, chunk.ctypes.data, n * isz), "h2d")
                no = ctypes.c_size_t()
                c0 = lib.lrb200_launch_count()
                _lib.check(lib.lrb200_graph_execute_device(self.g, xb + in_off, n, yb, ctypes.byref(no)), "execute")
                self.launches.append(lib.lrb200_launch_count() - c0)
                host = np.empty(no.value, np.complex64 if cplx_out else np.float32)
                if no.value:
                    _lib.check(lib.lrb200_memcpy_d2h(host.ctypes.data, yb, no.value * osz), "d2h")
                _lib.check(lib.lrb200_sync(), "sync")
                outs.append(host)
                pos += n
        finally:
            lib.lrb200_free(xb)
            lib.lrb200_free(yb)
        return np.concatenate(outs)

    def destroy(self):
        self.lib.lrb200_graph_destroy(self.g)


def check_output(shape, got, x, n0, what):
    ref, bound, gain = shape.expect(x, n0)
    assert got.shape == ref.shape, "%s: %d outputs, expected %d" % (what, len(got), len(ref))
    assert not np.isnan(got).any(), "%s: NaN at output %d" % (what, int(np.flatnonzero(np.isnan(got))[0]))
    if shape.ulp:
        ref32 = ref.astype(got.dtype)
        for part in ((np.real, np.imag) if np.iscomplexobj(got) else (np.real,)):
            g, r = part(got), part(ref32)
            bad = np.flatnonzero(np.abs(g - r) > np.spacing(np.abs(r)))
            assert not bad.size, "%s: output %d is %r, expected %r (1 ulp)" % (what, bad[0], got[bad[0]], ref32[bad[0]])
        return bound, gain
    ex = R.excess(got, ref, bound, gain)
    if ex > 1:
        n = len(got)
        d = R.wrapped((got - ref).real, gain) if gain else np.abs(got.astype(np.complex128) - ref)
        i = int(np.argmax(np.where(np.isfinite(bound), d / np.where(bound > 0, bound, 1e-300), 0)))
        raise AssertionError("%s: output %d of %d off by %.3g, bound %.3g (%.1fx)" % (what, i, n, d[i], bound[i], ex))
    return bound, gain


@pytest.mark.parametrize("name", list(CASES))
def test_fir_shape(name):
    lib = _lib.require_device()
    shape = CASES[name]()
    g = Graph(lib, shape)
    try:
        prefix, sub = shape.describe
        assert prefix is None or g.desc.startswith(prefix), g.desc
        assert sub is None or sub in g.desc, g.desc
        for n0, calls in shape.streams:
            x = shape.gen(sum(calls))
            c0 = lib.lrb200_launch_count()
            a = g.run(x, n0, calls, 0, shape.cplx_out)
            bound, gain = check_output(shape, a, x, n0, "%s n0=%d aligned" % (g.desc, n0))
            if shape.twice:
                c1 = lib.lrb200_launch_count()
                b = g.run(x, n0, calls, 8 if shape.cplx_in else 4, shape.cplx_out)
                c2 = lib.lrb200_launch_count()
                check_output(shape, b, x, n0, "%s n0=%d misaligned" % (g.desc, n0))
                assert c1 - c0 > c2 - c1, "the aligned run launched no interior kernel (%d vs %d launches)" % (c1 - c0, c2 - c1)
                assert R.excess(a, b, 2 * bound, gain) <= 1, "aligned and misaligned runs differ beyond their bounds"
    finally:
        g.destroy()
