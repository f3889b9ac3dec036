"""The overlap-save FIR kernels (fir_fft.cu: fir_fft1024_kernel in its complex, packed-real and Hilbert modes with the
fused translator and decimator, fir_fft_fdl_kernel for 514..8192 taps) and the direct kernels AUTO hands short calls
to, against float64 references with a per-output bound that scales with the output's own block (tests/fft_fir_ref.py).

A stream-wide tolerance is scaled to the loudest output, so a block that takes wrong samples, spectra or history while
the loud blocks look fine passes it.  Here every output is held to its own block's input norm, on bursty inputs that
step by 60 dB so that quiet blocks sit next to loud ones and quiet calls inherit loud histories; the mutants of
tests/fft_fir_ref.py (wrong block phasor, swapped packed lanes, dropped or shifted partitions, stale history, ...) exceed
the bound by 4x or more on every case's own input (tests/test_fft_fir_ref.py, on the CPU).

Each stream runs from lrb200_graph_seek(n0) through the C ABI with ragged lrb200_graph_execute_device calls.  Per call
the number of kernels launched must be the geometry model's, which pins the path and the work split the bound relies
on.  The stream runs again with its input one element further into the buffer (bitwise equal: these kernels have no
alignment-dependent path) and as one call (within the two runs' bounds of each other)."""
import numpy as np
import pytest

from luaradio_b200 import _lib
from tests import fft_fir_ref as F
from tests import test_gpu_fir_shapes as G

pytestmark = pytest.mark.gpu

DEV = _lib.LRB200_DEVICE
ALGO = {"auto": _lib.FIR_AUTO, "direct": _lib.FIR_DIRECT, "fft": _lib.FIR_FFT}
OS_M = (1, 2, 3, 31, 32, 33, 64, 65, 127, 128, 129, 255, 256, 257, 384, 511, 512, 513)
DEC_M = (33, 128, 513)
DEC_D = (2, 3, 5, 7, 25, 31, 32, 33, 64, 100, 1023, 1024, 1025, 4099)
ROT_M = (1, 33, 65, 129, 257, 513)
ROT_D = (1, 5, 33)
REAL_M = (1, 2, 33, 128, 257, 512, 513)
REAL_D = (1, 2, 5, 33)
HIL_M = (3, 9, 65, 129, 257, 511, 513)
FDL_M = (514, 1023, 1024, 1025, 1536, 2047, 2048, 2049, 2560, 4096, 4097, 6000, 8191, 8192)
SIGNALS = G.SIGNALS


def _taps(M, seed, cplx):
    return G.asym_taps(M, seed, cplx)


def _with_lead(calls, n0, D):
    """Decimating streams: before the long call, a call that ends where the next kept sample is the first input of the
    next call, so that the history reaches a kept output at any D."""
    if D == 1:
        return calls
    k = max(range(len(calls)), key=lambda i: calls[i])
    lead = -(n0 + sum(calls[:k])) % D
    return calls[:k] + ([lead] if lead else []) + [5] + calls[k:]


def _case(name, kind, h, D=1, turns=None, algo="fft", seeks=(0,), sig="noise", seed=0, calls=None):
    """One stage, one stream per seek; only the first carries the long call."""
    model = F.FirModel(kind, len(h), D, turns is not None, algo)
    streams = [(n0, _with_lead(list(calls) if calls else F.call_list(model, long_call=i == 0), n0, D))
               for i, n0 in enumerate(seeks)]
    return F.Case(name, kind, h, D, turns, algo, streams, sig, seed)


def _cases():
    cases = {}
    i = 0
    for kind in ("crcf", "cccf"):
        for M in OS_M:
            i += 1
            cases["os_%s_m%d" % (kind, M)] = lambda kind=kind, M=M, i=i: _case(
                "", kind, _taps(M, 100 + M, kind == "cccf"), seeks=(G.SEEKS[i % 8],), sig=SIGNALS[i % 3], seed=100 + M)
    for M in (128, 513):
        for k in (0, 1, M // 2, M - 2, M - 1):
            cases["os_crcf_m%d_impulse%d" % (M, k)] = lambda M=M, k=k: _case(
                "", "crcf", G.impulse(M, k), sig=SIGNALS[k % 3], seed=200 + k)
    for M in (129, 512):
        cases["os_crcf_m%d_alternating" % M] = lambda M=M: _case("", "crcf", G.alternating(M), sig="bursty", seed=300 + M)
    for kind in ("crcf", "cccf", "rrrf"):
        for M in DEC_M:
            for D in DEC_D:
                i += 1
                seeks = tuple(range(D)) if D <= 7 else (0, 1, D - 1, 2 ** 40 + 2)
                cases["dec_%s_m%d_d%d" % (kind, M, D)] = lambda kind=kind, M=M, D=D, i=i, seeks=seeks: _case(
                    "", kind, _taps(M, 400 + M + D, kind == "cccf"), D, seeks=seeks, sig=SIGNALS[i % 3], seed=400 + D)
    for kind in ("crcf", "cccf"):
        for M in ROT_M:
            for D in ROT_D:
                i += 1
                turns = G.OFFSETS[i % 8]
                # (the 1e-9-turn offset at a seek past 2^40, where its phase has run over a thousand turns and the
                # translator's direction shows)
                n0 = G.SEEKS[7] if abs(turns) < 1e-6 else G.SEEKS[(3 * i) % 8]
                cases["rot_%s_m%d_d%d" % (kind, M, D)] = lambda kind=kind, M=M, D=D, i=i, turns=turns, n0=n0: _case(
                    "", kind, _taps(M, 500 + M, kind == "cccf"), D, turns=turns, seeks=(n0,), sig=SIGNALS[i % 3],
                    seed=500 + M + D)
    for M in REAL_M:
        for D in REAL_D:
            i += 1
            cases["real_m%d_d%d" % (M, D)] = lambda M=M, D=D, i=i: _case(
                "", "rrrf", _taps(M, 600 + M, False), D, seeks=(G.SEEKS[i % 8] if D == 1 else i % D,),
                sig=SIGNALS[i % 3], seed=600 + M + D)
    for M in HIL_M:
        for algo in ("fft", "auto"):
            cases["hilbert_m%d_%s" % (M, algo)] = lambda M=M, algo=algo: _case(
                "", "hilbert", _taps(M, 700 + M, False), algo=algo, sig=SIGNALS[M % 3], seed=700 + M)
    for M in (515, 1025):
        cases["hilbert_m%d_catchall" % M] = lambda M=M: _case("", "hilbert", _taps(M, 700 + M, False), algo="auto",
                                                              sig="bursty", seed=700 + M)
    for kind in ("crcf", "cccf"):
        for M in FDL_M:
            i += 1
            cases["fdl_%s_m%d" % (kind, M)] = lambda kind=kind, M=M, i=i: _case(
                "", kind, _taps(M, 800 + M, kind == "cccf"), sig=SIGNALS[i % 3], seed=800 + M)
    for k in (511, 512, 513, 2047, 2048, 8191):
        cases["fdl_crcf_m8192_impulse%d" % k] = lambda k=k: _case("", "crcf", G.impulse(8192, k), sig="bursty", seed=900 + k)
    for kind in ("crcf", "cccf"):
        for M in (8193, 9000):
            cases["catchall_%s_m%d" % (kind, M)] = lambda kind=kind, M=M: _case(
                "", kind, _taps(M, 1000 + M, kind == "cccf"), algo="auto", sig="bursty", seed=1000 + M)
        cases["direct_%s_m257" % kind] = lambda kind=kind: _case(
            "", kind, _taps(257, 1257, kind == "cccf"), algo="direct", sig="bursty", seed=1257)
    for kind in ("crcf", "cccf", "rrrf"):
        for M in (514, 2000):
            for D in (2, 5):
                cases["direct_%s_m%d_d%d" % (kind, M, D)] = lambda kind=kind, M=M, D=D: _case(
                    "", kind, _taps(M, 1100 + M + D, kind == "cccf"), D, algo="auto", seeks=(0, D - 1), sig="bursty",
                    seed=1100 + M + D)
    for M in (128, 513, 2048):
        for kind in ("crcf", "cccf"):
            def auto(M=M, kind=kind):
                L = F.FirModel(kind, M).L
                calls = [8 * L - 1, 8 * L, 3, 8 * L + 1, 8 * L - 1, 2, 16 * L, 8 * L - 2, 8 * L + 5, 1000, 8 * L, 5]
                return _case("", kind, _taps(M, 1200 + M, kind == "cccf"), algo="auto", sig="bursty", seed=1200 + M,
                             calls=calls)
            cases["auto_%s_m%d" % (kind, M)] = auto
    return cases


CASES = _cases()


# ---- the harness ------------------------------------------------------------------------------------------------------
def blocks(lib, case):
    h = np.ascontiguousarray(case.h)
    M = case.M
    if case.kind == "hilbert":
        f = lib.lrb200_hilbert_create(h.ctypes.data, M, DEV)
    else:
        f = getattr(lib, "lrb200_fir_create_" + case.kind)(h.ctypes.data, M, 1, DEV)
    _lib.check(lib.lrb200_fir_set_algorithm(_lib.check_handle(f, "fir"), ALGO[case.algo]), "set_algorithm")
    hs = [lib.lrb200_rotator_create(case.turns, DEV)] if case.turns is not None else []
    hs.append(f)
    if case.D > 1:
        hs.append(lib.lrb200_downsample_create(case.D, 8 if case.cplx_out else 4, DEV))
    return hs


def describe(case):
    if case.turns is not None:
        return "rot+fir_%s[fused x%d]" % (case.kind, 3 if case.D > 1 else 2)
    name = "hilbert" if case.kind == "hilbert" else "fir_" + case.kind
    return name + ("[fused x2]" if case.D > 1 else "")


class _Stage:
    def __init__(self, case):
        self.blocks = lambda lib: blocks(lib, case)


def block_of(case, plans, calls, callno, g):
    """call-relative block of full-rate output g in the call that produced it (None for a direct kernel)"""
    start = int(np.sum(calls[:callno]))
    path = plans[callno][0]
    per = case.model.per if path == "fft" else (F.HOP if path == "fdl" else None)
    return (path, None if per is None else (int(g) - start) // per)


def check_stream(case, got, x, n0, calls, what):
    """Output count, NaN and the per-output bound; returns (bound, largest |got - ref| / bound)."""
    ref, bound, callno, full_idx = case.expect(x, n0, calls)
    assert got.shape == ref.shape, "%s: %d outputs, expected %d" % (what, len(got), len(ref))
    assert not np.isnan(got).any(), "%s: NaN at output %d" % (what, int(np.flatnonzero(np.isnan(got))[0]))
    d = np.abs(got.astype(np.complex128) - ref)
    ratio = np.where(bound > 0, d / np.where(bound > 0, bound, 1.0), np.where(d > 0, np.inf, 0.0))
    ex = float(np.max(ratio, initial=0.0))
    if ex > 1:
        i = int(np.argmax(ratio))
        plans = case.plans(n0, calls)
        path, blk = block_of(case, plans, calls, int(callno[i]), full_idx[i])
        raise AssertionError("%s: output %d of %d (call %d of length %d, %s block %s) off by %.3g, bound %.3g (%.1fx)" % (
            what, i, len(got), callno[i], calls[callno[i]], path, blk, d[i], bound[i], ex))
    return bound, ex


@pytest.mark.parametrize("name", list(CASES))
def test_fft_fir(name):
    lib = _lib.require_device()
    case = CASES[name]()
    g = G.Graph(lib, _Stage(case))
    try:
        assert g.desc == describe(case), g.desc
        worst = 0.0
        for n0, calls in case.streams:
            x = case.gen(sum(calls))
            what = "%s %s n0=%d" % (name, g.desc, n0)
            a = g.run(x, n0, calls, 0, case.cplx_out)
            want = [p[1] for p in case.plans(n0, calls)]
            assert g.launches == want, "%s: launches per call %s, the geometry model says %s (calls %s)" % (
                what, g.launches, want, calls)
            bound, ex = check_stream(case, a, x, n0, calls, what)
            worst = max(worst, ex)
            b = g.run(x, n0, calls, x.itemsize, case.cplx_out)
            assert g.launches == want, "%s: one element off: launches %s, expected %s" % (what, g.launches, want)
            diff = np.flatnonzero(a.view(np.uint32) != b.view(np.uint32))
            assert not diff.size, "%s: input one element further differs at output word %d" % (what, diff[0])
            c = g.run(x, n0, [len(x)], 0, case.cplx_out)
            bound1, ex1 = check_stream(case, c, x, n0, [len(x)], what + " one call")
            worst = max(worst, ex1)
            d = np.abs(a.astype(np.complex128) - c)
            assert np.all(d <= bound + bound1), "%s: ragged and one-call runs differ by %.3g at output %d" % (
                what, float(np.max(d - bound - bound1)), int(np.argmax(d - bound - bound1)))
        print("\n%s: largest |got - ref| / bound %.3g" % (name, worst))
    finally:
        g.destroy()
