"""The two-parallel fast-FIR form of the interior tuner+discriminator kernel (tuner.cu), checked on the CPU through its
numpy model (tests/tuner_ffa_model.py): exact in float64 against the direct form and the stream's FIR, and within the
discriminator's 1e-6 tolerance in float32."""
import os
import re

import numpy as np
import pytest

from oracle import lr_oracle as O
from tests import tuner_ffa_model as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "luaradio_b200", "csrc", "tuner.cu")).read()
RATE = 1102500.0


def test_model_and_kernel_agree_on_the_constants():
    assert int(re.search(r"#define LRB_PT_THREADS (\d+)", SRC).group(1)) == K.THREADS
    assert int(re.search(r"#define LRB_PT_R (\d+)", SRC).group(1)) == K.R
    assert int(re.search(r"constexpr int DISC_OV = (\d+);", SRC).group(1)) == K.DISC_OV
    assert int(re.search(r"constexpr int DISC_TAIL = (\d+);", SRC).group(1)) == K.DISC_TAIL
    assert "if (D == 5 && M > 65 && M <= 128) return 26;" in SRC
    assert "P.hs[q * D + p] = P.hr[2 * q * D + p] + P.hr[(2 * q + 1) * D + p]" in SRC


def _rotated(n):
    x = O.synth_fm_iq(0, n)
    i = np.arange(n, dtype=np.float64)
    return (x.astype(np.complex128) * np.exp(2j * np.pi * (-250e3 / RATE) * i)).astype(np.complex64)


def _taps():
    return O.f32_taps(O.firwin_lowpass(128, 100e3 / (RATE / 2)))


def _shaped_taps(kind, M):
    """Taps whose walking direction, padding and spare-tap alignment all show in the output (the low-pass is symmetric)."""
    if kind == "random":
        return np.random.default_rng(M).uniform(-1, 1, M).astype(np.float32)
    h = np.zeros(M, np.float32)
    h[{"impulse0": 0, "impulse_mid": M // 2 + 1, "impulse_last": M - 1}[kind]] = 1.0
    return h


FFA_CASES = [pytest.param(first, "lowpass", 128, id=str(first)) for first in (0, 1, 2, 4)] + [
    pytest.param(first, kind, M, id="%s-m%d-first%d" % (kind, M, first))
    for kind in ("random", "impulse0", "impulse_mid", "impulse_last") for M in (66, 67, 100, 127, 128)
    for first in range(5)]


@pytest.mark.parametrize("first,kind,M", FFA_CASES)
def test_fast_fir_equals_direct_form_float64(first, kind, M):
    """Both alignment shifts (spare tap leading or trailing) and every output slot of several tiles."""
    h = _taps() if kind == "lowpass" else _shaped_taps(kind, M)
    tiles = 6
    xr = _rotated(tiles * K.TS * K.D + 1000)
    got, ref = K.stream(xr, h, first, tiles, exact=True)
    tol = 1e-13 if kind == "lowpass" else 1e-13 * max(1.0, float(np.sum(np.abs(h))))
    assert np.max(np.abs(got - ref)) <= tol
    # the tiles lay out the stream's outputs y[m] = sum_k h[k] xr[first + m*D - k] (zero before the stream) in order
    xp = np.concatenate([np.zeros(M, np.complex128), xr.astype(np.complex128)])
    m = np.arange(len(ref))
    yref = sum(np.float64(h[k]) * xp[M + first + m * K.D - k] for k in range(M))
    assert np.max(np.abs(ref - yref)) <= tol


def test_fast_fir_discriminator_error_float32():
    """float32 sub-filter chains: the discriminator stays within the kernel's 1e-6 absolute tolerance of float64."""
    h = _taps()
    tiles = 160
    xr = _rotated(tiles * K.TS * K.D + 1000)
    got, ref = K.stream(xr, h, 0, tiles, exact=False)
    ex, _ = K.stream(xr, h, 0, tiles, exact=True)
    assert np.max(np.abs(got - ex)) <= 2e-6 * np.max(np.abs(ex))

    def disc(y):
        y = y.astype(np.complex128)
        return np.angle(y[1:] * np.conj(y[:-1])) / (2 * np.pi * 1.25)

    # the first 26 outputs are the filter's start-up transient (|y| ~ 1e-4), as in the kernel's own test
    err = np.abs(disc(got) - disc(ref))[26:]
    assert float(err.max()) <= 1e-6, float(err.max())
