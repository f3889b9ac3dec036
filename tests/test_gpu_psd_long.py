"""spectrum_utils.PSD on frames of 8192 <= N <= 2^20 points (psd_long.cu) against oracle.psd, bin by bin within the
bound of tests/psd_long_ref.py:

  * every power of two in that range, complex and real input, linear and logarithmic, 1, 2 and 37 frames per call;
  * the frames cycle through a strong tone next to one 60 dB weaker, white noise and an all-zero frame;
  * one call of 2^26 samples at N = 2^20, which runs the two-pass form in two scratch batches;
  * the guard-band harness of tests/test_gpu_bounds.py in DEVICE mode at aligned and unaligned offsets;
  * the frame lengths the block still refuses."""
import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from oracle import lr_oracle as O
from tests import psd_long_ref as M
from tests.test_gpu_bounds import CPX, FLT, Case, check_case

pytestmark = pytest.mark.gpu

RATE = 1e6


def frames_input(N, frames, cplx, seed):
    """Frame i: tones (i % 3 == 0), noise (1) or zeros (2)."""
    rng = np.random.default_rng(seed)
    t = np.arange(N)
    out = []
    for i in range(frames):
        kind = i % 3
        if kind == 0:
            k0 = 0.1234 * N + 0.37 * i
            x = np.exp(2j * np.pi * k0 * t / N) + 1e-3 * np.exp(2j * np.pi * (k0 + 7.5) * t / N)
        elif kind == 1:
            x = rng.standard_normal(N) + 1j * rng.standard_normal(N)
        else:
            x = np.zeros(N, np.complex128)
        out.append(x if cplx else x.real)
    x = np.concatenate(out)
    return x.astype(np.complex64) if cplx else x.astype(np.float32)


def oracle(x, N, logarithmic):
    return np.concatenate([O.psd(x[i:i + N], "hamming", RATE, logarithmic) for i in range(0, len(x), N)])


def check_psd(N, x, cplx, what):
    lin = radio.spectrum_utils.PSD(N, cplx, "hamming", RATE, False)
    log = radio.spectrum_utils.PSD(N, cplx, "hamming", RATE, True)
    scale = RATE * lin.window_energy
    ref_lin = oracle(x, N, False)
    M.check(lin.compute(x), x, lin.window, scale, ref_lin, what=what + " linear")
    M.check(log.compute(x), x, log.window, scale, ref_lin, oracle(x, N, True), logarithmic=True, what=what + " log")
    lin.close()
    log.close()


@pytest.mark.parametrize("frames", [1, 2, 37])
@pytest.mark.parametrize("cplx", [True, False], ids=["complex", "real"])
@pytest.mark.parametrize("N", M.LONG_SIZES)
def test_psd_long_frames(N, cplx, frames):
    x = frames_input(N, frames, cplx, seed=N + frames)
    check_psd(N, x, cplx, "N=%d %s frames=%d" % (N, "complex" if cplx else "real", frames))


def test_psd_long_call_crosses_the_scratch_batch():
    N = 1 << 20
    frames = (1 << 26) // N
    assert frames > M.batch_frames(N)
    x = frames_input(N, frames, True, seed=26)
    psd = radio.spectrum_utils.PSD(N, True, "hamming", RATE, False)
    got = psd.compute(x)
    psd.close()
    M.check(got, x, psd.window, RATE * psd.window_energy, oracle(x, N, False), what="2^26 samples")


def test_psd_frame_length_limits():
    for N in (1 << 21, 3 << 12, 1000):
        with pytest.raises(radio._lib.LibraryError, match="2..1048576"):
            radio.spectrum_utils.PSD(N, True)


def _bounds_case(N):
    win = np.array(O.window(N, "hamming", True), np.float32)
    scale = RATE * float(np.sum(win.astype(np.float64) ** 2))
    seen = {}

    def ref(xs):
        seen["x"] = xs[0]
        return [oracle(xs[0], N, False) if len(xs[0]) else np.zeros(0, np.float32)]

    def cmp(got, r, what):
        M.check(got, seen["x"], win, scale, r, what=what)
    return Case("lrb200_psd_create", lambda lib: lib.lrb200_psd_create(N, win.ctypes.data, scale, 0, 1, _lib.LRB200_DEVICE),
                [CPX], [FLT], [0, N, 2 * N, 3 * N], lambda rng, n: [frames_input(N, n // N, True, seed=n)], ref, cmp, exact=True)


@pytest.mark.parametrize("N", [8192, 32768, 1 << 18, 1 << 20])
def test_psd_long_bounds(N):
    check_case(_bounds_case(N))
