"""CPU checks of tests/psd_long_ref.py, the float32 model of the long-frame PSD kernels (psd_long.cu): its geometry, its
agreement with oracle.psd within the per-bin bound at every N, and that the bound is tight enough to catch a wrong
twiddle sign, a mistransposed row tile, a window missing on one tile and a wrong scale."""
import numpy as np
import pytest

from oracle import lr_oracle as O
from tests import psd_long_ref as M

RATE = 2.0


def _signal(N, frames, cplx, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(frames * N)
    tone = np.exp(2j * np.pi * 0.2031 * t) + 1e-3 * np.exp(2j * np.pi * (0.2031 + 5.5 / N) * t)
    x = 0.5 * tone + 0.1 * (rng.standard_normal(frames * N) + 1j * rng.standard_normal(frames * N))
    return x.astype(np.complex64) if cplx else x.real.astype(np.float32)


def _setup(N, frames, cplx, seed=1):
    x = _signal(N, frames, cplx, seed + N)
    w = np.array(O.window(N, "hamming", True), np.float32)
    scale = RATE * float(np.sum(w.astype(np.float64) ** 2))
    ref = np.concatenate([O.psd(x[i:i + N], "hamming", RATE, False) for i in range(0, len(x), N)])
    return x, w, scale, ref


def test_geometry():
    for N in M.LONG_SIZES:
        if N <= M.SINGLE_MAX:
            assert int(np.prod(M.radices(N))) == N
            continue
        N1, N2 = M.split(N)
        assert N1 * N2 == N and N1 <= N2 <= 1024
        for L in (N1, N2):
            assert int(np.prod(M.radices(L))) == L and M.TILE % L == 0
        # a column tile spans whole columns, a row tile whole rows, and every k1 n2 twiddle exponent is in the tables
        assert N2 % (M.TILE // N1) == 0 and N1 % (M.TILE // N2) == 0
        assert (N1 - 1) * (N2 - 1) < N and N // 1024 >= 1
        assert M.batch_frames(N) * N * 8 <= 256 << 20


@pytest.mark.parametrize("cplx", [True, False], ids=["complex", "real"])
@pytest.mark.parametrize("N", M.LONG_SIZES)
def test_model_within_bound(N, cplx):
    frames = 2 if N <= 1 << 17 else 1
    x, w, scale, ref = _setup(N, frames, cplx)
    # half of C_BOUND already holds: the kernels' radix-2 butterflies may round differently from the model's DFT matrices
    M.check(M.model_psd(x, w, scale, False), x, w, scale, ref, c=M.C_BOUND / 2, what="N=%d" % N)
    ref_log = np.concatenate([O.psd(x[i:i + N], "hamming", RATE, True) for i in range(0, len(x), N)])
    M.check(M.model_psd(x, w, scale, True), x, w, scale, ref, ref_log, logarithmic=True, what="N=%d log" % N)


def test_model_batches():
    """A call longer than one scratch batch is cut into batches; the batches see the same arithmetic."""
    N = 1 << 15
    saved = M.BATCH_SAMPLES
    x, w, scale, ref = _setup(N, 5, True)
    whole = M.model_psd(x, w, scale, False)
    try:
        M.BATCH_SAMPLES = 2 * N
        cut = M.model_psd(x, w, scale, False)
    finally:
        M.BATCH_SAMPLES = saved
    assert np.array_equal(whole, cut)
    M.check(cut, x, w, scale, ref)


@pytest.mark.parametrize("mutant", ["twiddle_sign", "transpose", "window", "scale"])
@pytest.mark.parametrize("N", [8192, 16384, 1 << 15, 1 << 18, 1 << 20])
def test_mutants_break_the_bound(N, mutant):
    if mutant == "transpose" and N <= M.SINGLE_MAX:
        pytest.skip("the one-CTA form has no transposed store")
    x, w, scale, ref = _setup(N, 1, True)
    got = M.model_psd(x, w, scale, False, mutant=mutant)
    with pytest.raises(AssertionError):
        M.check(got, x, w, scale, ref)


def test_zero_frame_is_exact():
    N = 8192
    w = np.array(O.window(N, "hamming", True), np.float32)
    x = np.zeros(N, np.complex64)
    ref = O.psd(x, "hamming", RATE, False)
    M.check(M.model_psd(x, w, 1.0, False), x, w, 1.0, ref)
    got = M.model_psd(x, w, 1.0, True)
    M.check(got, x, w, 1.0, ref, O.psd(x, "hamming", RATE, True), logarithmic=True)
    assert np.all(got == -np.inf)
