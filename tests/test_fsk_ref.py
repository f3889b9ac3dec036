"""The fused FSK detector's model and bound (tests/fsk_ref.py), on the CPU:

  * a float32 emulation of the kernel's arithmetic (fir_fft.cu mode IN 4: each branch is the cccf overlap-save path of
    tests/test_fft_fir_ref.py's emulation, then cmag_of and one subtraction) stays within a quarter of the bound, on a
    call with edge and interior blocks and on one shorter than a block;
  * mutants the bound must catch, each beyond four times it: the branches swapped (space - mark), and one branch's
    input history off by one sample;
  * the POCSAG oracle chain separates the two tones: the detector's sign follows the transmitted bits;
  * both oracle chains against the reference's own output of the example graphs (tests/golden/fsk/)."""
import numpy as np
import pytest

from tests import fft_fir_ref as F
from tests import fsk_ref as K
from tests.test_fft_fir_ref import _cmul, _forward, _gather, _inverse, _spectrum

F32 = np.float32


def _branch(h, x):
    """One branch's complex outputs of a call over all of x, from zero history, as the overlap-save kernel computes them."""
    Mt, n = len(h), len(x)
    L = F.FF_N - (Mt - 1)
    b = np.arange(-(-n // L))
    t = np.arange(F.FF_N)
    v = _gather(x, b[:, None] * L - (Mt - 1) + t[None], 0, n)
    Xr, Xi = _forward(v.real.astype(F32), v.imag.astype(F32))
    Hr, Hi = _spectrum(h)
    yr, yi = _inverse(*_cmul(Xr, Xi, Hr[None], Hi[None]))
    out = np.zeros(n, np.complex64)
    o = b[:, None] * L - (Mt - 1) + t[None]
    ok = (t[None] >= Mt - 1) & (o < n)
    out[o[ok]] = (yr + 1j * yi)[ok]
    return out


def _cmag(v):
    """common.cuh cmag_of: sqrt(fma(re, re, fl(im * im))), correctly rounded"""
    re, im = v.real.astype(np.float64), v.imag.astype(np.float64)
    return np.sqrt((re * re + (im * im).astype(F32)).astype(F32))


def emulate(ha, hb, x):
    return (_cmag(_branch(ha, x)).astype(np.float64) - _cmag(_branch(hb, x))).astype(F32)


def _signal(n, seed):
    """The detector's input: the FSK at baseband, 12.5 kS/s"""
    return K.fsk_iq(n, seed, offset=0.0, rate=K.RATE)


def excess(got, ref, bound):
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / bound))


@pytest.mark.parametrize("n", [20000, 700])
def test_float32_emulation_stays_within_a_quarter_of_the_bound(n):
    ha, hb = K.detector_taps()
    x = _signal(n, 5)
    ref, bound = K.detector_bound(ha, hb, x)
    ex = excess(emulate(ha, hb, x), ref, bound)
    print("\nn = %d: float32 emulation at %.3g of the bound" % (n, ex))
    assert ex < 0.25


def test_arbitrary_taps_not_mirrored():
    rng = np.random.default_rng(7)
    ha = (rng.standard_normal(65) + 1j * rng.standard_normal(65)).astype(np.complex64) / 8
    hb = (rng.standard_normal(65) + 1j * rng.standard_normal(65)).astype(np.complex64) / 8
    x = _signal(6000, 8)
    ref, bound = K.detector_bound(ha, hb, x)
    assert excess(emulate(ha, hb, x), ref, bound) < 0.25


def test_mutants_exceed_four_times_the_bound():
    ha, hb = K.detector_taps()
    x = _signal(20000, 9)
    ref, bound = K.detector_bound(ha, hb, x)
    swapped = emulate(hb, ha, x)
    late = (_cmag(_branch(ha, x)).astype(np.float64) - _cmag(_branch(hb, np.concatenate([[0], x[:-1]]).astype(np.complex64))))
    for name, got in (("branches swapped", swapped), ("history off by one", late)):
        ex = excess(got, ref, bound)
        print("\n%s: %.3g of the bound" % (name, ex))
        assert ex > 4.0, name


def test_pocsag_oracle_follows_the_bits():
    """Mark (-4.5 kHz) into in1: the detector output after the data filter is positive on mark bits, 128 outputs (the
    two 129/128-tap filters' group delays) after them."""
    n = 1 << 18
    rng_bits = np.random.default_rng(3)
    x = K.fsk_iq(n, 3)
    y = K.pocsag_oracle(x)
    spb = K.CAPTURE_RATE / 1200.0
    bits = rng_bits.integers(0, 2, int(n / spb) + 2) * 2 - 1
    y = y[128:]
    centre = ((np.arange(len(y)) * K.DECIM) / spb).astype(np.int64)
    mid = ((np.arange(len(y)) * K.DECIM) % spb) / spb
    sel = (mid > 0.3) & (mid < 0.7) & (np.arange(len(y)) > 200)
    agree = np.mean(np.sign(y[sel]) == -bits[centre[sel]])
    assert agree > 0.95, agree


@pytest.mark.parametrize("name", ["pocsag", "ax25"])
def test_oracle_wiring_matches_the_reference_golden(name):
    """The float64 oracle chains (tests/fsk_ref.py) reproduce the reference's own output of the example graphs
    (tests/golden/fsk/, tests/golden/make_fsk_golden.py) at the tuner goldens' 1e-5 (DESIGN.md §1)."""
    x, y, _ = K.load_golden(name)
    got = (K.pocsag_oracle if name == "pocsag" else K.ax25_oracle)(x)
    scale = max(1.0, float(np.max(np.abs(y))))
    assert len(got) == len(y) and np.max(np.abs(y)) > 1e-3
    err = float(np.max(np.abs(got - y)))
    print("\n%s: oracle against the reference %.3g (scale %.3g)" % (name, err, scale))
    assert err <= 1e-5 * scale
