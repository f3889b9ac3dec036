"""The POCSAG and AX.25 receivers' signal paths up to their data filters (examples/rtlsdr_pocsag.lua, rtlsdr_ax25.lua):
test signals, float64 oracle chains of both, the reference-executed golden vectors, and the float64 model and per-output bound of the fused FSK detector
(FskDetectBlock, fir_fft.cu overlap-save mode IN 4):

    y[o] = |(x * h_a)[o]| - |(x * h_b)[o]|        (h_a feeds Subtract's in1, h_b its in2)

Bound of an output o.  Each branch's complex FIR output carries either kernel's bound (tests/test_gpu_ert.py's stage
bound for complex data; u = 2^-24, W(o) = [o - L - (M - 1), o + L) the inputs of every block that can contain o):

    E(o) = C u ||x_W(o)||_2 ||H||_inf + 4 u |ref_o| + gamma_M sum_k |h_k| |x_(o-k)|

The magnitude |.| of a computed value v^ (cmag_of: one FMA over a rounded square, a correctly rounded square root) is
within MAG_REL |v^| of |v^| (tests/ert_ref.py), and ||v^| - |v|| <= |v^ - v|, so a branch's magnitude is within
E' = E + MAG_REL (|ref| + E).  The difference is one rounding: u |m_a^ - m_b^| <= u (|y_o| + E'_a + E'_b).  So

    |got_o - y_o| <= (1 + u) (E'_a + E'_b) + u |y_o|

tests/test_fsk_ref.py shows that a float32 emulation of the kernel stays within a quarter of it, and that the bound
catches swapped branches and a branch one sample late."""
import numpy as np

from luaradio_b200.utilities import filter_utils
from oracle import lr_oracle as O
from tests import ert_ref as E
from tests import fft_fir_ref as F

CAPTURE_RATE = 1e6
OFFSET = -100e3                 # the examples tune 100 kHz below the capture's centre
DECIM = 80
RATE = CAPTURE_RATE / DECIM     # 12.5 kS/s at the detector
MARK = (-5500.0, -3500.0)       # pocsagreceiver.lua:28-45: mark into Subtract's in1, space into in2
SPACE = (3500.0, 5500.0)
M = 129
# the golden vectors (tests/golden/make_fsk_golden.py): capture samples, seeds, ragged source vectors
GOLDEN_N = 48000                # 600 outputs: the interpreter runs about 100 capture samples per second
GOLDEN_SEED = {"pocsag": 51, "ax25": 52}


def golden_splits(n):
    """Ragged source vector bounds: an 8192-sample vector, one of 1 sample, one shorter than the ÷80 decimation, one of 20011,
    the rest."""
    return [0, 8192, 8193, 8193 + 77, 8193 + 77 + 20011, n]


def detector_taps():
    """(mark, space) complex band-pass taps as ComplexBandpassFilterBlock designs them at the detector's rate: the mark
    branch (-5.5..-3.5 kHz) feeds Subtract's in1, the space branch (+3.5..+5.5 kHz) its in2."""
    nyq = RATE / 2
    return tuple(np.asarray(filter_utils.firwin_complex_bandpass(M, [c / nyq for c in cut], "hamming"), np.complex64)
                 for cut in (MARK, SPACE))


def fsk_iq(n, seed, baud=1200.0, deviation=4.5e3, offset=-OFFSET, rate=CAPTURE_RATE, snr_db=25.0):
    """Continuous-phase binary FSK of random bits at `baud`, +-deviation around `offset` Hz, at `rate`, plus white noise."""
    rng = np.random.default_rng(seed)
    spb = rate / baud
    bits = rng.integers(0, 2, int(n / spb) + 2) * 2 - 1
    f = offset + deviation * bits[(np.arange(n) / spb).astype(np.int64)]
    ph = 2 * np.pi * np.cumsum(f) / rate
    noise = 10 ** (-snr_db / 20) / np.sqrt(2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return (0.5 * (np.exp(1j * ph) + noise)).astype(np.complex64)


def afsk_nbfm_iq(n, seed, baud=1200.0, offset=-OFFSET, rate=CAPTURE_RATE, deviation=3e3, snr_db=30.0):
    """Bell 202 AFSK (1200 Hz mark, 2200 Hz space, continuous phase) frequency-modulated at +-deviation, at offset Hz."""
    rng = np.random.default_rng(seed)
    spb = rate / baud
    bits = rng.integers(0, 2, int(n / spb) + 2)
    tone = np.where(bits[(np.arange(n) / spb).astype(np.int64)] == 1, 1200.0, 2200.0)
    audio = np.sin(2 * np.pi * np.cumsum(tone) / rate)
    ph = 2 * np.pi * np.cumsum(offset + deviation * audio) / rate
    noise = 10 ** (-snr_db / 20) / np.sqrt(2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return (0.5 * (np.exp(1j * ph) + noise)).astype(np.complex64)


def pocsag_oracle(x):
    """Tuner -> the detector -> LowpassFilter(128, 1200), float64 (oracle/lr_oracle.py blocks)."""
    t = O.tuner(OFFSET, 12e3, DECIM, CAPTURE_RATE).process(x)
    a, b = detector_taps()
    d = np.abs(O.FIRFilter(a, True).process(t)) - np.abs(O.FIRFilter(b, True).process(t))
    return O.lowpass_filter(128, 1200.0, RATE, False).process(d)


# AX.25 outputs compared from here on.  The chain starts from zero history, so the NBFM discriminator's input ramps up from
# nearly nothing: in its first ~30 samples its phase steps lie near +-pi, where any float32 difference between two correct
# implementations (the reference and the device, or fused and unfused device chains) flips the step's sign and moves the
# output by about 1.  The four filters behind it (128, 129, 128 and 128 taps) carry that into the first 1 + 127 + 128 +
# 127 + 127 + 1 outputs; from AX25_SETTLE on every output is a function of settled, well-conditioned samples only.
AX25_SETTLE = 520


def ax25_oracle(x):
    """Tuner -> NBFMDemodulator(3e3, 3e3) -> Hilbert(129) -> Translator(-1700) -> Lowpass(128, 750) ->
    Discriminator(1.25) -> Lowpass(128, 1200), float64 (examples/rtlsdr_ax25.lua)."""
    return O.Chain(O.tuner(OFFSET, 12e3, DECIM, CAPTURE_RATE),
                   O.lowpass_filter(128, 6e3, RATE, True), O.FrequencyDiscriminator(1.0),
                   O.lowpass_filter(128, 3e3, RATE, False), O.HilbertTransform(129),
                   O.FrequencyTranslator(-1700.0, RATE), O.lowpass_filter(128, 750.0, RATE, True),
                   O.FrequencyDiscriminator(1.25), O.lowpass_filter(128, 1200.0, RATE, False)).process(x)


def load_golden(name):
    """(capture, reference output, ragged source-vector bounds) of tests/golden/fsk/<name>_reference_executed.npz"""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fsk", name + "_reference_executed.npz"))
    return z["x"], z["y"], [int(v) for v in z["splits"]]


# ---- the fused detector -------------------------------------------------------------------------------------------------
def detector_ref(ha, hb, x):
    """float64 (branch a output, branch b output, |a| - |b|) over x from zero history."""
    ya = F.fir_ref(np.asarray(ha), np.asarray(x), wide=True)
    yb = F.fir_ref(np.asarray(hb), np.asarray(x), wide=True)
    return ya, yb, np.abs(ya) - np.abs(yb)


def _window_norm(ax, Mt, L):
    c = np.concatenate([[0.0], np.cumsum(np.asarray(ax, np.float64) ** 2)])
    o = np.arange(len(ax))
    lo, hi = np.clip(o - L - (Mt - 1), 0, len(ax)), np.clip(o + L, 0, len(ax))
    return np.sqrt(np.maximum(c[hi] - c[lo], 0.0))


def branch_bound(h, x, ref):
    """E(o) of the module docstring for one branch: either kernel FirBlock::path may run."""
    Mt = len(h)
    L = F.FF_N - (Mt - 1)
    ax = np.abs(np.asarray(x).astype(np.complex128))
    hn = F.spectrum_norms("cccf", h, 1)[0]
    direct = F.fir_ref(np.abs(np.asarray(h).astype(np.complex128)), ax, wide=True)
    return F.c_factor(1) * F.U * _window_norm(ax, Mt, L) * hn + 4 * F.U * np.abs(ref) + F.gamma(Mt) * direct


def detector_bound(ha, hb, x, ya=None, yb=None):
    """(reference, per-output bound) of the fused detector over x."""
    if ya is None:
        ya, yb, _ = detector_ref(ha, hb, x)
    y = np.abs(ya) - np.abs(yb)
    ea, eb = branch_bound(ha, x, ya), branch_bound(hb, x, yb)
    ea = ea + E.MAG_REL * (np.abs(ya) + ea)
    eb = eb + E.MAG_REL * (np.abs(yb) + eb)
    return y, (1 + F.U) * (ea + eb) + F.U * np.abs(y)
