"""Reference model of BinaryPhaseCorrectorBlock and RootRaisedCosineFilterBlock's taps, and the RDS signal path of
examples/rtlsdr_rds.lua built from them and the oracle package.

BinaryPhaseCorrector restates binaryphasecorrector.lua:43-77 with the window kept as a ring indexed by measurement number
mod N (the reference shifts it with memmove; the values are the same).  The average is the reference's recurrence
avg = (avg + phi/N) - last/N taken term for term: np.cumsum over the interleaved terms [+phi_0/N, -last_0/N, +phi_1/N, ...]
is a sequential sum, so it reproduces the reference's doubles bit for bit."""
import math

import numpy as np

from oracle import lr_oracle as O


def fir_root_raised_cosine(num_taps, sample_rate, beta, symbol_period):
    """filter_utils.lua:301-337 in float64, normalised to unity DC gain."""
    if num_taps % 2 == 0:
        raise ValueError("Number of taps must be odd.")
    h = np.empty(num_taps)
    edge = (beta / math.sqrt(2 * symbol_period)) * ((1 + 2 / math.pi) * math.sin(math.pi / (4 * beta))
                                                    + (1 - 2 / math.pi) * math.cos(math.pi / (4 * beta)))
    for n in range(num_taps):
        t = (n - (num_taps - 1) / 2) / sample_rate
        if t == 0:
            h[n] = (1 / math.sqrt(symbol_period)) * (1 - beta + 4 * beta / math.pi)
        elif abs(t + symbol_period / (4 * beta)) < 1e-5 or abs(t - symbol_period / (4 * beta)) < 1e-5:
            h[n] = edge
        else:
            num = math.cos((1 + beta) * math.pi * t / symbol_period) + math.sin((1 - beta) * math.pi * t / symbol_period) / (4 * beta * t / symbol_period)
            denom = 1 - (4 * beta * t / symbol_period) * (4 * beta * t / symbol_period)
            h[n] = ((4 * beta) / (math.pi * math.sqrt(symbol_period))) * num / denom
    scale = 0.0
    for v in h:                    # the reference's sequential sum
        scale += v
    return h / scale


def _fold(a32):
    """ComplexFloat32:arg() (atan2f) as a Lua number, folded into (-pi/2, pi/2] (binaryphasecorrector.lua:49-51)."""
    phi = a32.astype(np.float64)
    phi = np.where(phi < -math.pi / 2, phi + math.pi, phi)
    return np.where(phi > math.pi / 2, phi - math.pi, phi)


class BinaryPhaseCorrector:
    """binaryphasecorrector.lua:28-77, stateful across process() calls."""

    def __init__(self, num_samples, sample_interval=None):
        self.N = int(num_samples)
        self.I = 32 if sample_interval is None else int(sample_interval)
        self.reset()

    def reset(self):
        self.window = np.zeros(self.N, np.float32)     # slot k mod N: float32 phi of measurement k
        self.average = 0.0
        self.measurements = 0                          # global number of the next measurement
        self.consumed = 0

    def process(self, x):
        x = np.asarray(x, np.complex64)
        N, I, n = self.N, self.I, len(x)
        pos = np.arange((-self.consumed) % I, n, I)   # measurements at global indices k*I
        K = len(pos)
        a = np.arctan2(x.imag[pos], x.real[pos], dtype=np.float32)
        phi = _fold(a)
        phi32 = phi.astype(np.float32)
        k = self.measurements + np.arange(K, dtype=np.int64)
        j = np.arange(K)
        last = np.where(j < N, self.window[k % N], phi32[np.maximum(j - N, 0)])
        terms = np.empty(2 * K + 1)
        terms[0] = self.average
        terms[1::2] = phi / N
        terms[2::2] = -(last.astype(np.float64) / N)
        avgs = np.cumsum(terms)[0::2]                  # avgs[m] = average after m of this call's measurements
        which = np.searchsorted(pos, np.arange(n), side="right")
        avg = avgs[which]
        pr, pi = np.cos(-avg).astype(np.float32), np.sin(-avg).astype(np.float32)
        xr, xi = x.real.astype(np.float64), x.imag.astype(np.float64)
        pr, pi = pr.astype(np.float64), pi.astype(np.float64)
        y = np.empty(n, np.complex64)
        y.real = (xr * pr - xi * pi).astype(np.float32)
        y.imag = (xr * pi + xi * pr).astype(np.float32)
        m = min(K, N)
        if m:
            self.window[k[K - m:] % N] = phi32[K - m:]
        self.average = float(avgs[-1])
        self.measurements += K
        self.consumed += n
        return y


def rrc_filter(num_taps, beta, symbol_rate, rate, complex_input):
    """RootRaisedCosineFilterBlock(num_taps, beta, symbol_rate) at `rate`: an FIR with float32-rounded taps."""
    return O.FIRFilter(O.f32_taps(fir_root_raised_cosine(num_taps, rate, beta, 1 / symbol_rate)), complex_input)


class RDSPath:
    """examples/rtlsdr_rds.lua:13-24,38-43 from the FrequencyDiscriminatorBlock to the ComplexToRealBlock at `rate`
    (220.5 kHz: the source's 1.1025 MS/s after TunerBlock(-250e3, 200e3, 5)).  process() returns the RRC output (the
    example's spectrum tap), the phase corrector's output and its ComplexToReal."""

    def __init__(self, rate=220500.0):
        self.disc = O.FrequencyDiscriminator(1.25)
        self.hilbert = O.HilbertTransform(129)
        self.delay = O.Delay(129)
        self.pilot = O.complex_bandpass_filter(129, [18e3, 20e3], rate)
        self.pll = O.PLL(1500.0, 19e3 - 100, 19e3 + 100, 3.0, rate)
        self.lowpass = O.lowpass_filter(128, 4e3, rate, True)
        self.rrc = rrc_filter(101, 1, 1187.5, rate, True)
        self.bpc = BinaryPhaseCorrector(8000)

    def process(self, x):
        h = self.hilbert.process(self.disc.process(x))
        d = self.delay.process(h)
        p, _ = self.pll.process(self.pilot.process(h))
        r = self.rrc.process(self.lowpass.process(O.binary_op("multiplyconjugate", d, p)))
        b = self.bpc.process(r)
        return r, b, O.complex_to_real(b)


class BPSK31FrontEnd:
    """composites/bpsk31receiver.lua:27-37 up to its clock recoverer: Lowpass(128, 100) -> RRC(101, 1, 31.25) ->
    BinaryPhaseCorrector(50) -> ComplexToReal.  process() returns the phase corrector's output and its ComplexToReal."""

    def __init__(self, rate):
        self.lowpass = O.lowpass_filter(128, 100, rate, True)
        self.rrc = rrc_filter(101, 1, 31.25, rate, True)
        self.bpc = BinaryPhaseCorrector(50)

    def process(self, x):
        b = self.bpc.process(self.rrc.process(self.lowpass.process(x)))
        return b, O.complex_to_real(b)
