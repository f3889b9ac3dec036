"""Reference model of AGCBlock and PowerSquelchBlock (radio/blocks/signal/agc.lua, powersquelch.lua) for the tests.

The definition is `process_loop`: the reference's per-sample loop in its operation order, in Python floats (IEEE double,
like Lua numbers), with the power and gain state carried across calls.  `process` is the same arithmetic vectorised:

    P = lfilter([pa], [1, -(1-pa)], |x|^2)                   (zi carries (1-pa) P_prev)
    g = lfilter([ga], [1, -(1-ga)], T * (1/P[P >= theta]))   (on the gated subsequence; zi carries (1-ga) g_prev)

forward-filled over the closed samples.  For a first-order section lfilter's transposed direct form evaluates
(1-a) y[n-1] + b x[n] with the same two products and one sum as the reference, so the two forms agree bit for bit; the
tests check that on long streams with many gate flips."""
import math

import numpy as np
import scipy.signal


def _power(x):
    """|x|^2 in double: re*re + im*im of the float32 components (complexfloat32.lua:174), x*x for Float32."""
    if np.iscomplexobj(x):
        re = x.real.astype(np.float64)
        im = x.imag.astype(np.float64)
        return re * re + im * im
    v = np.asarray(x).astype(np.float64)
    return v * v


def _scale(x, s):
    """float32(s * x) per component, the product in double."""
    if np.iscomplexobj(x):
        y = np.empty(len(x), np.complex64)
        y.real = s * x.real.astype(np.float64)
        y.imag = s * x.imag.astype(np.float64)
        return y
    return (s * np.asarray(x).astype(np.float64)).astype(np.float32)


def _one_pole(alpha, u, y_prev):
    """y[n] = (1-alpha) y[n-1] + alpha u[n] from y_prev, as lfilter computes it."""
    a = 1 - alpha
    y, _ = scipy.signal.lfilter([alpha], [1, -a], u, zi=[a * y_prev])
    return y


class _Level:
    def __init__(self, power_alpha, threshold_dbfs):
        self.power_alpha = power_alpha
        self.threshold = 10 ** (threshold_dbfs / 10)
        self.reset()

    def reset(self):
        self.average_power = 0.0
        self.gain = 0.0

    def powers(self, x):
        """P[n] over x (state advanced), as the vectorised form computes it."""
        if len(x) == 0:
            return np.zeros(0)
        P = _one_pole(self.power_alpha, _power(x), self.average_power)
        self.average_power = float(P[-1])
        return P


class AGC(_Level):
    """agc.lua:41-115.  Constants derived in the reference's expression order (agc.lua:57-68)."""

    def __init__(self, mode, target=None, threshold=None, options=None, rate=2.0):
        options = options or {}
        self.gain_tau = {"fast": 0.1, "slow": 3.0}.get(mode, options.get("gain_tau"))
        self.power_tau = options.get("power_tau", 1.0)
        power_alpha = 1 / (1 + self.power_tau * rate)
        self.gain_alpha = 1 / (1 + self.gain_tau * rate)
        self.target = 10 ** ((-35 if target is None else target) / 10)
        _Level.__init__(self, power_alpha, -75 if threshold is None else threshold)

    def process_loop(self, x):
        pa, ga, T, theta = self.power_alpha, self.gain_alpha, self.target, self.threshold
        P, g = self.average_power, self.gain
        cplx = np.iscomplexobj(x)
        y = np.array(x, copy=True)
        for i in range(len(x)):
            if cplx:
                re, im = float(x[i].real), float(x[i].imag)
                P = (1 - pa) * P + pa * (re * re + im * im)
            else:
                v = float(x[i])
                P = (1 - pa) * P + pa * (v * v)
            if P >= theta:
                g = (1 - ga) * g + ga * (T * (1 / P))
                s = math.sqrt(g)
                y[i] = complex(np.float32(s * re), np.float32(s * im)) if cplx else np.float32(s * v)
        self.average_power, self.gain = P, g
        return y

    def process(self, x):
        x = np.asarray(x)
        P = self.powers(x)
        gate = P >= self.threshold
        y = np.array(x, copy=True)
        if gate.any():
            g_open = _one_pole(self.gain_alpha, self.target * (1 / P[gate]), self.gain)
            y[gate] = _scale(x[gate], np.sqrt(g_open))
            self.gain = float(g_open[-1])
        return y

    def gate(self, x):
        """(P, open) over x from the current state, without advancing it."""
        P = _one_pole(self.power_alpha, _power(np.asarray(x)), self.average_power) if len(x) else np.zeros(0)
        return P, P >= self.threshold


class PowerSquelch(_Level):
    """powersquelch.lua:24-75.  tau is always 0.001 (powersquelch.lua:26 reads an undefined global), so the second
    constructor argument is ignored."""

    def __init__(self, threshold, cutoff=None, rate=2.0):
        self.tau = 0.001
        _Level.__init__(self, 1 / (1 + self.tau * rate), threshold)

    def process_loop(self, x):
        pa, theta, P = self.power_alpha, self.threshold, self.average_power
        cplx = np.iscomplexobj(x)
        y = np.zeros_like(x)
        for i in range(len(x)):
            if cplx:
                re, im = float(x[i].real), float(x[i].imag)
                P = (1 - pa) * P + pa * (re * re + im * im)
            else:
                v = float(x[i])
                P = (1 - pa) * P + pa * (v * v)
            if P >= theta:
                y[i] = x[i]
        self.average_power = P
        return y

    def process(self, x):
        x = np.asarray(x)
        P = self.powers(x)
        return np.where(P >= self.threshold, x, np.zeros_like(x))

    def gate(self, x):
        P = _one_pole(self.power_alpha, _power(np.asarray(x)), self.average_power) if len(x) else np.zeros(0)
        return P, P >= self.threshold
