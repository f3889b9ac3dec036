"""Window-method FIR tap design on the host in float64 (taps are float32-rounded by the block).

Mirrors radio/utilities/filter_utils.lua:21-107 (ideal responses), :121-141 (firwin scaling),
:152-205 (real designs), :220-285 (complex designs), :350-376 (Hilbert).  Runs once per block in
initialize(); the GPU only ever sees the finished taps.
"""
import math

from . import window_utils


def _centre(num_taps):
    return (num_taps - 1) / 2.0


def fir_lowpass(num_taps, cutoff):
    c = _centre(num_taps)
    h = []
    for n in range(num_taps):
        if n == c:
            h.append(cutoff)
        else:
            h.append(math.sin(math.pi * cutoff * (n - c)) / (math.pi * (n - c)))
    return h


def fir_highpass(num_taps, cutoff):
    assert num_taps % 2 == 1, "Number of taps must be odd."
    c = _centre(num_taps)
    h = []
    for n in range(num_taps):
        if n == c:
            h.append(1 - cutoff)
        else:
            h.append(-math.sin(math.pi * cutoff * (n - c)) / (math.pi * (n - c)))
    return h


def fir_bandpass(num_taps, cutoffs):
    assert num_taps % 2 == 1, "Number of taps must be odd."
    assert len(cutoffs) == 2, "Cutoffs should be a length two array."
    c = _centre(num_taps)
    h = []
    for n in range(num_taps):
        if n == c:
            h.append(cutoffs[1] - cutoffs[0])
        else:
            h.append(math.sin(math.pi * cutoffs[1] * (n - c)) / (math.pi * (n - c))
                     - math.sin(math.pi * cutoffs[0] * (n - c)) / (math.pi * (n - c)))
    return h


def fir_bandstop(num_taps, cutoffs):
    assert num_taps % 2 == 1, "Number of taps must be odd."
    assert len(cutoffs) == 2, "Cutoffs should be a length two array."
    c = _centre(num_taps)
    h = []
    for n in range(num_taps):
        if n == c:
            h.append(1 - (cutoffs[1] - cutoffs[0]))
        else:
            h.append(math.sin(math.pi * cutoffs[0] * (n - c)) / (math.pi * (n - c))
                     - math.sin(math.pi * cutoffs[1] * (n - c)) / (math.pi * (n - c)))
    return h


def firwin(h, window_type, scale_freq):
    window_type = window_type or "hamming"
    w = window_utils.window(len(h), window_type)
    h = [a * b for a, b in zip(h, w)]
    c = _centre(len(h))
    scale = 0.0
    for n in range(len(h)):
        scale += h[n] * math.cos(math.pi * (n - c) * scale_freq)
    return [a / scale for a in h]


def firwin_lowpass(num_taps, cutoff, window_type=None):
    return firwin(fir_lowpass(num_taps, cutoff), window_type, 0.0)


def firwin_highpass(num_taps, cutoff, window_type=None):
    return firwin(fir_highpass(num_taps, cutoff), window_type, 1.0)


def firwin_bandpass(num_taps, cutoffs, window_type=None):
    return firwin(fir_bandpass(num_taps, cutoffs), window_type, (cutoffs[0] + cutoffs[1]) / 2.0)


def firwin_bandstop(num_taps, cutoffs, window_type=None):
    return firwin(fir_bandstop(num_taps, cutoffs), window_type, 0.0)


def complex_firwin(h, center_freq, window_type, scale_freq):
    window_type = window_type or "hamming"
    N = len(h)
    hc = [complex(h[n] * math.cos(math.pi * center_freq * n), h[n] * math.sin(math.pi * center_freq * n)) for n in range(N)]
    w = window_utils.window(N, window_type)
    hc = [a * b for a, b in zip(hc, w)]
    c = _centre(N)
    scale = 0j
    for n in range(N):
        scale += hc[n] * complex(math.cos(math.pi * (n - c) * scale_freq), math.sin(-1 * math.pi * (n - c) * scale_freq))
    return [a / scale for a in hc]


def firwin_complex_bandpass(num_taps, cutoffs, window_type=None):
    h = fir_lowpass(num_taps, (max(cutoffs) - min(cutoffs)) / 2.0)
    centre = (cutoffs[0] + cutoffs[1]) / 2.0
    return complex_firwin(h, centre, window_type, centre)


def firwin_complex_bandstop(num_taps, cutoffs, window_type=None):
    h = fir_highpass(num_taps, (max(cutoffs) - min(cutoffs)) / 2.0)
    scale_freq = 1.0 if (cutoffs[0] < 0.0 and 0.0 < cutoffs[1]) else 0.0
    return complex_firwin(h, (cutoffs[0] + cutoffs[1]) / 2.0, window_type, scale_freq)


def fir_hilbert_transform(num_taps, window_type=None):
    window_type = window_type or "hamming"
    if num_taps % 2 == 0:
        raise ValueError("Number of taps must be odd.")
    h = []
    for n in range(num_taps):
        n_shifted = n - (num_taps - 1) // 2
        h.append(0.0 if n_shifted % 2 == 0 else 2.0 / (n_shifted * math.pi))
    w = window_utils.window(num_taps, window_type)
    return [a * b for a, b in zip(h, w)]


def fir_root_raised_cosine(num_taps, sample_rate, beta, symbol_period):
    """filter_utils.lua:301-337: root raised cosine taps, normalised to unity DC gain."""
    if num_taps % 2 == 0:
        raise ValueError("Number of taps must be odd.")

    def approx_equal(a, b):
        return abs(a - b) < 1e-5

    h = []
    for n in range(num_taps):
        t = (n - (num_taps - 1) / 2) / sample_rate
        if t == 0:
            h.append((1 / math.sqrt(symbol_period)) * (1 - beta + 4 * beta / math.pi))
        elif approx_equal(t, -symbol_period / (4 * beta)) or approx_equal(t, symbol_period / (4 * beta)):
            h.append((beta / math.sqrt(2 * symbol_period)) * ((1 + 2 / math.pi) * math.sin(math.pi / (4 * beta))
                                                             + (1 - 2 / math.pi) * math.cos(math.pi / (4 * beta))))
        else:
            num = (math.cos((1 + beta) * math.pi * t / symbol_period)
                   + math.sin((1 - beta) * math.pi * t / symbol_period) / (4 * beta * t / symbol_period))
            denom = (1 - (4 * beta * t / symbol_period) * (4 * beta * t / symbol_period))
            h.append(((4 * beta) / (math.pi * math.sqrt(symbol_period))) * num / denom)
    scale = 0
    for v in h:
        scale = scale + v
    return [v / scale for v in h]
