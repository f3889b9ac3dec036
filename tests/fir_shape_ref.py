"""Float64 references, per-output error bounds and deliberately wrong references ("mutants") for the register-tiled FIR
stages: the tuner / tuner+discriminator (tuner.cu), the real (5, 27) decimator with or without the fused pole, the
resamplers (resample.cu) and the generic polyphase decimator (poly_generic.cu).

Every reference starts at global input index n0 with zero history, which is what a fresh (or reset) graph gives after
lrb200_graph_seek(n0): the translator phase is that of the global index, the kept samples are those with
(n0 + j) mod D == 0.  References are computed in float64 from the float32 taps and samples.

Bounds are per output.  With u = 2^-24 and T the taps the kernel walks per output (zero padding included):
    |y_got - y| <= K u S~ + 2 pi (n0 + n) 2^-64 S,   K = 2 (T + 1) + 16,
    S  = sum_k |h_k| |x_{n-k}|,   S~ = ||h||_1 max |x| over the inputs the output reads, widened by D on each side
(the fast-FIR sub-filter (G0 + G1)(u0 + u1) - A - B takes rounding error from the neighbouring sample block; the last
term is the 2^-64-turn fixed-point phase).  Behind a discriminator the angle difference, wrapped to (-pi, pi], is at
most asin(e_n / |y_n|) + asin(e_{n-1} / |y_{n-1}|) + 1e-6 rad (polynomial atan2, __fdividef, float32 product), divided
by the gain; an output whose neighbour bound reaches |y| is not checked (start-up, fades, noise check themselves)."""
from fractions import Fraction

import numpy as np
import scipy.signal
from scipy.ndimage import maximum_filter1d

from tests.test_gpu_bounds import fir_ref

U = 2.0 ** -24
DISC_ANGLE = 1e-6          # rad: polynomial atan2 (1.1e-7, common.cuh), __fdividef and the float32 product
POLE_WARM = 64             # outputs of warm-up in front of every run of the fused pole (tuner.cu PT_POLE_WARM)


# ---- references ---------------------------------------------------------------------------------------------------
def phase_turns(turns, n0, n):
    """frac(turns * (n0 + j)) for j < n, `turns` the float64 the library receives; exact up to the last rounding."""
    assert n < 1 << 26
    base = float((Fraction(turns) * n0) % 1)
    c = 134217729.0 * turns                # Veltkamp split: hi, lo have <= 26 significant bits, so hi*j, lo*j are exact
    hi = c - (c - turns)
    lo = turns - hi
    j = np.arange(n, dtype=np.float64)
    a, b = hi * j, lo * j
    s = (a - np.floor(a)) + (b - np.floor(b)) + base
    return s - np.floor(s)


def rotate(x, turns, n0):
    return np.asarray(x).astype(np.complex128) * np.exp(2j * np.pi * phase_turns(turns, n0, len(x)))


def kept(n0, D, n, phase=0):
    """Indices j < n of the kept samples, (n0 + j) mod D == phase (phase != 0: a wrong decimation phase)."""
    return np.arange((phase - n0) % D, n, D)


def tuner_full(h, x, turns, n0):
    """Translator(turns) -> FIR(h) at full rate (turns None: no translator)."""
    return fir_ref(h, rotate(x, turns, n0) if turns is not None else np.asarray(x), wide=True)


def tuner_ref(h, x, turns, D, n0=0):
    """Translator(turns) -> FIR(h) -> Downsampler(D) from global index n0, zero history."""
    return tuner_full(h, x, turns, n0)[kept(n0, D, len(x))]


def discrim(y, gain, lag=1):
    """FrequencyDiscriminator: arg(y[n] conj(y[n-lag])) / gain, y[-1] = 0 (lag 2 is a mutant)."""
    prev = np.concatenate([np.zeros(lag, y.dtype), y[:-lag]])
    return np.angle(y * np.conj(prev)) / gain


def resample_ref(h, x, L, D, c=1.0, phase_map=None, direct=False):
    """[c *] Upsampler(L) -> FIR(h) -> Downsampler(D): at upsampled index i = m D = q L + p,
    y[m] = sum_t h[p + t L] c x[q - t].  phase_map(p) replaces p in the taps (a mutant).  direct: sum the products
    directly instead of by FFT (exact for a single non-zero tap, whose outputs are c x or 0)."""
    x = np.asarray(x)
    u = x.astype(np.complex128 if np.iscomplexobj(x) else np.float64) * np.float64(c)
    i = np.arange(0, len(x) * L, D)
    q, p = np.divmod(i, L)
    y = np.zeros(len(i), u.dtype)
    h = np.asarray(h)
    for pp in range(L):
        hp = h[(phase_map(pp) if phase_map else pp)::L]
        sel = p == pp
        if len(hp) and sel.any():
            y[sel] = (np.convolve(u, hp)[:len(u)] if direct else fir_ref(hp, u, wide=True))[q[sel]]
    return y


def pole_taps(h, b, a, D):
    """The combined taps of FIR(h) -> IIR(b, 1 / (1 - c z^-1)) -> Downsampler(D) behind the noble identity (graph.cu),
    in float64, and the output-rate pole c^D."""
    c = -float(a[1]) / float(a[0])
    g = np.zeros(len(b) + D - 1)
    for k in range(D):
        g[k:k + len(b)] += c ** k * np.asarray(b, np.float64) / float(a[0])
    return np.convolve(np.asarray(h, np.float64), g), c ** D


def pole_ref(h, b, a, x, D, n0=0):
    """FIR(h) -> IIR(b, a) -> Downsampler(D) in float64, zero state."""
    u = fir_ref(h, np.asarray(x), wide=True)
    return scipy.signal.lfilter(np.asarray(b, np.float64), np.asarray(a, np.float64), u)[kept(n0, D, len(x))]


# ---- bounds -------------------------------------------------------------------------------------------------------
def window_max(a, lo, hi):
    """m[j] = max(a[j + lo .. j + hi]) over the stream (zero outside it)."""
    pad = max(abs(lo), abs(hi)) + 1
    ap = np.concatenate([np.zeros(pad), np.asarray(a, np.float64), np.zeros(pad)])
    s = hi - lo + 1
    m = maximum_filter1d(ap, s, mode="constant", cval=0.0, origin=-(s // 2))       # m[i] = max ap[i .. i + s - 1]
    return m[pad + lo:pad + lo + len(a)]


def k_factor(T):
    return 2 * (T + 1) + 16


def linear_bound(h, ax, idx, n0, T, D):
    """Bound of the FIR outputs at full-rate indices idx over input magnitudes ax, with the phase term of a translator
    at global index n0 + idx."""
    h = np.abs(np.asarray(h).astype(np.complex128))
    S = np.maximum(fir_ref(h, ax, wide=True), 0.0)[idx] if len(ax) else np.zeros(0)
    w = window_max(ax, -(len(h) - 1) - D, D)[idx]
    return k_factor(T) * U * float(np.sum(h)) * w + 2 * np.pi * (n0 + idx.astype(np.float64)) * 2.0 ** -64 * S


def tuner_bound(h, x, D, n0, T):
    ax = np.abs(np.asarray(x).astype(np.complex128))
    return linear_bound(h, ax, kept(n0, D, len(ax)), n0, T, D)


def disc_bound(y, e, gain):
    """Output-unit bound of the discriminator behind a stage with output y and bound e (inf where unchecked)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(np.abs(y) > 0, e / np.abs(y), np.inf)
    a = np.where(r < 1, np.arcsin(np.minimum(r, 1.0)), np.inf)
    prev = np.concatenate([[np.inf], a[:-1]])
    return (a + prev + DISC_ANGLE) / abs(gain)


def resample_bound(h, x, L, D, c, T):
    """Bound of resample_ref: the FIR over the non-zero products c x[q - t], window over the inputs widened by D."""
    ax = np.abs(np.asarray(x).astype(np.complex128)) * abs(float(c))
    q = np.arange(0, len(ax) * L, D) // L
    w = window_max(ax, -(-(-len(h) // L)) - D, D)[q] if len(ax) else np.zeros(0)
    return k_factor(T) * U * float(np.sum(np.abs(h))) * w


def pole_bound(h, b, a, x, D, z, T, n0=0):
    """FIR bound (of the combined taps) carried through z[m] = c^D z[m-1] + w[m], plus the recurrence's own rounding
    (the scan's float32 powers of c included: 16 u |z| per step, geometric) and the warm-up truncation the fused
    pole allows (|c^D|^64 <= 1e-8)."""
    hc, cD = pole_taps(h, b, a, D)
    ax = np.abs(np.asarray(x, np.float64))
    ew = linear_bound(hc, ax, kept(n0, D, len(ax)), n0, T, D)
    carried = scipy.signal.lfilter([1.0], [1.0, -abs(cD)], ew + 16 * U * np.abs(z))
    warm = 1e-8 * window_max(np.abs(z), -POLE_WARM, 0)
    return carried + warm


# ---- checks -------------------------------------------------------------------------------------------------------
def wrapped(d, gain):
    """Discriminator output difference as an angle wrapped to (-pi, pi], back in output units."""
    a = np.asarray(d, np.float64) * gain
    return np.abs((a + np.pi) % (2 * np.pi) - np.pi) / abs(gain)


def excess(got, ref, bound, gain=None):
    """max over outputs of |got - ref| / bound (0 where the bound is inf); > 1 is a failure."""
    n = min(len(got), len(ref), len(bound))
    got = np.asarray(got)[:n].astype(np.complex128)
    ref = np.asarray(ref)[:n].astype(np.complex128)
    d = wrapped((got - ref).real, gain) if gain else np.abs(got - ref)
    b = np.asarray(bound)[:n]
    ok = np.isfinite(b)
    if not ok.any():
        return 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.max(np.where(b[ok] > 0, d[ok] / b[ok], np.where(d[ok] > 0, np.inf, 0.0))))


# ---- mutants: plausible wrong references ------------------------------------------------------------------------------
def _mutant_taps(h):
    """Wrong tap sets; one that equals the taps by construction (the reversal of symmetric taps, dropping a zero last
    tap) is left out: the kernel's error could not show on those taps either."""
    m = {"reversed taps": h[::-1], "taps shifted +1": np.concatenate([np.zeros(1, h.dtype), h]),
         "taps shifted -1": h[1:], "last tap dropped": h[:-1]}
    if np.array_equal(h[::-1], h):
        del m["reversed taps"]
    if h[-1] == 0:
        del m["last tap dropped"]
    return m


def _conj_visible(h, turns, D, gain):
    """The conjugated translator differs from the truth: not for offset 0 or +-rate/2; behind a discriminator not for
    an offset below its resolution, nor (single tap) when the output-rate frequency error 2 D turns is whole turns."""
    if turns is None or (2 * turns) % 1 == 0:
        return False
    if gain:
        err = (2 * D * turns) % 1
        if abs(turns) < 1e-6 or (np.count_nonzero(h) == 1 and min(err, 1 - err) < 1e-6):
            return False
    return True


def tuner_mutants(h, x, turns, D, n0, gain=None):
    """Wrong references of [Translator ->] FIR -> Downsampler [-> Discriminator] (turns None: no translator)."""
    h = np.asarray(h)
    post = (lambda y: discrim(y, gain)) if gain else (lambda y: y)
    out = {name: post(tuner_ref(hm, x, turns, D, n0)) for name, hm in _mutant_taps(h).items()}
    full = tuner_full(h, x, turns, n0)
    for s in (1, -1):
        out["decimation phase %+d" % s] = post(full[kept(n0, D, len(x), s)])
    if _conj_visible(h, turns, D, gain):
        out["conjugated translator"] = post(tuner_ref(h, x, -turns, D, n0))
    if gain:
        out["discriminator against y[n-2]"] = discrim(full[kept(n0, D, len(x))], gain, lag=2)
    return out


def resample_mutants(h, x, L, D, c):
    h = np.asarray(h)
    out = {name: resample_ref(hm, x, L, D, c) for name, hm in _mutant_taps(h).items() if len(hm)}
    hp = np.concatenate([h, np.zeros(-len(h) % L, h.dtype)]).reshape(-1, L)
    if not np.array_equal(hp[:, ::-1], hp):
        out["phase L-1-p"] = resample_ref(h, x, L, D, c, phase_map=lambda p: L - 1 - p)
    if D > 1:
        u = resample_ref(h, x, L, 1, c)
        for s in (1, -1):
            out["decimation phase %+d" % s] = u[np.arange(s % D, len(u), D)]
    return out


def pole_mutants(h, b, a, x, D, n0=0):
    h = np.asarray(h)
    out = {name: pole_ref(hm, b, a, x, D, n0) for name, hm in _mutant_taps(h).items()}
    u = scipy.signal.lfilter(np.asarray(b, np.float64), np.asarray(a, np.float64), fir_ref(h, np.asarray(x), wide=True))
    for s in (1, -1):
        out["decimation phase %+d" % s] = u[kept(n0, D, len(x), s)]
    return out
