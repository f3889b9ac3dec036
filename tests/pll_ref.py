"""Float64 model, phase rebuild, per-output bound, acceptance thresholds and deliberately wrong variants ("mutants") of
PLLBlock's two GPU forms (pll.cu): the sequential kernel (pll_kernel) and the verified chunk-parallel one
(pll_sim_kernel, pll_verify_kernel, pll_out_kernel; lrb200_pll_set_mode(q, 1)).

Recurrence (pll.lua:140-170, restated by oracle.lr_oracle.PLL).  Per sample, with e the float32 phase-detector output,

    freq' = freq + beta e                 (the frequency before the clamp)
    phi   = phi + freq' + alpha e          wrapped to +-2 pi
    phim  = phim + m freq' + alpha e       wrapped to +-2 pi, out = exp(j phim) before the update
    freq  = clamp(freq', fmin, fmax)

Chunk-parallel decomposition (a call of n >= 2 L samples; shorter calls run the sequential form).  W = ceil(24 / (zeta
bw)) is the lead-in, L = max(4 W, 16384) the chunk length; chunk c covers [c L, min(c L + L, n)).

  * sim: chunk 0 starts from the carried (phi, freq); every other chunk from phi = atan2f(x[c L - W]) and the centre
    frequency, run over the W samples before it (their errors are discarded).  Over its own samples each chunk writes e,
    remembers its speculated start (phi0, freq0: its state at its first sample), sums its multiplied-phase advance dP
    with phim's own expression, wrapped at every step, and ends at (phi_end, freq_end).
  * verify: the lead-in assumes that it reaches the loop's true trajectory.  It does not when the input gives the loop
    nothing to pull with (zeros) or when the loop is not locked (noise, acquisition).  So each chunk's speculated start
    is checked, in stream order, against the true state T:
      - chunk 0: T is the carried state (chunk 0 starts from it, so it is always accepted);
      - chunk c >= 1: T is chunk c - 1's (phi_end, freq_end), after any re-run of chunk c - 1.
    Chunk c is accepted when |wrap(T.phi - phi0_c)| <= DPHI and |T.freq - freq0_c| <= DFREQ, the phase difference taken
    modulo 2 pi (phi wraps at +-2 pi, and a lead-in that starts from atan2f lands on either branch).  Otherwise it is
    re-run from T over its own samples with the sequential recurrence: err is rewritten, freq0 = T.freq, phi0 = T.phi
    and dP, phi_end, freq_end are recomputed.  A re-run chunk is the sequential form's, bit for bit, whenever T is (so
    err equals mode 0's on every sample before the first accepted chunk).
  * prefix: base_0 = the carried phim, base_{c+1} = wrap(base_c + dP_c); the carried state becomes the last chunk's
    (phi_end, freq_end) and wrap(base_last + dP_last).
  * out: from (base_c, freq0_c) each chunk advances phim over its samples from the stored e, as the sequential form.

Phase rebuild (`rebuild_phase`).  From a kernel's own e and the state at the start of the stream, freq' is recomputed
with the kernel's own double operations (so it is the kernel's freq' bit for bit: `fma=True` for the GPU, whose compiler
fuses freq + beta e into one rounding), and phi_multiplied[i] = phase0 + sum_{k<i} (m freq'_k + alpha e_k) is summed
exactly: every product is split into two doubles (Dekker), every double into integer multiples of 2^-50 and 2^-82, the
integers are summed exactly in int64 limbs and the result is reduced mod 2 pi once, in long double with a two-part 2 pi
(Cody-Waite).  Its own error: each term leaves at most 4 roundings of 2^-83 (8e-26 in all) and the reduction and the final
sums about 1e-16, so it stays below 1e-15 at 2^27 samples (test_pll_ref.py checks it against fractions.Fraction at a
phase of 2^30 rad).

Per-output bound (`phase_bound`).  |out[i] - exp(j phi_multiplied[i])| <= OUT_ROUND + C (i + 1) + K, i counted from the
start of the stream (or the last reset), where

  * OUT_ROUND = sqrt(2) 2^-25 + 1e-15: cos and sin of phim rounded to float32 (half an ulp below 1 is 2^-25) after a
    double sincos (a few ulp of 1);
  * C = u (4 pi + 3 I) + delta I / (2 pi - I) + 3 (u 4 pi + delta) / 32768, with u = 2^-53, delta = |2 pi - fl(2 pi)|
    = 2.45e-16 and I = |m| F + alpha pi the largest increment, F = max(|fmin|, |fmax|) + beta pi the largest |freq'|.
    phim's update rounds m freq' (<= u |m| F), phim + m freq' and the final sum (< 2 pi + I each) and alpha e (<= u alpha
    pi): at most u (4 pi + 3 I) per sample, whether or not the compiler fuses them.  A wrap subtracts fl(2 pi) exactly
    (Sterbenz) but is delta off 2 pi; after a wrap phim is within I of 0, so the next one needs 2 pi - I of travel:
    delta I / (2 pi - I) per sample and one delta.  The chunk-parallel form does the same per sample (dP is the same sum)
    and adds one rounding (< 4 pi) and one wrap per chunk and per call: chunks are >= 16384 samples and calls >= 32768,
    hence the last term;
  * K = 2 (u 4 pi + delta): the first wrap and the last partial chunk.

Because every partial sum of both forms stays below 4 pi, C is a few ulp of 2 pi: 1.8e-15 for the stereo loop, 1.2e-7
after 2^26 samples.  The sequential kernel meets it for any input; the chunk-parallel one also needs every chunk's
lead-in to have reached the sequential trajectory (a locked loop), or its freq0 differs from the freq' the rebuild
carries across the chunk boundary.

Parallel vs sequential.  After lock the lead-in leaves each chunk on the sequential trajectory up to the resolution of
the float32 phase detector (a VCO phase difference below float32 resolution changes no e, so nothing pulls it back):
ERR_TOL bounds |e_parallel - e_sequential| and out_tol(c) |out_parallel - out_sequential| after the first call, which
acquires in the sequential form, for a stream whose parallel calls have run c lead-ins in all (`lead_ins`).  Both come
from the model against O.PLL, with 4x headroom or more:

  * e: the worst case is 1.8e-7 (test_pll_ref.py's inputs, and noisy RDS / AM-synchronous streams of up to 320
    chunks); ERR_TOL = 1e-6;
  * out: two float32 roundings of the output (2 OUT_ROUND = 8.5e-8) plus what the lead-ins leave in the multiplied
    phase.  Each lead-in leaves its own difference there and they add up like a random walk: on a noisy RDS stream
    the model's out difference is 1.3e-7, 2.2e-7, 4.8e-7 and 5.6e-7 after 10, 40, 160 and 320 chunks, at most
    2 OUT_ROUND + 3.3e-8 sqrt(c).  out_tol(c) = 4 (2 OUT_ROUND + 3.3e-8 sqrt(c)).

A lead-in of W / 2 still reaches the sequential trajectory on every input tried, including one whose phase guess is
2.5 rad off (W is conservative), so no input here tells W / 2 from W: the lead-in mutant shortens it to W / 8, and the
input that shows it turns the sample its phase guess is taken from.  The lead-in length is therefore checked only
down to W / 8.

Thresholds (`thresholds`).  Write a start-state offset (dphi, dfreq) against the true trajectory.  While the offset is
small the float32 phase detector reads it as e' = e - dphi (atan2 of x conj(vco) turns with the VCO phase, whatever the
amplitude), so the offsets follow the linearised loop

    dfreq_{k+1} = dfreq_k - beta dphi_k
    dphi_{k+1}  = dphi_k + dfreq_{k+1} - alpha dphi_k
    dphim_{k+1} = dphim_k + m dfreq_{k+1} - alpha dphi_k          (dphim_0 = 0)

(the clamp cannot widen a frequency difference).  The error differs by dphi_k and out by at most dphim_k, for the whole
rest of the stream: a phase offset is never pulled back out of the multiplied phase (dphim tends to -m dphi_0 +
(m - 1) alpha / beta dfreq_0).  `gains` iterates the system from (1, 0) and (0, 1) until both have died out and returns
the largest |dphi_k| and |dphim_k| of each, G_e,phi, G_e,f, G_o,phi and G_o,f.  A chunk that starts exactly at the
thresholds therefore leaves at most

    |e - e_true|   <= G_e,phi DPHI + G_e,f DFREQ
    |out - out_t|  <= G_o,phi DPHI + G_o,f DFREQ

Two conditions are wanted: (a) every lead-in on a locked input accepted with a wide margin, so that locked input
re-runs nothing, and (b) a chunk that starts exactly at the thresholds within the tolerances of the parallel form.
The thresholds are a box (s alpha, s beta): the loop filter's step on one detector error s, the shape of what a lead-in
leaves (it reaches the trajectory until a few float32 ulps of e, eps = 2^-23, tell them apart: the model observes at
most 1.22 alpha eps and 0.57 beta eps over the inputs of test_pll_ref.py).  s is the largest that keeps a chunk
starting at the box's corner within ERR_BUDGET = ERR_TOL / 4 in error and OUT_BUDGET = out_tol(1) - 2 OUT_ROUND =
3.84e-7 in out (the two output roundings of any comparison are already in out_tol):

    s = min(ERR_BUDGET / (G_e,phi alpha + G_e,f beta), OUT_BUDGET / (G_o,phi alpha + G_o,f beta))

    loop      alpha    beta     DPHI     DFREQ     bound by   lead-in margin (phase, freq)
    stereo    7.6e-3   2.9e-5   1.2e-7   4.4e-10   out        > 250x
    rds       0.108    6.1e-3   7.1e-8   4.1e-9    out        ~10x, ~18x
    am_sync   0.293    5.1e-2   1.8e-7   3.2e-8    error      >= 4x, >= 12x

A lead-in that fails (zeros, noise, acquisition) misses by about the pilot's offset from the centre, 1e-5 rad/sample
or more, and by radians in phase: orders of magnitude outside every box.

Two limits of this choice.  (b) holds with 4x headroom for the error but only 1x for out: a 4x margin on out_tol(1)
would put DPHI at 1e-8 for rds and 7e-8 for am_sync, inside what a converged lead-in leaves on a noisy pilot, and such
a chunk would be run again for nothing.  And (a), 10x between the largest lead-in difference and the threshold, cannot
hold for the am_sync loop together with (b): its worst lead-in (4.3e-8 rad on a noisy pilot) times 10 already moves
out by 5.3e-7 > out_tol(1).  The tests assert 4x for (a) and ERR_TOL / 4 and out_tol(1) for (b).

The GPU's PllBlock computes the same gains and thresholds in double (pll.cu, pll_thresholds)."""
import math
from fractions import Fraction

import numpy as np

from oracle import lr_oracle as O

F32, F64 = np.float32, np.float64
U = 2.0 ** -53
TWO_PI = 6.283185307179586476925286766559          # fl(2 pi), the kernels' constant
TWO_PI_FRAC = Fraction("6.28318530717958647692528676655900576839433879875021164194988918461563281257241799725606965068")
DELTA = abs(float(TWO_PI_FRAC - Fraction(TWO_PI)))
OUT_ROUND = math.sqrt(2.0) * 2.0 ** -25 + 1e-15
MIN_CHUNK = 16384
ERR_TOL = 1e-6
OUT_TOL_CHUNK = 3.3e-8       # the model's worst out difference per sqrt(lead-in)
ERR_BUDGET = 2.5e-7          # ERR_TOL / 4
OUT_BUDGET = 3.84e-7         # out_tol(1) - 2 OUT_ROUND (3.849e-7), rounded down

# (loop bandwidth, fmin, fmax, multiplier, rate): the receivers' loops
LOOPS = {
    "stereo": (100.0, 19e3 - 50, 19e3 + 50, 2.0, 220500.0),        # WBFMStereoDemodulator's pilot PLL
    "rds": (1500.0, 19e3 - 100, 19e3 + 100, 3.0, 220500.0),        # the RDS receiver's baseband PLL
    "am_sync": (1000.0, 10e3 - 100, 10e3 + 100, 1.0, 48000.0),     # AMSynchronousDemodulator(10e3, ...) at 48 kS/s
}
# a carrier-recovery loop centred on 0 Hz: phi rotates slowly, so a lead-in's atan2f guess sits 2 pi from the true
# branch on about half the chunks (what the wrap of the phase difference is for)
BASEBAND = (1000.0, -100.0, 100.0, 1.0, 48000.0)

MUTANTS = (
    # the sim, prefix and out passes
    "unreduced_prefix", "base_one_chunk_late", "phim0_after_call", "short_lead_in", "centre_freq_in_out_pass",
    "no_e_term", "last_end_start_plus_L",
    # the verify pass ("accept_all" is the unverified form: every lead-in accepted)
    "accept_all", "rerun_from_speculated", "t_from_speculated_end", "stale_dP", "stale_freq0", "phase_without_wrap")
A_OFFSET = 2.0 ** 26          # unreduced_prefix: the running sum A where a 2^27-sample call leaves it (0.5 rad/sample)


class Loop:
    """The loop constants of pll.lua:113-131 (as pll.cu PllBlock and O.PLL), the lead-in and the chunk length."""

    def __init__(self, bw_hz, fmin_hz, fmax_hz, mult, rate):
        o = O.PLL(bw_hz, fmin_hz, fmax_hz, mult, rate)
        self.args = (bw_hz, fmin_hz, fmax_hz, mult, rate)
        self.alpha, self.beta, self.fmin, self.fmax, self.mult = o.alpha, o.beta, o.fmin, o.fmax, o.mult
        self.centre = o.freq
        damping = math.sqrt(2.0) / 2
        bw = 2 * math.pi * (bw_hz / rate) / (damping + 1 / (4 * damping))
        self.W = int(math.ceil(24.0 / (damping * bw)))
        self.L = max(4 * self.W, MIN_CHUNK)

    def oracle(self):
        return O.PLL(*self.args)


def loop(name, mult=None):
    """The Loop of LOOPS[name] (or BASEBAND), with another multiplier if given."""
    args = list(BASEBAND if name == "baseband" else LOOPS[name])
    if mult is not None:
        args[3] = mult
    return Loop(*args)


# ---- the thresholds -----------------------------------------------------------------------------------------------------
def gains(loop, tail=1e-12):
    """(G_e,phi, G_e,f, G_o,phi, G_o,f): the largest |dphi_k| and |dphim_k| of the linearised loop from a unit phase and
    a unit frequency offset (see the module docstring).  Iterated until the state is below `tail` of its start."""
    a, b, m = loop.alpha, loop.beta, loop.mult
    res = []
    for p, f in ((1.0, 0.0), (0.0, 1.0)):
        pm, ge, go = 0.0, abs(p), 0.0
        k = 0
        while True:
            f = f - b * p
            pm = pm + m * f - a * p
            p = p + f - a * p
            ge, go = max(ge, abs(p)), max(go, abs(pm))
            k += 1
            if k > 64 and abs(p) < tail * ge and abs(f) < tail * b * ge:
                break
        res.append((ge, go))
    (gep, gop), (gef, gof) = res
    return gep, gef, gop, gof


def thresholds(loop):
    """(DPHI rad, DFREQ rad/sample) of the acceptance test (see the module docstring)."""
    gep, gef, gop, gof = gains(loop)
    a, b = loop.alpha, loop.beta
    sc = min(ERR_BUDGET / (gep * a + gef * b), OUT_BUDGET / (gop * a + gof * b))
    return sc * a, sc * b


def wrap_diff(d):
    """d reduced modulo 2 pi to [-pi, pi] (rint(d / 2 pi) turns, as the kernel)."""
    return d - TWO_PI * np.rint(d / TWO_PI)


# ---- the model --------------------------------------------------------------------------------------------------------
def _detect(xr, xi, phi):
    """e = atan2f of x conj(vco), the VCO and the product rounded to float32 (lanes in parallel)."""
    vr, vi = np.cos(phi).astype(F32).astype(F64), np.sin(phi).astype(F32).astype(F64)
    pr = (xr * vr - xi * (-vi)).astype(F32)
    pi = (xr * (-vi) + xi * vr).astype(F32)
    return np.arctan2(pi, pr).astype(F64)


def _wrap(v):
    v = np.where(v > TWO_PI, v - TWO_PI, v)
    return np.where(v < -TWO_PI, v + TWO_PI, v)


class Model:
    """PLLBlock as the kernels compute it, call by call: mode 0 sequential, mode 1 verified chunk-parallel (n >= 2 L).
    `process(x)` returns (out complex64, err float32); `mutant` selects one of MUTANTS.  After each parallel call
    `decisions` lists every chunk's (accepted, |phase difference|, |frequency difference|); `chunks` and `reruns` count
    the speculated chunks (each call's chunks after the first) and how many of them were re-run since create or reset,
    as lrb200_pll_chunk_counts."""

    def __init__(self, loop, mode=1, mutant=None):
        assert mutant is None or mutant in MUTANTS, mutant
        self.loop, self.mode, self.mutant = loop, mode, mutant
        self.dphi, self.dfreq = thresholds(loop)
        self.reset()

    def reset(self):
        self.phi, self.phim, self.freq = 0.0, 0.0, self.loop.centre
        self.chunks, self.reruns, self.decisions = 0, 0, []

    def process(self, x):
        x = np.asarray(x, np.complex64)
        if self.mode == 1 and len(x) >= 2 * self.loop.L:
            return self._parallel(x)
        return self._sequential(x)

    def _sequential(self, x):
        # pll_kernel: one sample after another, scalar (the same operations as _detect and _wrap)
        lp = self.loop
        n = len(x)
        out, err = np.zeros(n, np.complex64), np.zeros(n, F32)
        phi, phim, freq = self.phi, self.phim, self.freq
        xr, xi = x.real.astype(F64).tolist(), x.imag.astype(F64).tolist()
        for i in range(n):
            out[i] = complex(F32(math.cos(phim)), F32(math.sin(phim)))
            vr, vi = float(F32(math.cos(phi))), float(F32(math.sin(phi)))
            pr = F32(xr[i] * vr - xi[i] * (-vi))
            pi = F32(xr[i] * (-vi) + xi[i] * vr)
            e = float(np.arctan2(pi, pr, dtype=F32))
            err[i] = e
            freq = freq + lp.beta * e
            phi = phi + freq + lp.alpha * e
            phim = phim + freq * lp.mult + lp.alpha * e
            freq = min(max(freq, lp.fmin), lp.fmax)
            phi = phi - TWO_PI if phi > TWO_PI else phi
            phi = phi + TWO_PI if phi < -TWO_PI else phi
            phim = phim - TWO_PI if phim > TWO_PI else phim
            phim = phim + TWO_PI if phim < -TWO_PI else phim
        self.phi, self.phim, self.freq = phi, phim, freq
        return out, err

    def _rerun(self, x, phi, freq):
        """The chunk from (phi, freq) with the sequential recurrence: (err, dP, phi_end, freq_end)."""
        keep = self.phi, self.phim, self.freq
        self.phi, self.phim, self.freq = phi, 0.0, freq
        _, err = self._sequential(x)
        r = err, self.phim, self.phi, self.freq
        self.phi, self.phim, self.freq = keep
        return r

    def _parallel(self, x):
        lp, mut = self.loop, self.mutant
        n, L = len(x), lp.L
        W = lp.W // 8 if mut == "short_lead_in" else lp.W
        nch = (n + L - 1) // L
        starts = np.arange(nch) * L
        ends = np.minimum(starts + L, n)
        if mut == "last_end_start_plus_L":
            ends[-1] = starts[-1] + L                      # reads (zeros here) and runs past the call
        span = int(np.max(ends - starts))
        xp = np.concatenate([x, np.zeros(int(ends[-1]) - n + 1, np.complex64)])
        xr, xi = xp.real.astype(F64), xp.imag.astype(F64)
        err = np.zeros(len(xp), F32)

        def advance(p, f, e):
            # phi_multiplied's step (pll_advance), from freq' = f
            if mut == "no_e_term":
                return _wrap(p + (f + lp.alpha * e) * lp.mult)
            return _wrap(p + f * lp.mult + lp.alpha * e)

        # sim (pll_sim_kernel): the lead-ins of chunks 1.., then every chunk over its own samples
        phi = np.empty(nch)
        freq = np.full(nch, lp.centre)
        phi[0], freq[0] = self.phi, self.freq
        if nch > 1:
            b = starts[1:] - W
            phi[1:] = np.arctan2(xp.imag[b], xp.real[b]).astype(F64)      # atan2f of the sample, as float32
            for t in range(W):
                e = _detect(xr[b + t], xi[b + t], phi[1:])
                f = freq[1:] + lp.beta * e
                phi[1:] = _wrap(phi[1:] + f + lp.alpha * e)
                freq[1:] = np.clip(f, lp.fmin, lp.fmax)
        phi0, freq0 = phi.copy(), freq.copy()
        dP = np.zeros(nch)
        for t in range(span):
            act = starts + t < ends
            idx = np.where(act, starts + t, 0)
            e = _detect(xr[idx], xi[idx], phi)
            f = freq + lp.beta * e
            err[idx[act]] = e[act]
            phi = np.where(act, _wrap(phi + f + lp.alpha * e), phi)
            dP = np.where(act, advance(dP, f, e), dP)
            freq = np.where(act, np.clip(f, lp.fmin, lp.fmax), freq)
        # verify (pll_verify_kernel), in stream order: phi, freq keep the speculated ends, phi_end, freq_end the true ones
        phi_end, freq_end = phi.copy(), freq.copy()
        self.decisions = []
        Tphi, Tfreq = self.phi, self.freq
        for c in range(nch):
            if c > 0:
                Tphi, Tfreq = (phi[c - 1], freq[c - 1]) if mut == "t_from_speculated_end" else (phi_end[c - 1], freq_end[c - 1])
            d = Tphi - phi0[c]
            dp = abs(d if mut == "phase_without_wrap" else float(wrap_diff(d)))
            df = abs(Tfreq - freq0[c])
            ok = mut == "accept_all" or (dp <= self.dphi and df <= self.dfreq)
            self.decisions.append((ok, dp, df))
            if ok:
                continue
            s, e_ = int(starts[c]), int(ends[c])
            sphi, sfreq = (phi0[c], freq0[c]) if mut == "rerun_from_speculated" else (Tphi, Tfreq)
            err[s:e_], dp_new, phi_end[c], freq_end[c] = self._rerun(xp[s:e_], sphi, sfreq)
            if mut != "stale_dP":
                dP[c] = dp_new
            if mut != "stale_freq0":
                freq0[c] = sfreq
            phi0[c] = sphi
        self.chunks += nch - 1
        self.reruns += sum(not ok for ok, _, _ in self.decisions[1:])
        # prefix
        base = np.empty(nch)
        phim0 = self.phim
        ph = phim0
        for c in range(nch):
            base[c] = ph
            ph = float(_wrap(np.array(ph + dP[c])))
        phim_end = ph
        if mut == "base_one_chunk_late":
            base = np.concatenate([base[1:], [phim_end]])
        if mut == "phim0_after_call":
            ph = phim_end
            for c in range(nch):
                base[c] = ph
                ph = float(_wrap(np.array(ph + dP[c])))
        # out (pll_out_kernel)
        out = np.zeros(len(xp), np.complex64)
        fr = np.full(nch, lp.centre) if mut == "centre_freq_in_out_pass" else freq0.copy()
        if mut == "unreduced_prefix":
            # the earlier pll_out_kernel: phim0 + m A + (1 - m) alpha E from running sums A of freq' + alpha e and E of
            # e that start where a long call leaves them (A = A_OFFSET); the reference phase is then shifted by m A_OFFSET
            dA, dE = np.zeros(nch), np.zeros(nch)
            for c in range(nch):
                e = err[starts[c]:ends[c]].astype(F64)
                dA[c] = np.add.accumulate(freq_prime(e, lp, freq0[c]) + lp.alpha * e)[-1]
                dE[c] = np.add.accumulate(e)[-1]
            A0 = A_OFFSET + np.concatenate([[0.0], np.cumsum(dA)[:-1]])
            E0 = np.concatenate([[0.0], np.cumsum(dE)[:-1]])
            A, E = A0.copy(), E0.copy()
            for t in range(span):
                act = starts + t < ends
                idx = np.where(act, starts + t, 0)
                p = phim0 + lp.mult * A + (1.0 - lp.mult) * lp.alpha * E
                p = p - TWO_PI * np.floor(p / TWO_PI)
                o = (np.cos(p).astype(F32) + 1j * np.sin(p).astype(F32)).astype(np.complex64)
                out[idx[act]] = o[act]
                e = err[idx].astype(F64)
                f = fr + lp.beta * e
                A = np.where(act, A + (f + lp.alpha * e), A)
                E = np.where(act, E + e, E)
                fr = np.where(act, np.clip(f, lp.fmin, lp.fmax), fr)
            phim_end = math.fmod(phim0 + lp.mult * (A_OFFSET + float(np.sum(dA))) + (1 - lp.mult) * lp.alpha * float(np.sum(dE)),
                                 TWO_PI)
        else:
            pm = base.copy()
            for t in range(span):
                act = starts + t < ends
                idx = np.where(act, starts + t, 0)
                o = (np.cos(pm).astype(F32) + 1j * np.sin(pm).astype(F32)).astype(np.complex64)
                out[idx[act]] = o[act]
                e = err[idx].astype(F64)
                f = fr + lp.beta * e
                pm = np.where(act, advance(pm, f, e), pm)
                fr = np.where(act, np.clip(f, lp.fmin, lp.fmax), fr)
        self.phi, self.phim, self.freq = float(phi_end[-1]), phim_end, float(freq_end[-1])
        return out[:n], err[:n]


# ---- phase rebuild ------------------------------------------------------------------------------------------------------
def _two_prod(a, b):
    """a b = p + r exactly (Dekker / Veltkamp, no FMA needed)."""
    def split(v):
        c = 134217729.0 * v
        hi = c - (c - v)
        return hi, v - hi
    p = a * b
    ah, al = split(a)
    bh, bl = split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def freq_prime(err, loop, freq0=None, fma=False):
    """freq'_k of the recurrence driven by e = err, from freq = freq0 (the centre frequency by default), with the
    kernel's double operations: fl(freq + fl(beta e)) (fma=False, numpy / Lua) or fl(freq + beta e) (fma=True)."""
    e = np.asarray(err, F32).astype(F64)
    n = len(e)
    p = loop.beta * e
    r = _two_prod(np.full(n, loop.beta), e)[1] if fma else None
    out = np.empty(n)
    f = loop.centre if freq0 is None else freq0
    i, B = 0, 64
    while i < n:
        j = min(n, i + B)
        seg = np.add.accumulate(np.concatenate(([f], p[i:j])))[1:]      # strictly left to right
        bad = (seg > loop.fmax) | (seg < loop.fmin)
        fused = None
        if fma:
            prev = np.concatenate(([f], seg[:-1]))
            s, t = _two_sum(prev, p[i:j])
            fused = s + (t + r[i:j])
            bad |= fused != seg
        k = int(np.argmax(bad)) if bad.any() else -1
        if k < 0:
            out[i:j] = seg
            f = seg[-1]
            i, B = j, min(2 * B, 1 << 16)
        else:
            out[i:i + k] = seg[:k]
            v = fused[k] if fma else seg[k]
            out[i + k] = v
            f = min(max(v, loop.fmin), loop.fmax)
            i, B = i + k + 1, 64
    return out


_S1, _S2 = 50, 82                  # the two fixed-point grids, 2^-50 and 2^-82
_C1 = Fraction(math.floor(TWO_PI_FRAC * 2 ** 29), 2 ** 29)          # 32 bits: k C1 is exact in long double for k < 2^31


def _ld(fr):
    hi = float(fr)
    return np.longdouble(hi) + np.longdouble(float(fr - Fraction(hi)))


_C1_LD, _C2_LD, _TWO_PI_LD = _ld(_C1), _ld(TWO_PI_FRAC - _C1), _ld(TWO_PI_FRAC)


def _fixed(v):
    """v = q1 2^-50 + q2 2^-82 + (at most 2^-83), q1, q2 int64 (|v| < 2^12)."""
    q1 = np.rint(np.ldexp(v, _S1))
    rem = v - np.ldexp(q1, -_S1)                   # exact
    return q1.astype(np.int64), np.rint(np.ldexp(rem, _S2)).astype(np.int64)


def _reduce(x):
    k = np.rint(x / _TWO_PI_LD)
    return (x - k * _C1_LD) - k * _C2_LD


def rebuild_phase(err, loop, phase0=0.0, freq0=None, fma=False):
    """phi_multiplied[i] = phase0 + sum_{k<i} (m freq'_k + alpha e_k), reduced to [-pi, pi], for i < len(err), as
    float64 (see the module docstring)."""
    assert np.finfo(np.longdouble).nmant >= 63, "the reduction needs an 80-bit long double"
    e = np.asarray(err, F32).astype(F64)
    n = len(e)
    assert n < 1 << 30
    fp = freq_prime(e, loop, freq0, fma)
    q1 = np.zeros(n, np.int64)
    q2 = np.zeros(n, np.int64)
    for a, b in ((loop.mult, fp), (loop.alpha, e)):
        p, r = _two_prod(np.full(n, a), b)
        for v in (p, r):
            s1, s2 = _fixed(v)
            q1 += s1
            q2 += s2
    # phase0: an integer number of 2^-18 plus a remainder on the two grids
    h0 = math.floor(phase0 * 2.0 ** 18)
    r1, r2 = _fixed(np.array([phase0 - math.ldexp(h0, -18)]))
    hi, lo = q1 >> 32, q1 & 0xFFFFFFFF
    H = np.concatenate(([0], np.cumsum(hi)[:-1])) + h0
    Lo = np.concatenate(([0], np.cumsum(lo)[:-1])) + int(r1[0])
    S2 = np.concatenate(([0], np.cumsum(q2)[:-1])) + int(r2[0])
    ld = np.longdouble
    xh = _reduce(H.astype(ld) * ld(2.0 ** -18))
    tot = xh + Lo.astype(ld) * ld(2.0 ** -_S1) + S2.astype(ld) * ld(2.0 ** -_S2)
    return _reduce(tot).astype(F64)[:n]


def rebuild_phase_exact(err, loop, phase0=0.0, freq0=None, fma=False):
    """The same sum with fractions.Fraction, reduced with 2 pi to 90 digits (short streams only)."""
    fp = freq_prime(err, loop, freq0, fma)
    e = np.asarray(err, F32).astype(F64)
    m, a = Fraction(loop.mult), Fraction(loop.alpha)
    acc = Fraction(phase0)
    out = []
    for k in range(len(e)):
        q = acc / TWO_PI_FRAC
        kk = math.floor(q + Fraction(1, 2))
        out.append(acc - kk * TWO_PI_FRAC)
        acc += m * Fraction(float(fp[k])) + a * Fraction(float(e[k]))
    return out


# ---- the bound ----------------------------------------------------------------------------------------------------------
def per_sample_constant(loop):
    F = max(abs(loop.fmin), abs(loop.fmax)) + loop.beta * math.pi
    inc = abs(loop.mult) * F + loop.alpha * math.pi
    assert inc < math.pi
    return U * (4 * math.pi + 3 * inc) + DELTA * inc / (2 * math.pi - inc) + 3 * (U * 4 * math.pi + DELTA) / 32768


def phase_bound(loop, n, i0=0):
    """The bound on |out[i] - exp(j phi_multiplied[i])| for i < n, i counted from i0 samples after the stream's start."""
    K = 2 * (U * 4 * math.pi + DELTA)
    return OUT_ROUND + K + per_sample_constant(loop) * (np.arange(n, dtype=F64) + i0 + 1)


def lead_ins(lengths, loop):
    """The lead-ins a stream of calls of these lengths runs: every chunk but the first of each parallel call."""
    return sum((n + loop.L - 1) // loop.L - 1 for n in lengths if n >= 2 * loop.L)


def out_tol(c):
    """The tolerance of |out_parallel - out_sequential| over a stream of c lead-ins (see the module docstring)."""
    return 4 * (2 * OUT_ROUND + OUT_TOL_CHUNK * math.sqrt(c))


def out_ratio(out, phase, bound):
    """max_i |out[i] - exp(j phase[i])| / bound[i]."""
    ref = np.exp(1j * np.asarray(phase, F64))
    d = np.abs(np.asarray(out).astype(np.complex128) - ref)
    return float(np.max(d / bound)) if len(d) else 0.0


# ---- test inputs --------------------------------------------------------------------------------------------------------
def pilot(loop, n, kind="clean", amplitude=1.0, seed=0, t0=0):
    """A tone at the loop's centre (+0.3 Hz) for samples t0 .. t0+n: 'clean', 'noisy' (10 dB SNR), 'offset' (+0.9 of
    the half-range), 'drift' (+-0.5 of the half-range, one slow sine over 2^21 samples), 'noise' (no tone), 'zeros'."""
    bw, fmin, fmax, _, rate = loop.args
    rng = np.random.default_rng(seed)
    t = np.arange(t0, t0 + n, dtype=F64)
    centre, half = 0.5 * (fmin + fmax), 0.5 * (fmax - fmin)
    if kind == "zeros":
        return np.zeros(n, np.complex64)
    if kind == "noise":
        return (amplitude * (rng.standard_normal(n) + 1j * rng.standard_normal(n)) / math.sqrt(2)).astype(np.complex64)
    if kind == "offset":
        ph = 2 * np.pi * (centre + 0.9 * half) / rate * t
    elif kind == "drift":
        T = float(1 << 21)
        ph = 2 * np.pi * centre / rate * t + 2 * np.pi * 0.5 * half / rate * T / (2 * np.pi) * (1 - np.cos(2 * np.pi * t / T))
    else:
        ph = 2 * np.pi * (centre + 0.3) / rate * t
    x = amplitude * np.exp(1j * (np.mod(ph, 2 * np.pi) + 0.4))
    if kind == "noisy":
        x = x + amplitude * math.sqrt(0.1 / 2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return x.astype(np.complex64)


LOCKED = ("clean", "noisy", "offset", "drift")
UNLOCKED = ("zeros_pilot", "gap", "noise_pilot", "pilot_noise_pilot", "zeros", "noise", "freq_step")


def make_input(lp, kind, seed=21):
    """(x, call lengths).  Locked pilots: a sequential acquisition call, then one parallel call of 4 L + 777.  The rest
    run as one parallel call from a fresh loop: zeros (2.5 L) -> pilot; pilot (1.5 L) -> zeros -> pilot from W / 20
    before chunk 4's boundary (its lead-in starts in the zeros and has not settled when the pilot is back); noise
    (2 L) -> pilot; pilot -> noise (2 L) -> pilot; pure zeros and pure noise; a pilot that steps from +0.9 to -0.9 of
    the half-range W / 10 before chunk 3's boundary, so that chunk's lead-in has not settled (6 L + 3 in all)."""
    L = lp.L
    if kind in LOCKED:
        n1 = min(L, lp.W + 8000)
        lengths = [n1, 4 * L + 777]
        return pilot(lp, sum(lengths), kind, seed=seed), lengths
    n = 6 * L + 3
    if kind in ("zeros", "noise"):
        return pilot(lp, n, kind, seed=seed), [n]
    if kind == "freq_step":
        bw, fmin, fmax, _, rate = lp.args
        centre, half = 0.5 * (fmin + fmax), 0.5 * (fmax - fmin)
        step = 3 * L - lp.W // 10
        f = np.where(np.arange(n) < step, centre + 0.9 * half, centre - 0.9 * half)
        ph = np.concatenate([[0.0], np.cumsum(2 * np.pi * f / rate)[:-1]])
        return np.exp(1j * (np.mod(ph, 2 * np.pi) + 0.4)).astype(np.complex64), [n]
    x = pilot(lp, n, "noisy", seed=seed)
    gap, pos = (5 * L // 2 - lp.W // 20, 3 * L // 2) if kind == "gap" else (5 * L // 2, 0) if kind == "zeros_pilot" else (2 * L, 0) if kind == "noise_pilot" else (2 * L, 2 * L)
    fill = np.zeros(gap, np.complex64) if kind in ("gap", "zeros_pilot") else pilot(lp, gap, "noise", seed=seed + 1)
    x[pos:pos + gap] = fill
    return x, [len(x)]


def run_verified(lp, x, lengths, mutant=None):
    """(out, err, model, decisions) of mode 1 over the calls; decisions: (first sample, accepted, |phase difference|,
    |frequency difference|) of every speculated chunk."""
    m = Model(lp, 1, mutant)
    outs, errs, dec = [], [], []
    pos = 0
    for n in lengths:
        o, e = m.process(x[pos:pos + n])
        outs.append(o)
        errs.append(e)
        if n >= 2 * lp.L:
            dec += [(pos + c * lp.L, ok, dp, df) for c, (ok, dp, df) in enumerate(m.decisions) if c > 0]
        pos += n
    return np.concatenate(outs), np.concatenate(errs), m, dec


def check(lp, x, lengths, ref, got, locked):
    """The assertions of the verified form, as a dict of name -> passed, plus the measured numbers: got = run_verified
    (or the GPU's out and err with the model's decisions) against ref = mode 0's (out, err)."""
    out, err, m, dec = got
    accepted = [d for d in dec if d[1]]
    tol = out_tol(len(accepted))
    de = float(np.max(np.abs(err.astype(np.float64) - ref[1])))
    do = float(np.max(np.abs(out.astype(np.complex128) - ref[0])))
    first = accepted[0][0] if accepted else len(x)
    res = {"err_tol": de <= ERR_TOL, "out_tol": do <= tol,
           "err_exact_before_first_accept": bool(np.array_equal(err[:first], ref[1][:first]))}
    nums = {"de": de / ERR_TOL, "do": do / tol, "accepted": len(accepted), "reruns": m.reruns, "chunks": m.chunks}
    if locked:
        res["no_reruns"] = m.reruns == 0
        if accepted:
            mp = max(d[2] for d in accepted) / m.dphi
            mf = max(d[3] for d in accepted) / m.dfreq
            nums["margin"] = 1.0 / max(mp, mf, 1e-300)
            res["margin_a"] = nums["margin"] >= 4.0
    print(nums, res)
    return res, nums
