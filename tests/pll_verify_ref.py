"""Model of PLLBlock's verified chunk-parallel form (aux_blocks.cu: pll_sim_kernel, pll_verify_kernel, pll_out_kernel;
lrb200_pll_set_mode(q, 1)), its acceptance thresholds and deliberately wrong variants ("mutants").

The sim pass of tests/pll_ref.py speculates: every chunk c >= 1 starts from phi = atan2f(x[c L - W]) and the centre
frequency and runs a W-sample lead-in, assuming that this reaches the loop's true trajectory.  It does not when the
input gives the loop nothing to pull with (zeros) or when the loop is not locked (noise, acquisition).  The verified form
records each chunk's speculated start (phi0, freq0) and checks it, in stream order, against the true state T:

  * chunk 0: T is the carried state (chunk 0 starts from it, so it is always accepted);
  * chunk c >= 1: T is chunk c - 1's final (phi_end, freq_end), after any re-run of chunk c - 1.

Chunk c is accepted when |wrap(T.phi - phi0_c)| <= DPHI and |T.freq - freq0_c| <= DFREQ, the phase difference taken
modulo 2 pi (phi wraps at +-2 pi, and a lead-in that starts from atan2f lands on either branch).  Otherwise it is
re-run from T over its own samples with the sequential recurrence: err is rewritten, freq0 = T.freq, phi0 = T.phi and
dP, phi_end, freq_end are recomputed.  A re-run chunk is the sequential form's, bit for bit, whenever T is (so err equals
mode 0's on every sample before the first accepted chunk).  The base prefix and the out pass are those of pll_ref.

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
most 1.22 alpha eps and 0.57 beta eps over the inputs of test_pll_ref.py and test_pll_verify_ref.py).  s is the largest
that keeps a chunk starting at the box's corner within ERR_BUDGET = ERR_TOL / 4 in error and OUT_BUDGET = out_tol(1) - 2
OUT_ROUND = 3.84e-7 in out (the two output roundings of any comparison are already in out_tol):

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

The GPU's PllBlock computes the same gains and thresholds in double (aux_blocks.cu, pll_thresholds)."""
import math

import numpy as np

from tests.pll_ref import ERR_TOL, OUT_ROUND, OUT_TOL_CHUNK, TWO_PI, Loop, Model, _detect, _wrap, out_tol, pilot  # noqa: F401

ERR_BUDGET = 2.5e-7                  # ERR_TOL / 4
OUT_BUDGET = 3.84e-7                 # out_tol(1) - 2 OUT_ROUND (3.849e-7), rounded down
VERIFY_MUTANTS = ("accept_all", "rerun_from_speculated", "t_from_speculated_end", "stale_dP", "stale_freq0",
                  "phase_without_wrap")


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


class VerifiedModel(Model):
    """PLLBlock's verified mode 1, call by call.  After each parallel call `decisions` lists every chunk's
    (accepted, |phase difference|, |frequency difference|); `chunks` and `reruns` count the speculated chunks (each
    call's chunks after the first) and how many of them were re-run since create or reset, as lrb200_pll_chunk_counts."""

    def __init__(self, loop, mutant=None):
        assert mutant is None or mutant in VERIFY_MUTANTS, mutant
        super().__init__(loop, 1)
        self.vmutant = mutant
        self.dphi, self.dfreq = thresholds(loop)

    def reset(self):
        super().reset()
        self.chunks, self.reruns, self.decisions = 0, 0, []

    def _rerun(self, x, phi, freq):
        """The chunk from (phi, freq) with the sequential recurrence: (err, dP, phi_end, freq_end)."""
        keep = self.phi, self.phim, self.freq
        self.phi, self.phim, self.freq = phi, 0.0, freq
        _, err = self._sequential(x)
        r = err, self.phim, self.phi, self.freq
        self.phi, self.phim, self.freq = keep
        return r

    def _parallel(self, x):
        lp, mut = self.loop, self.vmutant
        n, L, W = len(x), lp.L, lp.W
        nch = (n + L - 1) // L
        starts = np.arange(nch) * L
        ends = np.minimum(starts + L, n)
        xr, xi = x.real.astype(np.float64), x.imag.astype(np.float64)
        err = np.zeros(n, np.float32)
        # sim (pll_sim_kernel): lead-ins, then every chunk over its own samples
        phi = np.empty(nch)
        freq = np.full(nch, lp.centre)
        phi[0], freq[0] = self.phi, self.freq
        if nch > 1:
            b = starts[1:] - W
            phi[1:] = np.arctan2(x.imag[b], x.real[b]).astype(np.float64)
            for t in range(W):
                e = _detect(xr[b + t], xi[b + t], phi[1:])
                f = freq[1:] + lp.beta * e
                phi[1:] = _wrap(phi[1:] + f + lp.alpha * e)
                freq[1:] = np.clip(f, lp.fmin, lp.fmax)
        phi0, freq0 = phi.copy(), freq.copy()
        dP = np.zeros(nch)
        span = int(np.max(ends - starts))
        for t in range(span):
            act = starts + t < ends
            idx = np.where(act, starts + t, 0)
            e = _detect(xr[idx], xi[idx], phi)
            f = freq + lp.beta * e
            err[idx[act]] = e[act]
            phi = np.where(act, _wrap(phi + f + lp.alpha * e), phi)
            dP = np.where(act, _wrap(dP + f * lp.mult + lp.alpha * e), dP)
            freq = np.where(act, np.clip(f, lp.fmin, lp.fmax), freq)
        phi_end, freq_end = phi.copy(), freq.copy()
        spec_end = phi_end.copy(), freq_end.copy()
        # verify and prefix (pll_verify_kernel), in stream order
        decisions = []
        Tphi, Tfreq = self.phi, self.freq
        for c in range(nch):
            if c > 0:
                Tphi, Tfreq = (spec_end[0][c - 1], spec_end[1][c - 1]) if mut == "t_from_speculated_end" else (phi_end[c - 1], freq_end[c - 1])
            d = Tphi - phi0[c]
            dp = abs(d if mut == "phase_without_wrap" else float(wrap_diff(d)))
            df = abs(Tfreq - freq0[c])
            ok = mut == "accept_all" or (dp <= self.dphi and df <= self.dfreq)
            decisions.append((ok, dp, df))
            if ok:
                continue
            s, e_ = int(starts[c]), int(ends[c])
            sphi, sfreq = (phi0[c], freq0[c]) if mut == "rerun_from_speculated" else (Tphi, Tfreq)
            er, dp_new, pe, fe = self._rerun(x[s:e_], sphi, sfreq)
            err[s:e_] = er
            if mut != "stale_dP":
                dP[c] = dp_new
            if mut != "stale_freq0":
                freq0[c] = sfreq
            phi0[c], phi_end[c], freq_end[c] = sphi, pe, fe
        base = np.empty(nch)
        ph = self.phim
        for c in range(nch):
            base[c] = ph
            ph = float(_wrap(np.array(ph + dP[c])))
        self.decisions = decisions
        self.chunks += nch - 1
        self.reruns += sum(not ok for ok, _, _ in decisions[1:])
        # out (pll_out_kernel)
        out = np.zeros(n, np.complex64)
        pm, fr = base.copy(), freq0.copy()
        for t in range(span):
            act = starts + t < ends
            idx = np.where(act, starts + t, 0)
            o = (np.cos(pm).astype(np.float32) + 1j * np.sin(pm).astype(np.float32)).astype(np.complex64)
            out[idx[act]] = o[act]
            e = err[idx].astype(np.float64)
            f = fr + lp.beta * e
            pm = np.where(act, _wrap(pm + f * lp.mult + lp.alpha * e), pm)
            fr = np.where(act, np.clip(f, lp.fmin, lp.fmax), fr)
        self.phi, self.phim, self.freq = float(phi_end[-1]), ph, float(freq_end[-1])
        return out, err
