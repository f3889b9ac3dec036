"""Geometry model, float64 references, per-output error bounds and deliberately wrong references ("mutants") for the
overlap-save FIR kernels (fir_fft.cu: fir_fft1024_kernel, fir_fft_fdl_kernel) and the direct kernels that take over
from them (fir_direct.cu fir_generic_kernel, poly_generic.cu).

Geometry.  `FirModel` makes the choices FirBlock::path / launch_fft / launch_fdl_pc make, call by call: which
path runs, the blocks it cuts and how many kernels it launches (1 for the history update when M > 1, then per
(partition group) launch +1 for edge work and +1 for interior blocks, or +1 for a direct kernel that has outputs).  A
graph in device mode launches nothing of its own (graph.cu run_device only calls the stages), so the per-call count
of lrb200_launch_count() is the model's count.

References are float64 from the float32 taps and samples, starting at the seek index n0 with zero history
(tests/fir_shape_ref.py).  Hilbert: real part = x delayed by (M-1)/2 (integer division), imaginary part = the taps.

Bound of an overlap-save output o.  With u = 2^-24, w the inputs of o's block (single block: [b per - (M-1),
(b+1) per), which is both packed sub-blocks for real input; delay line: [512 (b-P), 512 (b+1))), clipped to the call
(the kernel reads zeros past n), and H_p the 1024-point DFT of the p-th 512-tap slice (all taps for a single block,
delay + j hilbert for the Hilbert transform):

    |got - ref| <= C u ||x_w||_2 sum_p ||H_p||_inf + S u |ref_o| (+ 2 pi (n0 + o) 2^-64 sum_k |h_k| |x_{o-k}|)

Derivation (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., Thm 24.2 and Lemma 3.5).  A radix-2
stage with computed weights |w^ - w| <= mu has normwise error eta = mu + gamma_4 (sqrt2 + mu).  The kernel's
butterflies (tools/gen_fft32.py) form a' = a + w b by two FMAs and b' = 2a - a' by a third, so b' carries the error of
a' plus one rounding: per stage eta' = sqrt2 eta + u.  The twiddle tables are float32 roundings of exact values
(mu = u: the 32-point constants, the 32 x 32 inter-pass table W1024^(a b), E).  The inter-pass twiddle product is one
more stage (mu + sqrt2 gamma_2 <= eta'), the transposes are exact, so a 1024-point transform in 32 x 32 four-step form
is 11 stages: ||X^ - X||_2 <= phi ||X||_2, phi = (1 + eta')^11 - 1, ||X||_2 = sqrt(N) ||x_w||_2.  The spectrum product
with H^ = fl(H / N) (|H^ - H / N| <= u |H / N|) and one complex multiply (sqrt2 gamma_2) gives
||Y^ - Y||_2 <= psi (||H||_inf / N) sqrt(N) ||x_w||_2, psi = phi + (1 + phi)(u + (1 + u) a), a = sqrt2 gamma_2; the
unscaled inverse transform has norm sqrt(N) and adds phi ||Y^||_2, so a block's error vector, hence each of its
outputs, is within (psi + phi (1 + psi)) ||H||_inf ||x_w||_2.  The delay line sums pc <= 4 products per launch by
2 pc FMAs (a = sqrt2 gamma_(2 pc + 1)) over sum_p ||H_p||_inf ||x_(b-p)||_2 <= sum_p ||H_p||_inf ||x_w||_2, and each
later launch adds its partial sum into y with one float add (u times the sum of both bounds).  The fused translator
multiplies the input by E^ at the load (relative error 2u + sqrt2 gamma_2, carried through the whole chain).  The
store term S u |ref_o| is 4u; with the translator the block phasor P_b adds its 2^-32-turn truncation, sincospif's
rounding (3u) and the multiply (sqrt2 gamma_2).  The last term is the translator's 2^-64-turn fixed-point phase, as
in fir_shape_ref.linear_bound.  C is derived, not fitted: tests/test_fft_fir_ref.py shows that a float32 emulation of
the kernels' arithmetic stays below a quarter of it.

Outputs of calls that ran a direct kernel use fir_shape_ref.linear_bound with T = M (the catch-all sums four
interleaved chains, each shorter than the sequential one the bound assumes)."""
import math
from fractions import Fraction

import numpy as np

from tests import fir_shape_ref as R
from tests import test_gpu_fir_shapes as G
from tests.test_gpu_bounds import fir_ref

U = R.U
FF_N = 1024
HOP = 512
MAXPC = 4
RING_W = 8                   # fir_fft.cu FD_W: warps, hence ring slots beyond the partitions
FFT_MAX_TAPS = 513
PG_MAXT = 960                # poly_generic.cu
SQ2 = math.sqrt(2.0)


def gamma(k):
    return k * U / (1 - k * U)


# ---- what FirBlock decides ----------------------------------------------------------------------------------------
def decim_plan(consumed, D, n):
    f = (D - consumed % D) % D
    return f, ((n - f + D - 1) // D if n > f else 0)


class FirModel:
    """FirBlock's choices for one stage: kind in crcf / cccf / rrrf / hilbert, M taps, fused decimation D, a fused
    translator (rotate), algo in auto / direct / fft."""

    def __init__(self, kind, M, D=1, rotate=False, algo="auto"):
        self.kind, self.M, self.D, self.rotate, self.algo = kind, M, D, rotate, algo
        if kind == "crcf" and not rotate:
            self.poly = (D == 1 and M <= 32) or (D == 5 and 65 < M <= 128)
        else:
            self.poly = kind == "rrrf" and D == 5 and 130 < M <= 135
        self.gen_poly = (not rotate and D in G.PG_DS and kind != "hilbert" and
                         -(-M // D) * D * (2 if kind == "cccf" else 1) <= PG_MAXT and G.pg_supports(kind, M, D))
        long_filter = M > FFT_MAX_TAPS
        self.fast = not (kind == "hilbert" and D != 1) and not (
            long_filter and not (kind in ("crcf", "cccf") and D == 1 and not rotate and M <= 16 * 512))
        self.part_taps = 512 if long_filter else M
        self.nparts = -(-M // 512) if long_filter else 1
        self.L = FF_N - (self.part_taps - 1)
        self.per = 2 * self.L if kind == "rrrf" else self.L

    def effective(self):
        if self.rotate:
            return "fft"
        if not self.fast or self.algo == "direct":
            return "direct"
        if self.algo == "fft":
            return "fft"
        if self.poly:
            return "direct"
        per_tap = 2.0 if self.kind == "cccf" else (1.0 if self.kind == "crcf" else (1.0 if self.gen_poly else 0.5))
        direct_cost = (3.0 if self.gen_poly else 8.0) * per_tap * self.M / self.D
        fft_cost = self.nparts * 31.0 * FF_N / self.L * (0.5 if self.kind == "rrrf" else 1.0)
        return "fft" if direct_cost > fft_cost else "direct"

    def plan(self, n, consumed):
        """(path, launches, geometry) of one call of n > 0 inputs after `consumed`; path is fft, fdl, poly_generic
        or direct (the catch-all); geometry the (b_lo, b_hi, nblocks) of each launch group."""
        assert n > 0
        if self.poly and self.algo != "fft":
            raise NotImplementedError("the register-tiled polyphase kernels are tests/test_gpu_fir_shapes.py's")
        _, no = decim_plan(consumed, self.D, n)
        hist = 1 if self.M > 1 else 0
        eff = self.effective()
        if self.gen_poly and eff == "direct":
            return "poly_generic", hist + (no > 0), []
        if not self.fast or eff != "fft" or (self.algo != "fft" and not self.rotate and n < 8 * self.L):
            return "direct", hist + (no > 0), []
        launches, geo = hist, []
        if self.nparts > 1:
            nb = -(-n // HOP)
            for p0 in range(0, self.nparts, MAXPC):
                pc = min(MAXPC, self.nparts - p0)
                b_lo = min(nb, pc + p0)
                b_hi = min(max(b_lo, n // HOP), nb)
                launches += (b_lo > 0 or nb > b_hi) + (b_hi > b_lo)
                geo.append((b_lo, b_hi, nb))
            return "fdl", launches, geo
        per = self.per
        nblocks = -(-n // per)
        b_lo = max(1, -(-(self.M - 1) // per))
        b_hi = min(nblocks, n // per)
        b_hi = max(b_hi, b_lo)
        if b_lo > nblocks:
            b_lo = b_hi = nblocks
        launches += (b_lo + nblocks - b_hi > 0) + (b_hi > b_lo)
        return "fft", launches, [(b_lo, b_hi, nblocks)]


# ---- taps, references ---------------------------------------------------------------------------------------------
def effective_taps(kind, h):
    """The taps the transform multiplies by: delay + j hilbert for the Hilbert transform."""
    if kind != "hilbert":
        return np.asarray(h)
    e = 1j * np.asarray(h, np.float64)
    e[(len(h) - 1) // 2] += 1.0
    return e


def full_ref(kind, h, x, turns, n0, delay=None):
    """Full-rate float64 output of [Translator ->] FIR / Hilbert over x from zero history (Hilbert: the real part is x
    delayed by `delay`, (M-1)/2 by default)."""
    x = np.asarray(x)
    if kind == "hilbert":
        d = (len(h) - 1) // 2 if delay is None else delay
        re = np.concatenate([np.zeros(d), x.astype(np.float64)])[:len(x)]
        return re + 1j * (fir_ref(h, x, wide=True) if len(h) else 0.0)
    if not len(h):
        return np.zeros(len(x), np.complex128 if np.iscomplexobj(x) or turns is not None else np.float64)
    return fir_ref(h, R.rotate(x, turns, n0) if turns is not None else x, wide=True)


def spectrum_norms(kind, h, nparts):
    """||H_p||_inf of the 1024-point DFTs of the 512-tap slices (one slice: all taps)."""
    he = effective_taps(kind, h).astype(np.complex128)
    if nparts == 1:
        return [float(np.max(np.abs(np.fft.fft(he, FF_N))))]
    return [float(np.max(np.abs(np.fft.fft(he[p * HOP:(p + 1) * HOP], FF_N)))) for p in range(nparts)]


def c_factor(nparts=1, rotate=False):
    """C of the overlap-save bound (module docstring)."""
    eta = U + gamma(4) * (SQ2 + U)
    eta2 = SQ2 * eta + U
    phi = (1 + eta2) ** 11 - 1
    a = SQ2 * gamma(2 * min(nparts, MAXPC) + 1) if nparts > 1 else SQ2 * gamma(2)
    psi = phi + (1 + phi) * (U + (1 + U) * a)
    c = psi + phi * (1 + psi)
    groups = -(-nparts // MAXPC)
    c += (groups - 1) * U * (1 + c) * 2
    if rotate:
        c = (1 + 2 * U + SQ2 * gamma(2)) * (1 + c) - 1
    return c / U


def store_factor(rotate):
    return 4.0 + ((2 * math.pi * 2.0 ** -32 + 3 * U + SQ2 * gamma(2)) / U if rotate else 0.0)


# ---- one case: a stage and its streams ------------------------------------------------------------------------------
class Case:
    """kind, float32 taps h (complex64 for cccf), fused decimation D, translator turns (None: none), algo, and the
    streams [(n0, [call lengths])] run through it; sig / seed / burst make the input."""

    def __init__(self, name, kind, h, D=1, turns=None, algo="fft", streams=(), sig="noise", seed=0, burst=None):
        self.name, self.kind, self.h, self.D, self.turns, self.algo = name, kind, np.asarray(h), D, turns, algo
        self.M = len(h)
        self.model = FirModel(kind, self.M, D, turns is not None, algo)
        self.streams, self.sig, self.seed = list(streams), sig, seed
        self.cplx_in = kind in ("crcf", "cccf")
        self.cplx_out = kind != "rrrf"
        self.burst = burst or burst_length(self.model)

    def gen(self, n):
        return signal(self.sig, n, self.seed, self.cplx_in, self.burst)

    def plans(self, n0, calls):
        out, consumed = [], n0
        for n in calls:
            out.append(self.model.plan(n, consumed))
            consumed += n
        return out

    def full(self, x, n0, h=None, turns=0):
        """the stage's full-rate output; h, turns: wrong taps or translator (the Hilbert delay stays (M-1)/2)"""
        return full_ref(self.kind, self.h if h is None else h, x, self.turns if turns == 0 else turns, n0,
                        (self.M - 1) // 2)

    def kept(self, n0, n, phase=0):
        return R.kept(n0, self.D, n, phase)

    def expect(self, x, n0, calls):
        """Float64 reference of the stream's outputs, their bounds, and the index of the call each belongs to."""
        total = len(x)
        assert sum(calls) == total
        ref_full = self.full(x, n0)
        bound = np.zeros(total)
        callno = np.zeros(total, np.int64)
        ax = np.abs(np.asarray(x).astype(np.complex128))
        csum = np.concatenate([[0.0], np.cumsum(ax * ax)])
        m = self.model
        hnorm = spectrum_norms(self.kind, self.h, m.nparts) if m.fast else None
        direct = np.zeros(total, bool)
        s = 0
        for c, ((path, _, _), n) in enumerate(zip(self.plans(n0, calls), calls)):
            callno[s:s + n] = c
            o = np.arange(n)
            if path in ("fft", "fdl"):
                if path == "fft":
                    b = o // m.per
                    lo, hi = b * m.per - (self.M - 1), (b + 1) * m.per
                else:
                    b = o // HOP
                    lo, hi = HOP * (b - m.nparts), HOP * (b + 1)
                lo = np.clip(s + lo, 0, total)
                hi = np.clip(s + np.minimum(hi, n), 0, total)
                xw = np.sqrt(np.maximum(csum[hi] - csum[lo], 0.0))
                bound[s:s + n] = (c_factor(m.nparts, m.rotate) * U * xw * sum(hnorm) +
                                  store_factor(m.rotate) * U * np.abs(ref_full[s:s + n]))
                if self.turns is not None:
                    S = np.maximum(fir_ref(np.abs(self.h.astype(np.complex128)), ax, wide=True), 0.0)[s:s + n]
                    bound[s:s + n] += 2 * np.pi * (n0 + s + o) * 2.0 ** -64 * S
            else:
                direct[s:s + n] = True
            s += n
        if direct.any():
            idx = np.flatnonzero(direct)
            bound[idx] = R.linear_bound(self.h, ax, idx, n0, self.M, self.D)
        k = self.kept(n0, total)
        ref = ref_full[k]
        if self.kind == "rrrf":
            ref = ref.real
        return ref, bound[k], callno[k], k

    # ---- mutants
    def mutants(self, x, n0, calls):
        """Wrong references of the stream (kept outputs), each left out only where it equals the truth by
        construction."""
        x = np.asarray(x)
        h, M, D, turns, m = self.h, self.M, self.D, self.turns, self.model
        total = len(x)
        k = self.kept(n0, total)
        fix = (lambda y: y.real) if self.kind == "rrrf" else (lambda y: y)
        out = {}
        for name, hm in R._mutant_taps(h).items():
            out[name] = fix(self.full(x, n0, hm)[k])
        full = self.full(x, n0)
        if D > 1:
            for sgn in (1, -1):
                out["decimation phase %+d" % sgn] = fix(full[self.kept(n0, total, sgn)])
        single = np.count_nonzero(h) == 1          # (one tap: only the kept samples' own phases, whole turns at 2 D turns)
        if R._conj_visible(h, turns, D, None) and not (single and abs((2 * D * turns + 0.5) % 1 - 0.5) < 1e-12):
            out["conjugated translator"] = self.full(x, n0, turns=-turns)[k]
        plans = self.plans(n0, calls)

        def past(at):
            """the M-1 inputs before stream index `at` (zeros before the stream)"""
            return np.concatenate([np.zeros(max(0, M - 1 - at), x.dtype), x[max(0, at - (M - 1)):at]])

        starts = np.concatenate([[0], np.cumsum(calls)[:-1]]).astype(int)
        if turns is not None:
            # (left out when the neighbour's phasor is the block's own: turns per whole turns, or below the bound's
            # resolution, as for the discriminator in fir_shape_ref._conj_visible: the 1e-9-turn offset)
            step = float((Fraction(turns) * m.per) % 1)
            for sgn in (1, -1):
                if 2 * np.pi * min(step, 1 - step) > 1e-3:
                    y = full.copy()
                    for (path, _, _), s, n in zip(plans, starts, calls):
                        if path == "fft":
                            y[s:s + n] *= np.exp(2j * np.pi * sgn * float((Fraction(turns) * m.per) % 1))
                    out["block phasor of block %+d" % sgn] = y[k]
        if np.count_nonzero(effective_taps(self.kind, h)[1:]):          # (a filter without memory ignores history)
            def with_history(hist_of):
                y = full.copy()
                for c, (s, n) in enumerate(zip(starts, calls)):
                    seg = np.concatenate([hist_of(c, s), x[s:s + n]])
                    y[s:s + n] = full_ref(self.kind, h, seg, turns, n0 + s - (M - 1))[M - 1:]
                return y

            zero = np.zeros(M - 1, x.dtype)
            out["history zeroed at each call"] = fix(with_history(lambda c, s: zero)[k])
            if len(calls) > 1:
                out["history one call stale"] = fix(with_history(lambda c, s: past(starts[c - 1] if c else 0))[k])
        if self.kind == "rrrf" and any(p[0] == "fft" for p in plans):
            y = full.copy()
            L = m.L
            for (path, _, _), s, n in zip(plans, starts, calls):
                if path != "fft":
                    continue
                nb = -(-n // m.per)
                seg = np.concatenate([past(s), x[s:s + n],
                                      np.zeros(nb * m.per - n, x.dtype)])
                yc = full_ref(self.kind, h, seg, None, 0)[M - 1:].reshape(nb, 2, L)[:, ::-1].reshape(-1)
                y[s:s + n] = yc[:n]
            out["packed-real lanes swapped"] = y.real[k]
        if self.kind == "hilbert":
            d = (M - 1) // 2
            for sgn in (1, -1):
                if d + sgn >= 0:
                    re = np.concatenate([np.zeros(d + sgn), x.astype(np.float64)])[:total]
                    out["hilbert delay %+d" % sgn] = (re + 1j * full.imag)[k]
        if m.nparts > 1:
            P = m.nparts
            sl = [h[p * HOP:(p + 1) * HOP] for p in range(P)]

            def build(pieces):
                """taps from (slice, delay) pairs"""
                n_t = max(d + len(t) for t, d in pieces) if pieces else 1
                hm = np.zeros(n_t, h.dtype)
                for t, d in pieces:
                    hm[d:d + len(t)] += t
                return hm

            cand = {}
            for p in sorted({0, P - 1}):
                cand["partition %d dropped" % p] = build([(sl[q], q * HOP) for q in range(P) if q != p])
            for sgn in (1, -1):
                cand["partitions one block %s" % ("early" if sgn > 0 else "late")] = build(
                    [(sl[0], 0)] + [(sl[q], (q - sgn) * HOP) for q in range(1, P)])
            if P > MAXPC:
                g0 = (P - 1) // MAXPC * MAXPC
                cand["later launch overwrites"] = build([(sl[q], q * HOP) for q in range(g0, P)])
            late = []
            for q in range(P):
                pc = min(MAXPC, P - q // MAXPC * MAXPC)
                late.append((sl[q], (q + (RING_W + pc - 1 if q % MAXPC else 0)) * HOP))
            if any(q % MAXPC for q in range(P)):
                cand["delay line one ring revolution late"] = build(late)
            for name, hm in cand.items():
                ht = np.concatenate([h, np.zeros(max(0, len(hm) - M), h.dtype)])
                hz = np.concatenate([hm, np.zeros(max(0, M - len(hm)), h.dtype)])
                if not np.array_equal(ht, hz):
                    out[name] = self.full(x, n0, hm)[k]
        return out


# ---- inputs -----------------------------------------------------------------------------------------------------------
def window_length(model):
    if model.nparts > 1:
        return HOP * (model.nparts + 1)
    return model.per + model.M - 1


def burst_length(model):
    """Bursty inputs step by 60 dB every B samples: B >= 3 windows and not a multiple of the block length or 512, so
    whole windows are quiet, some sit right after loud ones, and a quiet call inherits a loud history."""
    B = 3 * window_length(model) + 37
    while B % model.per == 0 or B % HOP == 0:
        B += 1
    return B


def signal(kind, n, seed, cplx, burst):
    if kind != "bursty":
        return G.signal(kind, n, seed, cplx)
    x = G.signal("noise", n, seed, cplx)
    return (x * np.where((np.arange(n) // burst) % 2 == 0, 1.0, 1e-3)).astype(x.dtype)


def call_list(model, long_call=True):
    """1, 2, M-2, M-1, M (the history assembled over several short calls), per-1, per, per+1, k per +- 1 with >= 2
    interior blocks, 8L-1, 8L, 8L+1 (the AUTO switch), one long call (>= 1 Mi inputs, 4 Mi for the delay line) and a
    short tail."""
    M, per, L = model.M, (HOP if model.nparts > 1 else model.per), model.L
    k = (M - 1) // per + 4
    calls = [1, 2] + [c for c in (M - 2, M - 1, M) if c > 0]
    calls += [per - 1, per, per + 1, 3, k * per - 1, k * per + 1, 8 * L - 1, 8 * L, 8 * L + 1]
    if long_call:
        calls.append((4 if model.nparts > 1 else 1) * (1 << 20) + 13)
    calls.append(777)
    return calls


def excess(got, ref, bound):
    return R.excess(got, ref, bound)
