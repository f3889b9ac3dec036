"""The PLL model of tests/pll_ref.py on the CPU: its sequential mode is O.PLL, the phase rebuild is exact, O.PLL meets the
per-output phase bound, the chunk-parallel model stays within ERR_TOL / out_tol of O.PLL once locked for the receivers'
loop constants, several multipliers, clean, noisy, off-centre and drifting pilots and extreme amplitudes, and every
mutant of the decomposition breaks the bound or a tolerance by more than 3x."""
import math
from fractions import Fraction

import numpy as np
import pytest

from tests import pll_ref as R


def _loop(name, mult=None):
    args = list(R.LOOPS[name])
    if mult is not None:
        args[3] = mult
    return R.Loop(*args)


def _first_call(lp):
    """The acquisition call: sequential (< 2 L), long enough for the loop to lock (W samples)."""
    return min(lp.L, lp.W + 8000)


def _run(lp, x, cuts, mode=1, mutant=None):
    m = R.Model(lp, mode, mutant)
    outs, errs = zip(*[m.process(x[a:b]) for a, b in zip(cuts[:-1], cuts[1:])])
    return np.concatenate(outs), np.concatenate(errs)


def test_sequential_model_is_the_oracle():
    lp = _loop("stereo")
    x = R.pilot(lp, 7000, "noisy", seed=3)
    o, e = _run(lp, x, [0, 1, 2500, 7000], mode=0)
    ro, re_ = lp.oracle().process(x)
    assert np.array_equal(o, ro) and np.array_equal(e, re_)


@pytest.mark.parametrize("fma", [False, True])
def test_rebuild_is_exact(fma):
    """rebuild_phase against fractions.Fraction at a phase offset of 2^30 rad and with every term large (m = 3 on the
    RDS loop): the error is at rounding level of the final float64, far below 1e-9 (the docstring's analysis carries
    it to 2^27 samples)."""
    lp = _loop("rds")
    x = R.pilot(lp, 1500, "noisy", seed=4)
    _, e = lp.oracle().process(x)
    for phase0 in (0.0, 2.0 ** 30 + 0.1234567):
        got = R.rebuild_phase(e, lp, phase0=phase0, fma=fma)
        ref = R.rebuild_phase_exact(e, lp, phase0=phase0, fma=fma)
        d = max(abs(float(Fraction(float(g)) - r)) for g, r in zip(got, ref))
        assert d <= 1e-15, d


def test_freq_prime_is_the_recurrence():
    """freq' from the error stream, through the clamp, equals the recurrence run sample by sample."""
    lp = _loop("stereo")
    k = np.arange(20000)
    e = (0.2 * np.sign(np.sin(2 * np.pi * k / 4000)) + np.random.default_rng(5).uniform(-0.1, 0.1, len(k))).astype(np.float32)
    got = R.freq_prime(e, lp)
    f, ref = lp.centre, []
    for v in e.astype(np.float64):
        f = f + lp.beta * v
        ref.append(f)
        f = min(max(f, lp.fmin), lp.fmax)
    assert np.array_equal(got, np.array(ref))                  # into both clamps and out again
    assert np.any(np.array(ref) > lp.fmax) and np.any(np.array(ref) < lp.fmin)


@pytest.mark.parametrize("kind", ["clean", "noisy", "noise"])
@pytest.mark.parametrize("name", list(R.LOOPS))
def test_oracle_meets_the_phase_bound(name, kind):
    lp = _loop(name)
    x = R.pilot(lp, 40000, kind, seed=6)
    o, e = lp.oracle().process(x)
    r = R.out_ratio(o, R.rebuild_phase(e, lp), R.phase_bound(lp, len(o)))
    print("error / bound %.3g" % r)
    assert r <= 1.0


def _parallel_vs_oracle(lp, kind, amplitude, mutant=None, seed=7, glitch=False):
    """A sequential acquisition call, then one chunk-parallel call of 2 L + 777 samples (3 chunks, the last ragged),
    then a sequential call of 1000.  Returns (|e - e_ref| max, |out - out_ref| max) after the first call.  glitch: the
    samples W / 8 before each chunk boundary are turned by 2.5 rad (a phase guess far off for a lead-in of W / 8)."""
    n1 = _first_call(lp)
    n2 = 2 * lp.L + 777
    x = R.pilot(lp, n1 + n2 + 1000, kind, amplitude, seed=seed)
    if glitch:
        at = n1 + np.arange(1, 3) * lp.L - lp.W // 8
        x[at] *= np.complex64(np.exp(2.5j))
    o, e = _run(lp, x, [0, n1, n1 + n2, n1 + n2 + 1000], mutant=mutant)
    ro, re_ = lp.oracle().process(x)
    if mutant == "unreduced_prefix":
        # the mutant's phase starts m A_OFFSET further on: compare with the oracle turned by the same angle
        off = Fraction(lp.mult) * Fraction(R.A_OFFSET)
        off -= math.floor(off / R.TWO_PI_FRAC) * R.TWO_PI_FRAC
        ro[n1:] = (ro[n1:].astype(np.complex128) * np.exp(1j * float(off))).astype(np.complex64)
    assert np.array_equal(e[:n1], re_[:n1]) and np.array_equal(o[:n1], ro[:n1])      # the exact first call
    de = float(np.max(np.abs(e[n1:].astype(np.float64) - re_[n1:])))
    do = float(np.max(np.abs(o[n1:].astype(np.complex128) - ro[n1:])))
    return de, do


CASES = ([(name, m, "clean", 1.0) for name in R.LOOPS for m in (1.0, 2.0, 3.0, 0.25, -1.0)]
         + [(name, None, kind, 1.0) for name in R.LOOPS for kind in ("noisy", "offset", "drift")]
         + [(name, None, "clean", a) for name in R.LOOPS for a in (1e-3, 1e3)])


@pytest.mark.parametrize("name,mult,kind,amplitude", CASES)
def test_parallel_model_meets_the_tolerance(name, mult, kind, amplitude):
    lp = _loop(name, mult)
    de, do = _parallel_vs_oracle(lp, kind, amplitude)
    tol = R.out_tol(R.lead_ins([2 * lp.L + 777], lp))
    print("err %.3g of ERR_TOL, out %.3g of out_tol" % (de / R.ERR_TOL, do / tol))
    assert de <= R.ERR_TOL and do <= tol


def test_parallel_model_over_many_chunks():
    """A noisy RDS stream of two parallel calls, 41 chunks in all: the out difference grows with the lead-ins and stays
    within out_tol."""
    lp = _loop("rds")
    n1, calls = _first_call(lp), [20 * lp.L + 3, 21 * lp.L - 1]
    x = R.pilot(lp, n1 + sum(calls), "noisy", seed=8)
    o, e = _run(lp, x, list(np.cumsum([0, n1] + calls)))
    ro, re_ = lp.oracle().process(x)
    de = float(np.max(np.abs(e[n1:].astype(np.float64) - re_[n1:])))
    do = float(np.max(np.abs(o[n1:].astype(np.complex128) - ro[n1:])))
    tol = R.out_tol(R.lead_ins(calls, lp))
    print("err %.3g of ERR_TOL, out %.3g of out_tol" % (de / R.ERR_TOL, do / tol))
    assert de <= R.ERR_TOL and do <= tol


# each mutant and an input on which it shows
MUTANT_INPUTS = {
    "unreduced_prefix": ("stereo", "clean"),
    "base_one_chunk_late": ("rds", "clean"),
    "phim0_after_call": ("rds", "clean"),
    "short_lead_in": ("rds", "glitch"),
    "centre_freq_in_out_pass": ("rds", "offset"),
    "no_e_term": ("rds", "noisy"),
    "last_end_start_plus_L": ("rds", "clean"),
}


def test_full_lead_in_is_not_disturbed_by_the_glitch():
    lp = _loop("rds")
    de, do = _parallel_vs_oracle(lp, "clean", 1.0, glitch=True)
    assert de <= R.ERR_TOL and do <= R.out_tol(R.lead_ins([2 * lp.L + 777], lp))


@pytest.mark.parametrize("mutant", R.MUTANTS)
def test_every_mutant_is_caught(mutant):
    name, kind = MUTANT_INPUTS[mutant]
    lp = _loop(name)
    de, do = _parallel_vs_oracle(lp, "clean" if kind == "glitch" else kind, 1.0, mutant=mutant, glitch=kind == "glitch")
    tol = R.out_tol(R.lead_ins([2 * lp.L + 777], lp))
    worst = max(de / R.ERR_TOL, do / tol)
    print("%s: err %.3g of ERR_TOL, out %.3g of out_tol" % (mutant, de / R.ERR_TOL, do / tol))
    assert worst > 3.0
