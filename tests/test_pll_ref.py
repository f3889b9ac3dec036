"""The PLL model of tests/pll_ref.py on the CPU.  Its sequential mode is O.PLL, the phase rebuild is exact and O.PLL meets
the per-output phase bound.  Once locked, the verified chunk-parallel model stays within ERR_TOL / out_tol of O.PLL,
re-running nothing, for the receivers' loop constants, several multipliers, clean, noisy, off-centre and drifting pilots
and extreme amplitudes.  Against the sequential model (mode 0), for the stereo, RDS and AM-synchronous loops, on locked
pilots and on inputs the lead-in cannot follow (zeros, noise, gaps), mode 1 is within ERR_TOL / out_tol from the first
sample, its err equals mode 0's bit for bit up to the first accepted chunk, locked input re-runs nothing and the
thresholds keep their margins.  Every mutant fails one of these checks."""
import math
from fractions import Fraction

import numpy as np
import pytest

from tests import pll_ref as R


def _first_call(lp):
    """The acquisition call: sequential (< 2 L), long enough for the loop to lock (W samples)."""
    return min(lp.L, lp.W + 8000)


def _run(lp, x, cuts, mode=1, mutant=None):
    m = R.Model(lp, mode, mutant)
    outs, errs = zip(*[m.process(x[a:b]) for a, b in zip(cuts[:-1], cuts[1:])])
    return np.concatenate(outs), np.concatenate(errs), m


def test_sequential_model_is_the_oracle():
    lp = R.loop("stereo")
    x = R.pilot(lp, 7000, "noisy", seed=3)
    o, e, _ = _run(lp, x, [0, 1, 2500, 7000], mode=0)
    ro, re_ = lp.oracle().process(x)
    assert np.array_equal(o, ro) and np.array_equal(e, re_)


@pytest.mark.parametrize("fma", [False, True])
def test_rebuild_is_exact(fma):
    """rebuild_phase against fractions.Fraction at a phase offset of 2^30 rad and with every term large (m = 3 on the
    RDS loop): the error is at rounding level of the final float64, far below 1e-9 (the docstring's analysis carries
    it to 2^27 samples)."""
    lp = R.loop("rds")
    x = R.pilot(lp, 1500, "noisy", seed=4)
    _, e = lp.oracle().process(x)
    for phase0 in (0.0, 2.0 ** 30 + 0.1234567):
        got = R.rebuild_phase(e, lp, phase0=phase0, fma=fma)
        ref = R.rebuild_phase_exact(e, lp, phase0=phase0, fma=fma)
        d = max(abs(float(Fraction(float(g)) - r)) for g, r in zip(got, ref))
        assert d <= 1e-15, d


def test_freq_prime_is_the_recurrence():
    """freq' from the error stream, through the clamp, equals the recurrence run sample by sample."""
    lp = R.loop("stereo")
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
    lp = R.loop(name)
    x = R.pilot(lp, 40000, kind, seed=6)
    o, e = lp.oracle().process(x)
    r = R.out_ratio(o, R.rebuild_phase(e, lp), R.phase_bound(lp, len(o)))
    print("error / bound %.3g" % r)
    assert r <= 1.0


def _parallel_vs_oracle(lp, kind, amplitude, mutant=None, seed=7, glitch=False):
    """A sequential acquisition call, then one chunk-parallel call of 2 L + 777 samples (3 chunks, the last ragged),
    then a sequential call of 1000.  Returns (|e - e_ref| max, |out - out_ref| max) after the first call, and the model.  glitch: the
    samples W / 8 before each chunk boundary are turned by 2.5 rad (a phase guess far off for a lead-in of W / 8)."""
    n1 = _first_call(lp)
    n2 = 2 * lp.L + 777
    x = R.pilot(lp, n1 + n2 + 1000, kind, amplitude, seed=seed)
    if glitch:
        at = n1 + np.arange(1, 3) * lp.L - lp.W // 8
        x[at] *= np.complex64(np.exp(2.5j))
    o, e, m = _run(lp, x, [0, n1, n1 + n2, n1 + n2 + 1000], mutant=mutant)
    ro, re_ = lp.oracle().process(x)
    if mutant == "unreduced_prefix":
        # the mutant's phase starts m A_OFFSET further on: compare with the oracle turned by the same angle
        off = Fraction(lp.mult) * Fraction(R.A_OFFSET)
        off -= math.floor(off / R.TWO_PI_FRAC) * R.TWO_PI_FRAC
        ro[n1:] = (ro[n1:].astype(np.complex128) * np.exp(1j * float(off))).astype(np.complex64)
    assert np.array_equal(e[:n1], re_[:n1]) and np.array_equal(o[:n1], ro[:n1])      # the exact first call
    de = float(np.max(np.abs(e[n1:].astype(np.float64) - re_[n1:])))
    do = float(np.max(np.abs(o[n1:].astype(np.complex128) - ro[n1:])))
    return de, do, m


CASES = ([(name, m, "clean", 1.0) for name in R.LOOPS for m in (1.0, 2.0, 3.0, 0.25, -1.0)]
         + [(name, None, kind, 1.0) for name in R.LOOPS for kind in ("noisy", "offset", "drift")]
         + [(name, None, "clean", a) for name in R.LOOPS for a in (1e-3, 1e3)])


@pytest.mark.parametrize("name,mult,kind,amplitude", CASES)
def test_parallel_model_meets_the_tolerance(name, mult, kind, amplitude):
    lp = R.loop(name, mult)
    de, do, m = _parallel_vs_oracle(lp, kind, amplitude)
    tol = R.out_tol(R.lead_ins([2 * lp.L + 777], lp))
    print("err %.3g of ERR_TOL, out %.3g of out_tol, %d re-runs" % (de / R.ERR_TOL, do / tol, m.reruns))
    assert de <= R.ERR_TOL and do <= tol and m.reruns == 0


def test_parallel_model_over_many_chunks():
    """A noisy RDS stream of two parallel calls, 41 chunks in all: the out difference grows with the lead-ins and stays
    within out_tol."""
    lp = R.loop("rds")
    n1, calls = _first_call(lp), [20 * lp.L + 3, 21 * lp.L - 1]
    x = R.pilot(lp, n1 + sum(calls), "noisy", seed=8)
    o, e, m = _run(lp, x, list(np.cumsum([0, n1] + calls)))
    ro, re_ = lp.oracle().process(x)
    de = float(np.max(np.abs(e[n1:].astype(np.float64) - re_[n1:])))
    do = float(np.max(np.abs(o[n1:].astype(np.complex128) - ro[n1:])))
    tol = R.out_tol(R.lead_ins(calls, lp))
    print("err %.3g of ERR_TOL, out %.3g of out_tol, %d re-runs" % (de / R.ERR_TOL, do / tol, m.reruns))
    assert de <= R.ERR_TOL and do <= tol and m.reruns == 0


def test_full_lead_in_is_not_disturbed_by_the_glitch():
    lp = R.loop("rds")
    de, do, m = _parallel_vs_oracle(lp, "clean", 1.0, glitch=True)
    assert de <= R.ERR_TOL and do <= R.out_tol(R.lead_ins([2 * lp.L + 777], lp)) and m.reruns == 0


def run_sequential(lp, x):
    return R.Model(lp, 0).process(x)


@pytest.mark.parametrize("kind", R.LOCKED + R.UNLOCKED)
@pytest.mark.parametrize("name", list(R.LOOPS))
def test_verified_model_against_sequential(name, kind):
    lp = R.loop(name)
    x, lengths = R.make_input(lp, kind)
    ref = run_sequential(lp, x)
    got = R.run_verified(lp, x, lengths)
    res, nums = R.check(lp, x, lengths, ref, got, kind in R.LOCKED)
    assert all(res.values()), (res, nums)
    if kind == "zeros":
        assert got[2].reruns == got[2].chunks > 0          # no lead-in gets anywhere on zeros
    if kind in ("gap", "zeros_pilot"):
        assert got[2].reruns >= 2


@pytest.mark.parametrize("name", list(R.LOOPS))
def test_accept_all_misses_on_the_gap(name):
    """The old form (every lead-in accepted) is 0.3 to 2 off mode 0 after the zero gap: the input discriminates."""
    lp = R.loop(name)
    x, lengths = R.make_input(lp, "gap")
    ref = run_sequential(lp, x)
    out = R.run_verified(lp, x, lengths, "accept_all")[0]
    tail = len(x) - lp.L
    do = float(np.max(np.abs(out[tail:].astype(np.complex128) - ref[0][tail:])))
    print("accept-all out difference after the gap %.3g" % do)
    assert do > 1e3 * R.out_tol(10)


@pytest.mark.parametrize("kind", ["clean", "noisy"])
def test_wrap_of_the_phase_difference(kind):
    """On the baseband loop, a locked pilot: nothing is re-run, though about half the lead-ins start 2 pi away."""
    lp = R.loop("baseband")
    x, lengths = R.make_input(lp, kind)
    lengths = [lengths[0], 12 * lp.L + 5]
    x = R.pilot(lp, sum(lengths), kind, seed=22)
    got = R.run_verified(lp, x, lengths)
    res, _ = R.check(lp, x, lengths, run_sequential(lp, x), got, True)
    assert all(res.values()), res
    assert R.run_verified(lp, x, lengths, "phase_without_wrap")[2].reruns >= 3


def _corner_deviation(lp, sp, sf):
    """max |dphi_k|, max |dphim_k| of the linearised loop from (sp DPHI, sf DFREQ)."""
    dphi, dfreq = R.thresholds(lp)
    p, f, pm, me, mo = sp * dphi, sf * dfreq, 0.0, sp * dphi, 0.0
    for _ in range(200 * lp.W):
        f = f - lp.beta * p
        pm = pm + lp.mult * f - lp.alpha * p
        p = p + f - lp.alpha * p
        me, mo = max(me, abs(p)), max(mo, abs(pm))
    return me, mo


@pytest.mark.parametrize("name", list(R.LOOPS))
def test_threshold_corner_stays_within_the_tolerances(name):
    """(b): a chunk that starts at the thresholds' corner, either sign, stays within ERR_TOL / 4 in error and out_tol(1)
    in out (two output roundings plus the offset's own), in the linearised loop and in the model itself."""
    lp = R.loop(name)
    assert R.ERR_BUDGET <= R.ERR_TOL / 4 and R.OUT_BUDGET <= R.out_tol(1) - 2 * R.OUT_ROUND
    for sp in (1.0, -1.0):
        for sf in (1.0, -1.0):
            me, mo = _corner_deviation(lp, sp, sf)
            assert me <= R.ERR_BUDGET * (1 + 1e-9) and mo <= R.OUT_BUDGET * (1 + 1e-9), (me, mo)
    # the model: the sequential recurrence on a locked pilot, from the true state and from it moved to the corner
    n1 = min(lp.L, lp.W + 8000)
    x = R.pilot(lp, n1 + 20 * lp.W, "clean", seed=23)
    m = R.Model(lp, 0)
    m.process(x[:n1])
    dphi, dfreq = R.thresholds(lp)
    ref = R.Model(lp, 0)
    ref.phi, ref.phim, ref.freq = m.phi, m.phim, m.freq
    o0, e0 = ref.process(x[n1:])
    for sp in (1.0, -1.0):
        for sf in (1.0, -1.0):
            mv = R.Model(lp, 0)
            mv.phi, mv.phim, mv.freq = m.phi + sp * dphi, m.phim, m.freq + sf * dfreq
            o, e = mv.process(x[n1:])
            de = float(np.max(np.abs(e.astype(np.float64) - e0)))
            do = float(np.max(np.abs(o.astype(np.complex128) - o0)))
            print("corner (%+d, %+d): err %.3g of ERR_TOL / 4, out %.3g of out_tol(1)" % (sp, sf, de / (R.ERR_TOL / 4), do / R.out_tol(1)))
            assert de <= R.ERR_TOL / 4 and do <= R.out_tol(1)


def test_thresholds_follow_the_loop_constants():
    """The box is (s alpha, s beta); failed lead-ins (about the pilot's 0.3 Hz offset from the centre) are orders of
    magnitude outside it."""
    for name in R.LOOPS:
        lp = R.loop(name)
        dphi, dfreq = R.thresholds(lp)
        assert dphi / lp.alpha == pytest.approx(dfreq / lp.beta, rel=1e-12)
        offset = 2 * np.pi * 0.3 / lp.args[4]
        assert dfreq < offset / 100, (name, dfreq, offset)


# each mutant and an input on which it shows.  The sim, prefix and out-pass mutants: one parallel call of a locked pilot
# between two sequential ones, against O.PLL (_parallel_vs_oracle)
PASS_MUTANT_INPUTS = {
    "unreduced_prefix": ("stereo", "clean"),
    "base_one_chunk_late": ("rds", "clean"),
    "phim0_after_call": ("rds", "clean"),
    "short_lead_in": ("rds", "glitch"),
    "centre_freq_in_out_pass": ("rds", "offset"),
    "no_e_term": ("rds", "noisy"),
    "last_end_start_plus_L": ("rds", "clean"),
}
# the verify-pass mutants: make_input's inputs, against mode 0 (check)
VERIFY_MUTANT_INPUTS = {
    "accept_all": ("am_sync", "gap"),
    "rerun_from_speculated": ("rds", "gap"),
    "t_from_speculated_end": ("am_sync", "zeros_pilot"),
    "stale_dP": ("rds", "gap"),
    "stale_freq0": ("rds", "gap"),
    "phase_without_wrap": ("baseband", "clean"),
}


@pytest.mark.parametrize("mutant", R.MUTANTS)
def test_every_mutant_is_caught(mutant):
    if mutant in VERIFY_MUTANT_INPUTS:
        name, kind = VERIFY_MUTANT_INPUTS[mutant]
        lp = R.loop(name)
        x, lengths = R.make_input(lp, kind)
        if name == "baseband":
            lengths = [lengths[0], 12 * lp.L + 5]
            x = R.pilot(lp, sum(lengths), kind, seed=22)
        res, nums = R.check(lp, x, lengths, run_sequential(lp, x), R.run_verified(lp, x, lengths, mutant), kind in R.LOCKED)
        assert not all(res.values()), (mutant, res, nums)
        return
    name, kind = PASS_MUTANT_INPUTS[mutant]
    lp = R.loop(name)
    de, do, m = _parallel_vs_oracle(lp, "clean" if kind == "glitch" else kind, 1.0, mutant=mutant, glitch=kind == "glitch")
    tol = R.out_tol(R.lead_ins([2 * lp.L + 777], lp))
    worst = max(de / R.ERR_TOL, do / tol)
    print("%s: err %.3g of ERR_TOL, out %.3g of out_tol, %d re-runs" % (mutant, de / R.ERR_TOL, do / tol, m.reruns))
    if mutant == "short_lead_in":
        # the verify pass repairs it: the W / 8 lead-ins that the glitch throws off miss their predecessors' end states
        # and are run again, so the output stays within tolerance.  The input is a locked pilot, on which the full
        # lead-in re-runs nothing (test_full_lead_in_is_not_disturbed_by_the_glitch): a re-run is the mutant showing.
        assert m.reruns > 0
    else:
        assert worst > 3.0
