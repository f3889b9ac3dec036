"""The verified chunk-parallel PLL model of tests/pll_verify_ref.py on the CPU, against the sequential model (mode 0):
for the stereo, RDS and AM-synchronous loops, on locked pilots and on inputs the lead-in cannot follow (zeros, noise,
gaps), mode 1 is within ERR_TOL / out_tol of mode 0 from the first sample, its err equals mode 0's bit for bit up to
the first accepted chunk, locked input re-runs nothing, the thresholds keep their margins, and every mutant of the
verify pass fails at least one of these checks."""
import numpy as np
import pytest

from tests import pll_ref as R
from tests import pll_verify_ref as V

LOCKED = ("clean", "noisy", "offset", "drift")
UNLOCKED = ("zeros_pilot", "gap", "noise_pilot", "pilot_noise_pilot", "zeros", "noise", "freq_step")
# a carrier-recovery loop centred on 0 Hz: phi rotates slowly, so a lead-in's atan2f guess sits 2 pi from the true
# branch on about half the chunks (what the wrap of the phase difference is for)
BASEBAND = (1000.0, -100.0, 100.0, 1.0, 48000.0)


def loop(name):
    return R.Loop(*(BASEBAND if name == "baseband" else R.LOOPS[name]))


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
        return R.pilot(lp, sum(lengths), kind, seed=seed), lengths
    n = 6 * L + 3
    if kind in ("zeros", "noise"):
        return R.pilot(lp, n, kind, seed=seed), [n]
    if kind == "freq_step":
        bw, fmin, fmax, _, rate = lp.args
        centre, half = 0.5 * (fmin + fmax), 0.5 * (fmax - fmin)
        step = 3 * L - lp.W // 10
        f = np.where(np.arange(n) < step, centre + 0.9 * half, centre - 0.9 * half)
        ph = np.concatenate([[0.0], np.cumsum(2 * np.pi * f / rate)[:-1]])
        return np.exp(1j * (np.mod(ph, 2 * np.pi) + 0.4)).astype(np.complex64), [n]
    x = R.pilot(lp, n, "noisy", seed=seed)
    gap, pos = (5 * L // 2 - lp.W // 20, 3 * L // 2) if kind == "gap" else (5 * L // 2, 0) if kind == "zeros_pilot" else (2 * L, 0) if kind == "noise_pilot" else (2 * L, 2 * L)
    fill = np.zeros(gap, np.complex64) if kind in ("gap", "zeros_pilot") else R.pilot(lp, gap, "noise", seed=seed + 1)
    x[pos:pos + gap] = fill
    return x, [len(x)]


def run_verified(lp, x, lengths, mutant=None):
    m = V.VerifiedModel(lp, mutant)
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


def run_sequential(lp, x):
    return R.Model(lp, 0).process(x)


def check(lp, x, lengths, ref, got, locked):
    """The assertions of the verified form, as a dict of name -> passed, plus the measured numbers."""
    out, err, m, dec = got
    accepted = [d for d in dec if d[1]]
    tol = R.out_tol(len(accepted))
    de = float(np.max(np.abs(err.astype(np.float64) - ref[1])))
    do = float(np.max(np.abs(out.astype(np.complex128) - ref[0])))
    first = accepted[0][0] if accepted else len(x)
    res = {"err_tol": de <= R.ERR_TOL, "out_tol": do <= tol,
           "err_exact_before_first_accept": bool(np.array_equal(err[:first], ref[1][:first]))}
    nums = {"de": de / R.ERR_TOL, "do": do / tol, "accepted": len(accepted), "reruns": m.reruns, "chunks": m.chunks}
    if locked:
        res["no_reruns"] = m.reruns == 0
        if accepted:
            mp = max(d[2] for d in accepted) / m.dphi
            mf = max(d[3] for d in accepted) / m.dfreq
            nums["margin"] = 1.0 / max(mp, mf, 1e-300)
            res["margin_a"] = nums["margin"] >= 4.0
    print(nums, res)
    return res, nums


@pytest.mark.parametrize("kind", LOCKED + UNLOCKED)
@pytest.mark.parametrize("name", list(R.LOOPS))
def test_verified_model_against_sequential(name, kind):
    lp = loop(name)
    x, lengths = make_input(lp, kind)
    ref = run_sequential(lp, x)
    got = run_verified(lp, x, lengths)
    res, nums = check(lp, x, lengths, ref, got, kind in LOCKED)
    assert all(res.values()), (res, nums)
    if kind == "zeros":
        assert got[2].reruns == got[2].chunks > 0          # no lead-in gets anywhere on zeros
    if kind in ("gap", "zeros_pilot"):
        assert got[2].reruns >= 2


@pytest.mark.parametrize("name", list(R.LOOPS))
def test_accept_all_misses_on_the_gap(name):
    """The old form (every lead-in accepted) is 0.3 to 2 off mode 0 after the zero gap: the input discriminates."""
    lp = loop(name)
    x, lengths = make_input(lp, "gap")
    ref = run_sequential(lp, x)
    out = run_verified(lp, x, lengths, "accept_all")[0]
    tail = len(x) - lp.L
    do = float(np.max(np.abs(out[tail:].astype(np.complex128) - ref[0][tail:])))
    print("accept-all out difference after the gap %.3g" % do)
    assert do > 1e3 * R.out_tol(10)


@pytest.mark.parametrize("kind", ["clean", "noisy"])
def test_wrap_of_the_phase_difference(kind):
    """On the baseband loop, a locked pilot: nothing is re-run, though about half the lead-ins start 2 pi away."""
    lp = loop("baseband")
    x, lengths = make_input(lp, kind)
    lengths = [lengths[0], 12 * lp.L + 5]
    x = R.pilot(lp, sum(lengths), kind, seed=22)
    got = run_verified(lp, x, lengths)
    res, _ = check(lp, x, lengths, run_sequential(lp, x), got, True)
    assert all(res.values()), res
    assert run_verified(lp, x, lengths, "phase_without_wrap")[2].reruns >= 3


def _corner_deviation(lp, sp, sf):
    """max |dphi_k|, max |dphim_k| of the linearised loop from (sp DPHI, sf DFREQ)."""
    dphi, dfreq = V.thresholds(lp)
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
    lp = loop(name)
    assert V.ERR_BUDGET <= R.ERR_TOL / 4 and V.OUT_BUDGET <= R.out_tol(1) - 2 * R.OUT_ROUND
    for sp in (1.0, -1.0):
        for sf in (1.0, -1.0):
            me, mo = _corner_deviation(lp, sp, sf)
            assert me <= V.ERR_BUDGET * (1 + 1e-9) and mo <= V.OUT_BUDGET * (1 + 1e-9), (me, mo)
    # the model: the sequential recurrence on a locked pilot, from the true state and from it moved to the corner
    n1 = min(lp.L, lp.W + 8000)
    x = R.pilot(lp, n1 + 20 * lp.W, "clean", seed=23)
    m = R.Model(lp, 0)
    m.process(x[:n1])
    dphi, dfreq = V.thresholds(lp)
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
        lp = loop(name)
        dphi, dfreq = V.thresholds(lp)
        assert dphi / lp.alpha == pytest.approx(dfreq / lp.beta, rel=1e-12)
        offset = 2 * np.pi * 0.3 / lp.args[4]
        assert dfreq < offset / 100, (name, dfreq, offset)


# each mutant and an input on which it shows
MUTANT_INPUTS = {
    "accept_all": ("am_sync", "gap"),
    "rerun_from_speculated": ("rds", "gap"),
    "t_from_speculated_end": ("am_sync", "zeros_pilot"),
    "stale_dP": ("rds", "gap"),
    "stale_freq0": ("rds", "gap"),
    "phase_without_wrap": ("baseband", "clean"),
}


@pytest.mark.parametrize("mutant", V.VERIFY_MUTANTS)
def test_every_mutant_is_caught(mutant):
    name, kind = MUTANT_INPUTS[mutant]
    lp = loop(name)
    x, lengths = make_input(lp, kind)
    if name == "baseband":
        lengths = [lengths[0], 12 * lp.L + 5]
        x = R.pilot(lp, sum(lengths), kind, seed=22)
    res, nums = check(lp, x, lengths, run_sequential(lp, x), run_verified(lp, x, lengths, mutant), kind in LOCKED)
    assert not all(res.values()), (mutant, res, nums)
