"""The references, bounds and mutants of tests/fir_shape_ref.py, checked without a GPU:

  * the references equal the pinned oracle on the oracle's own cases;
  * the bounds cannot fail a correct kernel: float32 emulations of the kernels' sums (ascending and descending FMA
    chains, the fast-FIR model of the tuner+discriminator) over the GPU cases' own taps and inputs stay below 1/4 of them;
  * the inputs separate right from wrong: every mutant differs from the reference by more than 10x the bound at some
    output of every GPU case (tests/test_gpu_fir_shapes.py), and the symmetric default low-pass is shown blind to the
    reversed-taps mutant."""
import numpy as np
import pytest

from oracle import lr_oracle as O
from tests import fir_shape_ref as R
from tests import test_gpu_fir_shapes as G
from tests import tuner_ffa_model as K

RATE = G.WBFM_RATE


# ---- the references against the oracle ------------------------------------------------------------------------------
def _close(a, b, tol=1e-6):
    a, b = np.asarray(a).astype(np.complex128), np.asarray(b).astype(np.complex128)
    assert a.shape == b.shape
    assert float(np.max(np.abs(a - b), initial=0.0)) <= tol


def test_tuner_and_discriminator_match_the_oracle():
    x = O.synth_fm_iq(0, 20000)
    for offset, D in ((-250e3, 5), (100e3, 4), (0.0, 5)):
        chain = O.tuner(offset, 200e3, D, RATE)
        taps = chain.blocks[1].taps
        y = R.tuner_ref(taps, x, offset / RATE, D)
        _close(y, O.tuner(offset, 200e3, D, RATE).process(x))
        _close(R.discrim(y, 2 * np.pi * 1.25), O.FrequencyDiscriminator(1.25).process(y.astype(np.complex64)))


@pytest.mark.parametrize("L,D,cplx", [(3, 1, True), (4, 1, False), (3, 2, True), (5, 3, False), (7, 5, True)])
def test_resampler_matches_the_oracle(L, D, cplx):
    rng = np.random.default_rng(L * 10 + D)
    x = (rng.uniform(-1, 1, 3000) + (1j * rng.uniform(-1, 1, 3000) if cplx else 0)).astype(np.complex64 if cplx else np.float32)
    chain = O.interpolator(L, cplx) if D == 1 else O.rational_resampler(L, D, cplx)
    taps = chain.blocks[2].taps
    _close(R.resample_ref(taps, x, L, D, float(L)), chain.process(x))


def test_fir_pole_downsampler_matches_the_oracle():
    x = np.random.default_rng(5).uniform(-1, 1, 20000).astype(np.float32)
    h = G.asym_taps(128, 1)
    for b, a in (O.fm_deemphasis_taps(75e-6, 1e5), O.singlepole_lowpass_taps(3e3, 1e6)):
        ref = O.Chain(O.FIRFilter(h, False), O.IIRFilterFast(b, a, False), O.Downsampler(5)).process(x)
        _close(R.pole_ref(h, b, a, x, 5), ref)


def test_phase_is_exact_at_large_indices():
    from fractions import Fraction
    for turns in G.OFFSETS:
        for n0 in G.SEEKS:
            p = R.phase_turns(turns, n0, 3000)
            for j in (0, 1, 1234, 2999):
                exact = float((Fraction(turns) * (n0 + j)) % 1)
                d = abs(p[j] - exact)
                assert min(d, 1 - d) <= 4e-16, (turns, n0, j)


# ---- the bounds cannot fail a correct kernel ------------------------------------------------------------------------
def _f32(a):
    return a.astype(np.complex64) if np.iscomplexobj(a) else a.astype(np.float32)


def _fma_chain(taps, cols, reverse):
    """sum_k taps[k] * cols(k) as a float32 FMA chain (products exact in float64, one rounding per step)."""
    order = range(len(taps) - 1, -1, -1) if reverse else range(len(taps))
    acc = None
    for k in order:
        t = np.asarray(taps[k]).astype(np.complex128) if np.iscomplexobj(taps) else np.float64(taps[k])
        v = cols(k).astype(np.complex128 if np.iscomplexobj(cols(k)) or np.iscomplexobj(taps) else np.float64)
        acc = _f32(t * v if acc is None else acc.astype(v.dtype) + t * v)
    return acc


def _direct_emulations(h, xin, idx):
    """Kept outputs idx of the FIR h over xin (the float32 samples the kernel filters), both summation orders."""
    M = len(h)
    xp = np.concatenate([np.zeros(M, xin.dtype), xin])
    return [_fma_chain(h, lambda k: xp[M + idx - k], rev) for rev in (False, True)]


EMULATED = (["tuner+discrim_m%d" % M for M in (66, 67, 100, 127, 128)] +
            ["tuner+discrim_m101_impulse50", "tuner+discrim_m66_impulse65", "tuner+discrim_m128_alternating",
             "tuner_m97", "decim_crcf_m71", "decim_rrrf_m133", "decim_rrrf_m135_impulse134",
             "fir*deemph_m128_pole", "fir*lowpass_m130_split", "rs_3x2_crcf_scaled_m%d" % G.rs_max_taps(3, 2, 8),
             "rs_7x5_rrrf_m%d" % G.rs_max_taps(7, 5, 4), "rs_160x147", "pg_cccf_d5_m480", "pg_rrrf_d3_m960"])
EMU_LEN = 40000


@pytest.mark.parametrize("name", EMULATED)
def test_float32_emulations_stay_within_a_quarter_of_the_bound(name):
    shape = G.CASES[name]()
    n0, calls = shape.streams[-1]
    x = shape.gen(sum(calls))[:EMU_LEN]
    ref, bound, gain = shape.expect(x, n0)
    got = []
    if name.startswith(("tuner", "decim_crcf")):
        h, turns = shape.taps, shape.turns
        xr = _f32(R.rotate(x, turns, n0)) if turns is not None else x
        idx = R.kept(n0, 5, len(x))
        got += _direct_emulations(h, xr, idx)
        if name.startswith("tuner+discrim"):
            tiles = (len(idx) - 1) // K.TS
            ffa, _ = K.stream(xr, h, (-n0) % 5, tiles, exact=False)
            got.append(ffa)
        if gain:
            got = [R.discrim(g.astype(np.complex128), gain) for g in got]
    elif name.startswith(("decim_rrrf", "pg_")):
        h, D = shape.taps, shape.D
        got += _direct_emulations(h, x, R.kept(n0, D, len(x)))
    elif name.startswith("fir*"):
        h, b, a = shape.taps, shape.b, shape.a
        hc, cD = R.pole_taps(h, b, a, 5)
        for w in _direct_emulations(hc.astype(np.float32), x, R.kept(n0, 5, len(x))):
            z, c = np.zeros(len(w), np.float32), np.float32(cD)
            prev = np.float32(0)
            for m in range(len(w)):
                prev = np.float32(np.float64(c) * prev + w[m])
                z[m] = prev
            got.append(z)
    else:
        h, L, D, c = shape.taps, shape.L, shape.D, shape.c
        cx = _f32(x.astype(np.complex128 if np.iscomplexobj(x) else np.float64) * c)
        i = np.arange(0, len(x) * L, D)
        q, p = np.divmod(i, L)
        hp = np.concatenate([h, np.zeros(-len(h) % L, h.dtype)]).reshape(-1, L)
        xp = np.concatenate([np.zeros(len(hp), cx.dtype), cx])
        for rev in (False, True):
            taps = lambda t: hp[t, p]                                           # noqa: E731
            order = range(len(hp) - 1, -1, -1) if rev else range(len(hp))
            acc = None
            for t in order:
                v = taps(t).astype(np.float64) * xp[len(hp) + q - t].astype(np.complex128 if np.iscomplexobj(cx) else np.float64)
                acc = _f32(v if acc is None else acc + v)
            got.append(acc)
    for g in got:
        assert R.excess(g, ref, bound, gain) < 0.25, "%s: %.3g of the bound" % (name, R.excess(g, ref, bound, gain))


# ---- the inputs separate right from wrong -----------------------------------------------------------------------------
def _margins(shape):
    """Smallest over mutants of (largest |mutant - reference| / bound over the outputs), over the case's streams."""
    worst = (np.inf, None)
    for n0, calls in shape.streams:
        x = shape.gen(sum(calls))
        ref, bound, gain = shape.expect(x, n0)
        for name, mut in shape.mutants(x, n0).items():
            m = R.excess(mut, ref, bound, gain)
            if m < worst[0]:
                worst = (m, "%s (n0=%d)" % (name, n0))
    return worst


FAMILIES = ("tuner+discrim", "tuner_", "decim_crcf", "rot+fir", "decim_rrrf", "fir*", "rs_", "pg_")


@pytest.mark.parametrize("family", FAMILIES)
def test_every_mutant_exceeds_ten_times_the_bound(family):
    report = []
    for name, make in G.CASES.items():
        if not name.startswith(family):
            continue
        margin, which = _margins(make())
        report.append((margin, name, which))
        assert margin > 10, "%s: mutant '%s' stays within %.3gx of the bound" % (name, which, margin)
    assert report
    margin, name, which = min(report)
    print("\n%s: %d cases, smallest mutant margin %.3gx (%s, %s)" % (family, len(report), margin, name, which))


def test_symmetric_lowpass_cannot_see_the_tap_order():
    """The blind spot the asymmetric taps close: on the default 128-tap low-pass the reversed taps give the same
    reference (within the bound), so no test on it can tell which way a kernel walks its taps."""
    taps = O.lowpass_filter(128, 100e3, RATE, True).taps
    x = O.synth_fm_iq(0, 20000)
    turns = -250e3 / RATE
    ref = R.tuner_ref(taps, x, turns, 5)
    rev = R.tuner_ref(taps[::-1].copy(), x, turns, 5)
    assert R.excess(rev, ref, R.tuner_bound(taps, x, 5, 0, G.TUNER_T)) <= 1


def test_case_table_covers_every_instantiated_shape():
    import os
    import re
    src = open(os.path.join(os.path.dirname(G.__file__), "..", "luaradio_b200", "csrc", "resample.cu")).read()
    pairs = set((int(a), int(b)) for a, b in re.findall(r"LRB_RS\((\d+), (\d+)\)", src))
    assert pairs == set(G.RS_PAIRS)
    src = open(os.path.join(os.path.dirname(G.__file__), "..", "luaradio_b200", "csrc", "poly_generic.cu")).read()
    body = src[src.index("bool poly_generic_supports"):]
    ds = [int(d) for d in re.findall(r"case (\d+):", body[:body.index("default")])]
    assert tuple(ds) == G.PG_DS
    for M in range(66, 129):
        assert "tuner+discrim_m%d" % M in G.CASES and "tuner_m%d" % M in G.CASES and "decim_crcf_m%d" % M in G.CASES
