"""CPU checks of the models of iir.cu's two kernels (tests/iir_small_ref.py): the float32 models stay within the per-output
bound for every filter of the GPU sets, the bound sits close above the output's own rounding, and each deliberate mutant
breaks it by a clear margin."""
import numpy as np
import pytest

from oracle import lr_oracle as O
from tests import iir_small_ref as S

SCAN = S.scan_filters()
GENERAL = S.general_filters()
# ragged calls: 0, 1 and 2 samples, T - 1 .. 2T + 1 for the tile T = 4096 and the LOCAL payload 3584
CALLS = (3 * S.T + 17, 0, 1, 2, 40, S.T - 1, S.T, S.T + 1, 3583, 3584, 3585, 2 * S.T + 1, 7167, 8192)
GEN_CALLS = (3 * S.T + 17, 0, 1, 40, S.T - 1, S.T + 1, 8191, 20000)
# the bound above u32 |y_ref|, in units of the output's RMS on uniform noise (see test_bound_is_tight)
TIGHT_LOCAL, TIGHT_SLOW, TIGHT_GENERAL = 3e-5, 1e-3, 1e-2
# the resonator that does not decay: one thread runs each call, and the bound grows with the stream (see
# test_general_bound_is_tight)
NODECAY_CALLS = (0, 1, 2, 37, 600, 1200)


def _noise(rng, n, cplx):
    v = rng.uniform(-1, 1, n)
    if cplx:
        v = v + 1j * rng.uniform(-1, 1, n)
    return v.astype(np.complex64 if cplx else np.float32)


def stream(cplx, calls=CALLS, seed=1, burst=0):
    """uniform noise over the calls; burst > 0 gates it on and off every `burst` samples, so that some restarts and
    look-back cut-offs fall into silence, where what they leave out is the whole output"""
    rng = np.random.default_rng(seed)
    xs, pos = [], 0
    for n in calls:
        v = _noise(rng, n, cplx)
        if burst:
            v = v * (((pos + np.arange(n)) // burst) % 2 == 0)
        xs.append(v.astype(np.complex64 if cplx else np.float32))
        pos += n
    return xs


def tone(calls, f=0.01, cplx=False):
    x = np.exp(2j * np.pi * f * np.arange(sum(calls)))
    x = (x if cplx else x.real).astype(np.complex64 if cplx else np.float32)
    return list(np.split(x, np.cumsum(calls)[:-1]))


def _scan_excess(b, a, xs, cplx, D=1, mutant=None, walk=1):
    y, ref, bnd, _ = S.scan_bound(b, a, xs, cplx, D)
    if mutant is None and walk == 1:
        return S.excess(y, ref, bnd)
    m = S.ScanModel(b, a, cplx, D, mutant, walk)
    with np.errstate(all="ignore"):
        got = np.concatenate([m.process(x) for x in xs])
    return S.excess(got, ref, bnd)


def _general_excess(b, a, xs, cplx, mutant=None):
    ref, bnd, _ = S.general_bound(b, a, xs, cplx)
    m = S.GeneralModel(b, a, cplx, mutant)
    got = np.concatenate([m.process(x) for x in xs])
    return S.excess(got, ref, bnd)


def test_filter_sets_take_the_small_kernels():
    for name, (b, a) in SCAN.items():
        assert len(b) <= 9 and len(a) <= 2, name
    for name, (b, a) in GENERAL.items():
        assert len(b) <= 10 and len(a) <= 10 and (len(a) > 2 or len(b) == 10), name
    # the two resonators: W just under the 65536-sample limit, and no decay within it
    assert 60000 < S.GeneralModel(*GENERAL["resonator_w64k"], False).W < S.GEN_LIMIT
    assert S.GeneralModel(*GENERAL["resonator_nodecay"], False).W == -1
    # 0.947 and 0.948 sit either side of the LOCAL threshold
    assert S.is_local(np.float32(0.947)) and not S.is_local(np.float32(0.948))


@pytest.mark.parametrize("name", ["p0.5_nb3", "pslow_nb2", "deemph", "p-1_nb2"])
def test_scan_model_tracks_the_recurrence(name):
    """3000 samples against the per-sample oracle"""
    b, a = SCAN[name]
    x = stream(False, (3000,))
    y, _, bnd, _ = S.scan_bound(b, a, x, False)
    orc = O.IIRFilter(b, a, False).process(x[0]).astype(np.float64)
    assert np.all(np.abs(y - orc) <= bnd + S.U32 * np.abs(orc))


@pytest.mark.parametrize("name", ["butter4_lowpass", "cheby1_3_bandpass", "fir10_pole"])
def test_general_model_tracks_the_recurrence(name):
    b, a = GENERAL[name]
    x = stream(False, (3000,))
    ref, bnd, _ = S.general_bound(b, a, x, False)
    got = S.GeneralModel(b, a, False).process(x[0])
    orc = O.IIRFilter(b, a, False).process(x[0]).astype(np.float64)
    assert np.all(np.abs(got - orc) <= bnd + S.U32 * np.abs(orc))


def _rms(v):
    return float(np.sqrt(np.mean(np.abs(v) ** 2)))


@pytest.mark.parametrize("name", list(SCAN))
def test_scan_bound_is_tight(name):
    """Above the output's own rounding the bound stays below 3e-5 of the output's RMS for a pole with |c| < 0.95 and
    below 1e-3 for the slow and non-decaying ones.  Where |c| -> 1, each sample's rounding reaches the next
    1 / (1 - |c|) outputs (16000 for the 10 Hz pole at 1 MHz): the measured level is about 2e-4 .. 7e-4 of the RMS
    on these streams (19 tiles), 10x below the 1e-5 absolute tolerance these filters were held to before."""
    b, a = SCAN[name]
    c = S.scan_coefs(b, a)[1]
    level = TIGHT_LOCAL if abs(c) < 0.95 else TIGHT_SLOW
    f = 0.01 if abs(c) < 0.95 else 2e-5                 # a tone in the pass band
    for xs in (stream(False), tone(CALLS, 0.5 - f if c < 0 else f)):
        _, ref, bnd, _ = S.scan_bound(b, a, xs, False)
        assert np.max(bnd - S.U32 * np.abs(ref)) <= level * _rms(ref)


@pytest.mark.parametrize("name", list(GENERAL))
def test_general_bound_is_tight(name):
    """1e-2 of the RMS for the designs (measured 5e-6 .. 8e-3): the direct form's rounding is amplified by
    sum |h| (sum |b||x| + sum |a||y|).  r = 0.99964 gets a tone at its resonance and 2e-2 (sum |h| is 3e3; measured
    1.4e-2).  For r = 1 - 1e-6, sum |h| grows with the stream's length, 1e-2 of the RMS per ~2500 samples, so it runs
    the short calls of NODECAY_CALLS (measured 7e-3 on noise and tones)."""
    b, a = GENERAL[name]
    if name == "resonator_nodecay":
        inputs, level = (stream(False, NODECAY_CALLS), tone(NODECAY_CALLS, 0.05), tone(NODECAY_CALLS, 0.1)), TIGHT_GENERAL
    elif name.startswith("resonator"):
        inputs, level = (tone(GEN_CALLS, 0.05),), 2e-2
    else:
        inputs, level = (stream(False, GEN_CALLS), tone(GEN_CALLS, 0.2 if "band" in name else 0.01)), TIGHT_GENERAL
    for xs in inputs:
        ref, bnd, _ = S.general_bound(b, a, xs, False)
        assert np.max(bnd - S.U32 * np.abs(ref)) <= level * _rms(ref)


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", list(SCAN))
def test_scan_model_within_bound(name, cplx):
    b, a = SCAN[name]
    xs = stream(cplx)
    assert _scan_excess(b, a, xs, cplx) <= 1.0
    # the longest walk (aggregates only) is within the same bound
    assert _scan_excess(b, a, xs, cplx, walk=None) <= 1.0


@pytest.mark.parametrize("D", [3, 7])
@pytest.mark.parametrize("name", ["p0.5_nb3", "p0.948_nb2", "pslow_nb9", "deemph"])
def test_scan_model_within_bound_decimated(name, D):
    b, a = SCAN[name]
    assert _scan_excess(b, a, stream(False), False, D) <= 1.0


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", list(GENERAL))
def test_general_model_within_bound(name, cplx):
    b, a = GENERAL[name]
    assert _general_excess(b, a, stream(cplx, NODECAY_CALLS if name == "resonator_nodecay" else GEN_CALLS), cplx) <= 1.0


def test_coefficient_term():
    """0 whenever a0 = +-2^k.  For a0 = 3 or 0.7 on the slow pole it is 0.4 .. 0.9 of the whole arithmetic term, and it
    grows as 1 / (1 - |c|) towards the unit circle, where the arithmetic term does not: a systematic error of the
    block, not of the kernel.  iir_create sends such filters to IirOrderBlock (tests/test_gpu_iir_small.py)."""
    xs = stream(False)
    for name in ("p0.5_a0=4", "pslow_a0=4", "p0.5_a0=-1", "pslow_a0=-1"):
        _, _, _, terms = S.scan_bound(*SCAN[name], xs, False)
        assert np.all(terms["coef"] == 0.0), name
    for name, (b, a) in S.inexact_filters().items():
        if name.startswith("pslow"):
            _, _, _, terms = S.scan_bound(b, a, xs, False)
            assert np.max(terms["coef"]) > 0.3 * np.max(terms["alg"]), name


def _mutant_case(mutant, name):
    """(stream, D, walk) on which a scan mutant is checked"""
    if mutant == "dead":
        # one call (the look-back stays within a launch): a burst, then 62 silent tiles; the raised cut-off drops a
        # predecessor 55 tiles back (10 Hz pole), where the true one keeps it
        return [np.concatenate([stream(False, (8 * S.T,))[0], np.zeros(62 * S.T + 5, np.float32)])], 1, None
    if mutant == "phase":
        return stream(False), 3, 1
    return stream(False, burst=1000), 1, 1


@pytest.mark.parametrize("mutant", S.SCAN_MUTANTS)
@pytest.mark.parametrize("name", list(SCAN))
def test_scan_mutant_breaks_bound(name, mutant):
    b, a = SCAN[name]
    xs, D, walk = _mutant_case(mutant, name)
    if not S.scan_mutant_applies(mutant, b, a, -(-sum(len(x) for x in xs) // S.T), D):
        pytest.skip("the mutant cannot differ from the truth for this filter (iir_small_ref.scan_mutant_applies)")
    assert _scan_excess(b, a, xs, False, D, mutant, walk) > 3.0


@pytest.mark.parametrize("mutant", S.GENERAL_MUTANTS)
@pytest.mark.parametrize("name", list(GENERAL))
def test_general_mutant_breaks_bound(name, mutant):
    b, a = GENERAL[name]
    m = S.GeneralModel(b, a, False)
    if m.W < 0:
        xs = stream(False, GEN_CALLS)
    else:
        # a short call, then one of 12 chunks whose input falls silent `lead` samples before every other chunk's
        # start: the true output from there on is the decaying tail of the recurrence, which a thread warmed up from
        # inside the silence misses entirely.  A shortened warm-up starts inside a silence of 3W/4; the sample before
        # a chunk, stored by its predecessor, must come from a thread that ran through the whole silence (W - 1).
        chunk = m.plan(1 << 30)[0]
        n = 12 * chunk
        lead = m.W - 1 if mutant == "first" else 3 * m.W // 4
        x = stream(False, (n,), seed=2)[0]
        for s0 in range(chunk, n, 2 * chunk):
            x[s0 - lead:s0 + chunk // 2] = 0
        xs = stream(False, (5000,)) + [x]
    if not S.general_mutant_applies(mutant, b, a, max(len(x) for x in xs)):
        pytest.skip("the mutant cannot differ from the truth for this filter (iir_small_ref.general_mutant_applies)")
    assert _general_excess(b, a, xs, False, mutant) > 3.0


@pytest.mark.parametrize("mutant", [None, "phase", "xhist", "ystate"])
def test_closed_bound_across_the_launch_split(monkeypatch, mutant):
    """scan_closed_excess, the bound of the 2^27 + 4099-sample GPU call, on the same path at a small scale: launches of
    5T + 3 samples, D = 3, so the second and third launches start with a non-zero decimation phase.  The model stays
    within it; dropping the phase, the input history or the carried output at the split breaks it."""
    monkeypatch.setattr(S, "LAUNCH", 5 * S.T + 3)
    b, a = SCAN["p-0.948_nb2"]
    x = stream(False, (12 * S.T + 4099,), seed=3)[0]
    m = S.ScanModel(b, a, False, 3, mutant)
    with np.errstate(all="ignore"):
        y = m.process(x)
    e = S.scan_closed_excess(b, a, x, y, 3, block=10000)
    if mutant is None:
        _, ref, bnd, _ = S.scan_bound(b, a, [x], False, 3)
        assert e <= 1.0 and S.excess(y, ref, bnd) <= 1.0
    else:
        assert e > 3.0
