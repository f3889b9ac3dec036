"""The ERT receiver's signal path with no device (composites/ertreceiver.lua:38-43: ComplexMagnitude -> Lowpass(128,
4 * 32768) -> Downsampler(6) -> ManchesterMatchedFilter(32768)):

  * ManchesterMatchedFilterBlock's taps against the reference's spec generator (manchestermatchedfilter_spec.py:6-12:
    int(rate / baudrate) taps of -1, then as many of +1, negated with `invert`) at integer and non-integer symbol periods,
    and the oracle against the reference's committed vectors;
  * the geometry model of the overlap-save kernel's fused-magnitude mode (tests/ert_ref.py MagFirModel):
    packed-real blocks, the overlap-save kernel on every call, the launch counts of the rrrf mode it shares them with;
  * the Python planner sees the four blocks as one GPU run, and the Lua glue gives the reference's subclass the GPU FIR
    (the Lua planner's test for a GPU block)."""
import numpy as np
import pytest

import luaradio_b200 as radio
from tests import ert_ref as E
from tests import fft_fir_ref as F
from tests.golden_util import JIG_RATE, epsilon_ok, load_spec

ERT_RATE = 72 * 32768.0             # 2.359296 MS/s: 12 samples per symbol after the decimation by 6


def spec_taps(baudrate, sample_rate, invert):
    """manchestermatchedfilter_spec.py:6-12, the reference's own tap generator."""
    symbol_period = int(sample_rate / baudrate)
    h = np.array([-1] * symbol_period + [1] * symbol_period)
    return ((h * -1) if invert else h).astype(np.float32)


@pytest.mark.parametrize("rate,baud", [(2.0, 0.1), (2.0, 0.3), (10.0, 2.5), (ERT_RATE / 6, 32768.0), (ERT_RATE / 5, 32768.0), (1e6, 32768.0),
                                       (2.4e6 / 6, 32768.0), (32768.0, 32768.0), (50000.0, 32768.0)])
@pytest.mark.parametrize("invert", [False, True])
def test_tap_design_matches_the_spec_generator(rate, baud, invert):
    want = spec_taps(baud, rate, invert)
    got = radio.ManchesterMatchedFilterBlock.design(rate, baud, invert)
    assert got.dtype == np.float32 and np.array_equal(got, want), (rate, baud, got, want)
    assert np.array_equal(E.manchester_matched_filter(baud, rate, invert).taps, want)


def test_a_rate_below_the_baud_rate_is_refused():
    with pytest.raises(AssertionError, match="below the baud rate"):
        radio.ManchesterMatchedFilterBlock.design(32767.0, 32768.0, False)
    with pytest.raises(AssertionError, match="below the baud rate"):
        E.manchester_matched_filter(32768.0, 1000.0)
    with pytest.raises(AssertionError, match="Missing argument #1"):
        radio.ManchesterMatchedFilterBlock(None)


def test_block_signature_is_float32_only():
    b = radio.ManchesterMatchedFilterBlock(32768)
    assert isinstance(b, radio.FIRFilterBlock) and not b.invert
    b.differentiate([radio.types.Float32])
    assert b.get_output_type() is radio.types.Float32
    with pytest.raises(AssertionError, match="No compatible type signatures"):
        radio.ManchesterMatchedFilterBlock(32768, True).differentiate([radio.types.ComplexFloat32])


def test_oracle_on_the_reference_vectors():
    block, vectors, eps = load_spec("ert/manchestermatchedfilter_spec")
    assert block == "ManchesterMatchedFilterBlock" and len(vectors) == 2
    for v in vectors:
        baud, invert = v["args"][0], bool(v["args"][1])
        assert len(E.manchester_taps(baud, JIG_RATE, invert)) == 2 * int(JIG_RATE / baud)
        o = E.manchester_matched_filter(baud, JIG_RATE, invert)
        ok, msg = epsilon_ok(o.process(v["inputs"][0]), v["outputs"][0], eps)
        assert ok, "%s: %s" % (v["desc"], msg)
        o = E.manchester_matched_filter(baud, JIG_RATE, invert)
        x = v["inputs"][0]
        ok, msg = epsilon_ok(np.concatenate([o.process(x[i:i + 7]) for i in range(0, len(x), 7)]), v["outputs"][0], eps)
        assert ok, "%s, in calls of 7: %s" % (v["desc"], msg)


# ---- the fused-magnitude mode's geometry --------------------------------------------------------------------------------
MAG_M = (1, 2, 33, 128, 257, 512, 513)
MAG_D = (2, 5, 6, 33)


@pytest.mark.parametrize("M", MAG_M)
@pytest.mark.parametrize("D", MAG_D)
def test_magnitude_mode_plans_like_the_packed_real_mode(M, D):
    """Complex in, real out, two real blocks per transform: the blocks and launches of the rrrf mode with the FFT forced,
    on every call length, whatever the FIR's algorithm, since no other kernel has the magnitude prologue."""
    rrrf = F.FirModel("rrrf", M, D, algo="fft")
    mag = E.MagFirModel(M, D)
    assert not mag.poly and not mag.gen_poly and mag.fast and mag.effective() == "fft"
    assert mag.per == rrrf.per == 2 * (1024 - (M - 1))
    for consumed in (0, D - 1, 2 ** 40 + 2):
        for n in F.call_list(mag):
            assert mag.plan(n, consumed) == rrrf.plan(n, consumed), (n, consumed)


def test_magnitude_mode_launch_counts_of_the_ert_stage():
    """Lowpass(128) at D = 6: L = 897, 1794 inputs per transform; a call launches the history update, the edge kernel
    and, once it has an interior block, the interior kernel."""
    m = E.MagFirModel(128, 6)
    assert m.L == 897 and m.per == 1794
    assert m.plan(1, 0) == ("fft", 2, [(1, 1, 1)])
    assert m.plan(1794, 0) == ("fft", 2, [(1, 1, 1)])
    assert m.plan(8192, 0) == ("fft", 3, [(1, 4, 5)])
    assert m.plan(8192, 5) == ("fft", 3, [(1, 4, 5)])
    assert m.plan(1 << 24, 0) == ("fft", 3, [(1, (1 << 24) // 1794, -(-(1 << 24) // 1794))])
    # the decimating rrrf FIR it replaces leaves calls shorter than 8 L to a direct kernel under AUTO
    assert F.FirModel("rrrf", 128, 6).plan(8 * 897 - 1, 0)[0] in ("direct", "poly_generic")
    assert m.plan(8 * 897 - 1, 0)[0] == "fft"
    with pytest.raises(AssertionError):
        E.MagFirModel(514, 6)


def test_magnitude_mode_bound_covers_a_float32_magnitude():
    """The reference takes |x| in float64; the bound's magnitude term covers the kernel's float32 |x| (fed exactly to a
    float64 FIR) on inputs that span 60 dB."""
    rng = np.random.default_rng(5)
    n = 20000
    x = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * np.where((np.arange(n) // 3000) % 2, 1e-3, 1.0)).astype(np.complex64)
    h = F.G.asym_taps(128, 7)
    case = E.MagCase("", h, 6, streams=[(0, [n])])
    ref, bound, _, k = case.expect(x, 0, [n])
    mag32 = np.sqrt((x.real.astype(np.float32) ** 2 + x.imag.astype(np.float32) ** 2).astype(np.float32)).astype(np.float32)
    got = F.fir_ref(h, mag32.astype(np.float64), wide=True)[k]
    assert np.all(np.abs(got - ref) <= bound)


# ---- planners and glue ---------------------------------------------------------------------------------------------------
def ert_top(x=np.zeros(16, np.complex64), rate=ERT_RATE):
    top, sinks = radio.CompositeBlock(), [radio.ArraySink() for _ in range(3)]
    mf = radio.ManchesterMatchedFilterBlock(32768)
    top.connect(radio.ArraySource(x, rate), radio.ComplexMagnitudeBlock(), radio.LowpassFilterBlock(128, 4 * 32768),
                radio.DownsamplerBlock(6), mf)
    for s in sinks:
        top.connect(mf, s)
    return top


def test_python_planner_runs_the_front_end_as_one_chain():
    top = ert_top()
    top._prepare_to_run(initialize=False)
    assert top._plan_gpu_dags() == []
    assert [[b.name for b in run] for run, _, _ in top._plan_gpu_runs()] == [
        ["ComplexMagnitudeBlock", "LowpassFilterBlock", "DownsamplerBlock", "ManchesterMatchedFilterBlock"]]


def test_lua_glue_gives_the_subclass_the_gpu_fir(monkeypatch):
    """manchestermatchedfilter.lua:25 makes the block with block.factory(name, FIRFilterBlock) and its initialize() ends in
    FIRFilterBlock.initialize: the GPU form firfilter_patch.lua installs on FIRFilterBlock is the subclass's, so the
    Lua planner (composite_patch.lua on_gpu: make_device_handle) treats it as a GPU block with nothing added."""
    from tests.test_lua_exec import patched_radio
    it, lib, types, radio_lua = patched_radio(monkeypatch)
    block = it.require("radio.core.block")
    fir = radio_lua.hash["FIRFilterBlock"]
    mmf = it.call(block.hash["factory"], ["ManchesterMatchedFilterBlock", fir])[0]
    for name in ("make_device_handle", "process_real_input_real_taps", "initialize"):
        assert it.index(mmf, name) is it.index(fir, name), name
