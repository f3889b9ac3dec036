"""BinaryPhaseCorrectorBlock, RootRaisedCosineFilterBlock and the RDS signal path without a GPU: the reference model
(tests/rds_oracle.py) pinned on the reference's spec vectors and on what the reference's own binaryphasecorrector.lua and
the rtlsdr_rds.lua signal path computed, the tap design, the Python constructors, the Lua glue's create calls, and the
scheduler's plan for the RDS graph."""
import json
import os
import re

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from luaradio_b200.types import ComplexFloat32, Float32
from luaradio_b200.utilities import filter_utils
from tests import rds_oracle as R
from tests.golden.make_rds_golden import BPC_CASES, CALLS, RDS_RATE, chunks
from tests.golden_util import GOLDEN_DIR, epsilon_ok, load_spec

RDS_DIR = os.path.join(GOLDEN_DIR, "rds")
REPO = os.path.dirname(os.path.dirname(GOLDEN_DIR))

# (reference file, field or method lua/radio_b200/digital_patch.lua relies on), recorded in tests/golden/rds/digital_glue_hooks.json
GLUE_RELIES_ON_DIGITAL = [
    ("radio/blocks/signal/binaryphasecorrector.lua", "self.num_samples"),
    ("radio/blocks/signal/binaryphasecorrector.lua", "self.sample_interval"),
    ("radio/blocks/signal/binaryphasecorrector.lua", "function BinaryPhaseCorrectorBlock:process(x)"),
    ("radio/blocks/signal/rootraisedcosinefilter.lua", 'block.factory("RootRaisedCosineFilterBlock", FIRFilterBlock)'),
    ("radio/blocks/signal/rootraisedcosinefilter.lua", "FIRFilterBlock.initialize(self)"),
]


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype in (np.float32, np.complex64) else np.uint64)


def test_oracle_matches_the_spec_vectors():
    """binaryphasecorrector_spec (4 vectors, 1e-6): whole, in ragged calls and sample by sample.  The spec's generator
    takes a true windowed mean; the oracle follows the reference's recurrence, within the spec's epsilon."""
    block, vectors, eps = load_spec("rds/binaryphasecorrector_spec")
    assert block == "BinaryPhaseCorrectorBlock" and len(vectors) == 4
    for v in vectors:
        x, want = v["inputs"][0], v["outputs"][0]
        ok, msg = epsilon_ok(R.BinaryPhaseCorrector(*v["args"]).process(x), want, eps)
        assert ok, "%s: %s" % (v["desc"], msg)
        o = R.BinaryPhaseCorrector(*v["args"])
        ok, msg = epsilon_ok(np.concatenate([o.process(x[a:b]) for a, b in ((0, 0), (0, 1), (1, 20), (20, 20), (20, len(x)))]), want, eps)
        assert ok, "%s (ragged): %s" % (v["desc"], msg)
        o = R.BinaryPhaseCorrector(*v["args"])
        ok, msg = epsilon_ok(np.concatenate([o.process(x[i:i + 1]) for i in range(len(x))]), want, eps)
        assert ok, "%s (sample by sample): %s" % (v["desc"], msg)


@pytest.mark.parametrize("case", ["n%d_i%d" % (N, I) for N, I, _ in BPC_CASES])
def test_oracle_equals_the_reference_lua_executed_bit_for_bit(case):
    """binaryphasecorrector.lua executed over ragged calls (empty ones, ones shorter than I, ones not a multiple of I):
    every output bit and the final moving average; for the small windows the stream is longer than N * I."""
    g = np.load(os.path.join(RDS_DIR, "bpc_reference_executed.npz"))
    N, I, n = next(c for c in BPC_CASES if "n%d_i%d" % c[:2] == case)
    x, want = g[case + "_x"], g[case + "_y"]
    assert len(x) == n and len(chunks(n)) == len(CALLS) + 1
    assert N >= 1000 or n > N * I
    o = R.BinaryPhaseCorrector(N, I)
    got = np.concatenate([o.process(x[a:b]) for a, b in chunks(n)])
    assert np.array_equal(bits(got), bits(want)), int(np.argmax(bits(got) != bits(want)))
    assert o.average == float(g[case + "_average"])
    # one call gives the same bits
    assert np.array_equal(bits(R.BinaryPhaseCorrector(N, I).process(x)), bits(want))


def test_root_raised_cosine_taps_match_the_reference():
    """filter_utils_spec.lua:48-52 (101 taps, 1 MHz, beta 0.5, symbol period 1000 s) at 1e-6, for the library's design and the model's;
    both raise the reference's error for an even tap count."""
    want = np.load(os.path.join(GOLDEN_DIR, "filter_utils_vectors.npz"))["fir_root_raised_cosine"]
    for f in (filter_utils.fir_root_raised_cosine, R.fir_root_raised_cosine):
        ok, msg = epsilon_ok(np.asarray(f(101, 1e6, 0.5, 1e3), np.float32), want, 1e-6)
        assert ok, msg
        with pytest.raises(ValueError, match=r"Number of taps must be odd\."):
            f(100, 1e6, 0.5, 1e3)
    # the two designs agree to the last bit of float32 on the RDS and BPSK31 shapes
    for args in ((101, RDS_RATE, 1, 1 / 1187.5), (101, 8000.0, 1, 1 / 31.25), (101, 2.0, 0.7, 1000.0)):
        assert np.array_equal(np.float32(filter_utils.fir_root_raised_cosine(*args)), np.float32(R.fir_root_raised_cosine(*args)))


def test_root_raised_cosine_spec_vectors():
    """rootraisedcosinefilter_spec (6 vectors, rate 2 as the reference's jig, complex and real input) at 1e-6."""
    block, vectors, eps = load_spec("rds/rootraisedcosinefilter_spec")
    assert block == "RootRaisedCosineFilterBlock" and len(vectors) == 6
    for v in vectors:
        x, want = v["inputs"][0], v["outputs"][0]
        ok, msg = epsilon_ok(R.rrc_filter(*v["args"], rate=2.0, complex_input=np.iscomplexobj(x)).process(x), want, eps)
        assert ok, "%s: %s" % (v["desc"], msg)


def test_constructors_raise_the_reference_errors():
    """binaryphasecorrector.lua:29 and rootraisedcosinefilter.lua:31-33: the same messages, in the same order."""
    with pytest.raises(AssertionError, match=r"Missing argument #1 \(num_samples\)"):
        radio.BinaryPhaseCorrectorBlock()
    b = radio.BinaryPhaseCorrectorBlock(8000)
    assert (b.num_samples, b.sample_interval) == (8000, 32)
    assert radio.BinaryPhaseCorrectorBlock(50, 7).sample_interval == 7
    b.differentiate([ComplexFloat32])
    assert b.get_output_type() is ComplexFloat32
    with pytest.raises(Exception):
        radio.BinaryPhaseCorrectorBlock(8000).differentiate([Float32])
    with pytest.raises(AssertionError, match=r"Missing argument #1 \(num_taps\)"):
        radio.RootRaisedCosineFilterBlock(None, 1, 1187.5)
    with pytest.raises(AssertionError, match=r"Missing argument #2 \(beta\)"):
        radio.RootRaisedCosineFilterBlock(101)
    with pytest.raises(AssertionError, match=r"Missing argument #3 \(symbol_rate\)"):
        radio.RootRaisedCosineFilterBlock(101, 1)
    r = radio.RootRaisedCosineFilterBlock(101, 1, 1187.5)
    assert isinstance(r, radio.FIRFilterBlock) and r.taps.length == 101
    for t in (ComplexFloat32, Float32):           # both signatures
        r.differentiate([t])
        assert r.get_output_type() is t


def test_glue_hooks_recorded_from_the_reference():
    with open(os.path.join(RDS_DIR, "digital_glue_hooks.json")) as f:
        present = {(rel, needle) for rel, needles in json.load(f)["present"].items() for needle in needles}
    assert not [h for h in GLUE_RELIES_ON_DIGITAL if h not in present]
    with open(os.path.join(GOLDEN_DIR, "reference_glue_hooks.json")) as f:
        registered = set(json.load(f)["registered_classes"])
    with open(os.path.join(REPO, "lua", "radio_b200", "digital_patch.lua")) as f:
        patched = set(re.findall(r"radio\.(\w+Block)\b", f.read()))
    assert patched == {"BinaryPhaseCorrectorBlock"} and patched <= registered
    assert "RootRaisedCosineFilterBlock" in registered
    with open(os.path.join(REPO, "lua", "radio_b200", "init.lua")) as f:
        assert "require('radio_b200.digital_patch')(radio)" in f.read()
    # the binding declares the new entry point exactly as the header does (cdef.lua is generated from it)
    from tools.gen_lua_cdef import HEADER, OUT, header_statements
    decl = [s for s in header_statements(open(HEADER).read()) if "lrb200_phasecorrector_create" in s]
    assert decl == ["lrb200_block_t* lrb200_phasecorrector_create(unsigned num_samples, unsigned sample_interval, unsigned flags)"]
    assert decl[0] + ";" in open(OUT).read()


def test_reference_rrc_class_creates_the_fir_with_its_own_taps():
    """rootraisedcosinefilter.lua with firfilter_patch.lua and digital_patch.lua installed (executed against the mock
    library by make_rds_golden.py): initialize() makes ONE lrb200_fir_create_crcf call, with the reference-designed taps --
    bit for bit the taps this library's RootRaisedCosineFilterBlock designs."""
    g = np.load(os.path.join(RDS_DIR, "rrc_glue_create.npz"))
    assert str(g["symbol"]) == "lrb200_fir_create_crcf" and (int(g["ntaps"]), int(g["decim"]), int(g["flags"])) == (101, 1, 0)
    want = np.float32(filter_utils.fir_root_raised_cosine(101, float(g["rate"]), 1, 1 / 1187.5))
    assert np.array_equal(bits(g["taps"]), bits(want))


# BinaryPhaseCorrectorBlock as the glue sees it: the fields binaryphasecorrector.lua:28-33 sets (the mock radio of
# tests/lua_mock/ leaves the digital blocks out)
DIGITAL_MOCK = """
local block = require('radio.core.block')
local types = require('radio.types')
return function (radio)
    local BPC = block.factory("BinaryPhaseCorrectorBlock")
    function BPC:instantiate(num_samples, sample_interval)
        self.num_samples = assert(num_samples, "Missing argument #1 (num_samples)")
        self.sample_interval = sample_interval or 32
        self:add_type_signature({block.Input("in", types.ComplexFloat32)}, {block.Output("out", types.ComplexFloat32)})
    end
    radio.BinaryPhaseCorrectorBlock = BPC
end
"""


def digital_radio(monkeypatch):
    """The mock radio with blocks_patch.lua and digital_patch.lua applied, as radio_b200/init.lua applies them."""
    from tests.test_lua_exec import patched_radio
    it, lib, types, lradio = patched_radio(monkeypatch)
    it.call(it.run(DIGITAL_MOCK)[0], [lradio])
    it.call(it.require("radio_b200.digital_patch"), [lradio])
    lib.calls.clear()
    return it, lib, types, lradio


def test_glue_creates_the_phase_corrector_handle(monkeypatch):
    """digital_patch.lua with the mock library: initialize() passes num_samples and sample_interval (default 32) with HOST
    pointers, make_device_handle() with DEVICE; process is the shared body."""
    from tests.test_lua_exec import Handle, vec
    it, lib, types, lradio = digital_radio(monkeypatch)
    C = types.hash["ComplexFloat32"]
    meth = lambda obj, name, *a: it.call(it.index(obj, name), [obj] + list(a))
    b200 = it.require("radio_b200.platform")
    for args, want in (((8000,), (8000, 32)), ((50, 15), (50, 15))):
        b = it.call(lradio.hash["BinaryPhaseCorrectorBlock"], list(args))[0]
        lib.calls.clear()
        meth(b, "initialize")
        assert lib.calls == [("lrb200_phasecorrector_create", want + (0,))]
        assert isinstance(b.hash["handle"], Handle) and b.hash["out"].hash["data_type"] is C
        lib.calls.clear()
        meth(b, "make_device_handle")
        assert lib.calls == [("lrb200_phasecorrector_create", want + (1,))]
        lib.calls.clear()
        y = meth(b, "process", vec(types, "ComplexFloat32", 4096))[0]
        assert [c[0] for c in lib.calls] == ["lrb200_block_max_output", "lrb200_block_execute"] and y.hash["length"] == 4096
    assert lradio.hash["BinaryPhaseCorrectorBlock"].hash["process"] is b200.hash["process"]


def test_oracle_rds_path_against_the_reference_executed_golden():
    """rds_reference_executed.npz: the rtlsdr_rds.lua signal path as the stock reference computed it (its CompositeBlock
    and the pure-Lua process() of its blocks, PLL included).  The oracle wired the same way reproduces the RRC output, the
    phase corrector's output and its ComplexToReal."""
    g = np.load(os.path.join(RDS_DIR, "rds_reference_executed.npz"))
    x, s = g["x"], list(g["splits"])
    p = R.RDSPath(float(g["rate"]))
    outs = [p.process(x[a:b]) for a, b in zip(s[:-1], s[1:])]
    rrc, bpc, real = (np.concatenate([o[k] for o in outs]) for k in range(3))
    scale = float(np.max(np.abs(g["rrc"])))
    assert len(bpc) == len(x) and scale > 1e-3
    # float32 accumulation in the reference's Lua FIR loops against float64 here; relative to the signal's size
    for got, want in ((rrc, g["rrc"]), (bpc, g["bpc"]), (real, g["real"])):
        assert np.max(np.abs(got - want)) <= 1e-5 * scale
    # the corrector rotated its input (its 8000-entry window holds ~140 measurements here, so by a small angle)
    assert np.max(np.abs(g["bpc"] - g["rrc"])) > 1e-3 * scale


def rds_graph():
    """examples/rtlsdr_rds.lua:13-24,38-43,48: the source at 1.1025 MS/s through ComplexToRealBlock, with sinks on the
    phase corrector (the sampler's data input), on ComplexToReal (the clock recoverer) and on the RRC (the spectrum plot)."""
    x = np.zeros(16, np.complex64)
    top = radio.CompositeBlock()
    src = radio.ArraySource(x, 1102500.0)
    hilbert, delay = radio.HilbertTransformBlock(129), radio.DelayBlock(129)
    pll, mixer = radio.PLLBlock(1500.0, 19e3 - 100, 19e3 + 100, 3.0), radio.MultiplyConjugateBlock()
    rrc, bpc, c2r = radio.RootRaisedCosineFilterBlock(101, 1, 1187.5), radio.BinaryPhaseCorrectorBlock(8000), radio.ComplexToRealBlock()
    top.connect(src, radio.TunerBlock(-250e3, 200e3, 5), radio.FrequencyDiscriminatorBlock(1.25), hilbert, delay)
    top.connect(hilbert, radio.ComplexBandpassFilterBlock(129, [18e3, 20e3]), pll)
    top.connect(delay, "out", mixer, "in1")
    top.connect(pll, "out", mixer, "in2")
    top.connect(mixer, radio.LowpassFilterBlock(128, 4e3), rrc, bpc)
    top.connect(bpc, c2r, radio.ArraySink())
    top.connect(bpc, radio.ArraySink())
    top.connect(rrc, radio.ArraySink())
    top._prepare_to_run(initialize=False)
    return top


def test_planner_puts_the_rds_path_in_one_device_dag():
    top = rds_graph()
    dags = top._plan_gpu_dags()
    assert len(dags) == 1
    members, ext_in, ext_out = dags[0]
    gpu = [b for b in top._concrete_order if b.name not in ("ArraySource", "ArraySink")]
    assert set(members) == set(gpu) and len(gpu) == 13
    assert ext_in.owner.name == "ArraySource"
    assert sorted(p.owner.name for p in ext_out) == ["BinaryPhaseCorrectorBlock", "ComplexToRealBlock", "RootRaisedCosineFilterBlock"]
    assert top._plan_gpu_runs(set(members)) == []


def test_lua_dag_planner_agrees_on_the_rds_path(monkeypatch):
    """plan_gpu_dags (Lua, executed) against CompositeBlock._plan_gpu_dags (Python) on the RDS graph: same members, same
    outside feed, same outside-read outputs."""
    from tests.test_lua_exec import LUA_GPU_BASE, export_graph
    it, lib, types, lradio = digital_radio(monkeypatch)
    top = rds_graph()
    base = dict(LUA_GPU_BASE, RootRaisedCosineFilterBlock="FIRFilterBlock", BinaryPhaseCorrectorBlock="BinaryPhaseCorrectorBlock")
    lua_gpu = {b: base[b.name] for b in top._concrete_order if b.name in base}
    from luaradio_b200.signal_blocks import GPUBlock
    assert all(b in lua_gpu for b in top._concrete_order if isinstance(b, GPUBlock))
    (members_py, ext_in_py, ext_out_py), = top._plan_gpu_dags()
    lua_of, conns = export_graph(it, lradio, types, top, lua_gpu)
    name_of = {id(lb): b for b, lb in lua_of.items()}
    plans = it.call(it.require("radio_b200.composite_patch").hash["plan_gpu_dags"], [conns])[0].array()
    assert len(plans) == 1
    members = plans[0].hash["members"].array()
    assert {id(m) for m in members} == {id(lua_of[b]) for b in members_py} and len(members) == len(members_py)
    assert name_of[id(plans[0].hash["ext_in"].hash["owner"])] is ext_in_py.owner
    assert sorted(name_of[id(p.hash["owner"])].name for p in plans[0].hash["ext_out"].array()) == sorted(p.owner.name for p in ext_out_py)


def _have_gpu():
    try:
        return _lib.load().lrb200_device_count() > 0
    except Exception:
        return False


def test_create_fails_without_a_device():
    if _have_gpu():
        pytest.skip("a GPU is present")
    lib = _lib.load()
    assert not lib.lrb200_phasecorrector_create(8000, 32, 0)
    assert b"no CPU fallback" in lib.lrb200_last_error()
    blk = radio.BinaryPhaseCorrectorBlock(8000)
    blk.get_rate = lambda: 44100.0
    blk.differentiate([ComplexFloat32])
    with pytest.raises(_lib.LibraryError, match="no CPU fallback"):
        blk.initialize()
