"""AGCBlock and PowerSquelchBlock without a GPU: the reference model (tests/level_oracle.py) pinned on the reference's spec
vectors and on what the reference's own agc.lua / powersquelch.lua computed, its vectorised form against its loop, the
Python constructors, the Lua glue's create calls, and the scheduler's plan for the two rx_am flow graphs."""
import json
import os
import re

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from luaradio_b200.types import ComplexFloat32, Float32
from tests import level_oracle as L
from tests.golden.make_level_golden import CALLS, CASES, N, RATE, chunks
from tests.golden_util import GOLDEN_DIR, epsilon_ok, load_spec

LEVEL_DIR = os.path.join(GOLDEN_DIR, "level")

# (reference file, field or method lua/radio_b200/level_patch.lua relies on), recorded in tests/golden/level/level_glue_hooks.json
GLUE_RELIES_ON_LEVEL = [
    ("radio/blocks/signal/agc.lua", "self.target"), ("radio/blocks/signal/agc.lua", "self.threshold"),
    ("radio/blocks/signal/agc.lua", "self.gain_tau"), ("radio/blocks/signal/agc.lua", "self.power_tau"),
    ("radio/blocks/signal/agc.lua", "self.process_real"), ("radio/blocks/signal/agc.lua", "self.process_complex"),
    ("radio/blocks/signal/powersquelch.lua", "self.threshold"), ("radio/blocks/signal/powersquelch.lua", "self.tau"),
    ("radio/blocks/signal/powersquelch.lua", "self.process_real"), ("radio/blocks/signal/powersquelch.lua", "self.process_complex"),
]


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype in (np.float32, np.complex64) else np.uint64)


def oracle_for(ctor, rate):
    """The oracle for a Lua constructor string of make_level_golden.CASES."""
    import ast
    name, args = ctor.split("(", 1)
    args = args[:-1].replace("nil", "None").replace("{", "dict(").replace("}", ")").replace("'", '"')
    vals = ast.literal_eval("[" + args.replace("dict(", "{").replace(")", "}").replace(" = ", '": ').replace("{gain_tau", '{"gain_tau')
                            .replace("{power_tau", '{"power_tau').replace(", power_tau", ', "power_tau') + "]")
    return (L.AGC if name == "AGCBlock" else L.PowerSquelch)(*vals, rate=rate)


@pytest.mark.parametrize("spec", ["agc_spec", "powersquelch_spec"])
def test_oracle_matches_the_spec_vectors(spec):
    """Both forms of the oracle on the reference's spec vectors (rate 2.0, as the reference's jig), at their 1e-6: whole,
    in ragged calls and sample by sample."""
    block, vectors, eps = load_spec("level/" + spec)
    assert len(vectors) == {"agc_spec": 6, "powersquelch_spec": 4}[spec]
    for v in vectors:
        x, want = v["inputs"][0], v["outputs"][0]
        mk = lambda: (L.AGC if block == "AGCBlock" else L.PowerSquelch)(*v["args"], rate=2.0)
        for form in ("process_loop", "process"):
            ok, msg = epsilon_ok(getattr(mk(), form)(x), want, eps)
            assert ok, "%s / %s (%s): %s" % (block, v["desc"], form, msg)
            o = mk()
            ok, msg = epsilon_ok(np.concatenate([getattr(o, form)(x[a:b]) for a, b in ((0, 1), (1, 100), (100, len(x)))]), want, eps)
            assert ok, "%s / %s (%s, ragged): %s" % (block, v["desc"], form, msg)
            o = mk()
            ok, msg = epsilon_ok(np.concatenate([getattr(o, form)(x[i:i + 1]) for i in range(len(x))]), want, eps)
            assert ok, "%s / %s (%s, sample by sample): %s" % (block, v["desc"], form, msg)


@pytest.mark.parametrize("case", [c[0] for c in CASES])
def test_oracle_equals_the_reference_lua_executed_bit_for_bit(case):
    """agc.lua / powersquelch.lua executed (instantiate, initialize at 1 kHz, process() over ragged calls): the oracle
    reproduces the linearised constants, every output bit and the carried state, in both of its forms."""
    g = np.load(os.path.join(LEVEL_DIR, "level_reference_executed.npz"))
    name, ctor, cplx, fields = next(c for c in CASES if c[0] == case)
    x, want = g[name + "_x"], g[name + "_y"]
    assert len(x) == N and np.iscomplexobj(x) == cplx and len(chunks(N)) == len(CALLS) + 1
    for form in ("process_loop", "process"):
        o = oracle_for(ctor, RATE)
        got = np.concatenate([getattr(o, form)(x[a:b]) for a, b in chunks(N)])
        assert np.array_equal(bits(got), bits(want)), (form, int(np.argmax(bits(got) != bits(want))))
        mine = {"power_alpha": o.power_alpha, "alpha": o.power_alpha, "threshold": o.threshold, "average_power": o.average_power,
                "tau": getattr(o, "tau", None), "gain_alpha": getattr(o, "gain_alpha", None), "target": getattr(o, "target", None),
                "gain_tau": getattr(o, "gain_tau", None), "power_tau": getattr(o, "power_tau", None), "gain": o.gain}
        for f in fields:
            assert mine[f] == float(g["%s_%s" % (name, f)]), (form, f)
    # the gate opened and closed within the run (agc_custom_complex keeps the default -75 dBFS threshold: open throughout)
    _, gate = oracle_for(ctor, RATE).gate(x)
    d = np.diff(gate.astype(int))
    assert gate.any() and (case == "agc_custom_complex" or ((d == -1).any() and (d == 1).any()))


def bursty(n, cplx, seed=5, seg=300):
    """Noise whose level jumps between -100 and 0 dBFS every `seg` samples: the gate flips many times."""
    rng = np.random.default_rng(seed)
    env = np.repeat(10 ** rng.uniform(-5, 0, n // seg + 1), seg)[:n]
    if cplx:
        return (env * (rng.standard_normal(n) + 1j * rng.standard_normal(n)) / np.sqrt(2)).astype(np.complex64)
    return (env * rng.standard_normal(n)).astype(np.float32)


@pytest.mark.parametrize("cplx", [False, True])
def test_fast_form_equals_the_loop_bit_for_bit(cplx):
    x = bursty(100000, cplx)
    cuts = [0, 1, 2, 2049, 40000, 40001, 100000]
    for mk in (lambda: L.AGC("custom", -20, -40, {"gain_tau": 0.01, "power_tau": 0.002}, rate=1000.0),
               lambda: L.AGC("fast", -35, -45, {"power_tau": 0.01}, rate=1000.0), lambda: L.PowerSquelch(-40, rate=1000.0)):
        a, b = mk(), mk()
        flips = np.count_nonzero(np.diff(a.gate(x)[1].astype(int)))
        assert flips > 200
        ya = np.concatenate([a.process_loop(x[p:q]) for p, q in zip(cuts, cuts[1:])])
        yb = np.concatenate([b.process(x[p:q]) for p, q in zip(cuts, cuts[1:])])
        assert np.array_equal(bits(ya), bits(yb))
        assert (a.average_power, a.gain) == (b.average_power, b.gain)


def test_constructors_raise_the_reference_errors_in_order():
    """agc.lua:42-51 and powersquelch.lua:25: the same messages, checked in the same order."""
    with pytest.raises(AssertionError, match=r'Missing argument #1 \(mode\), can be "fast", "slow", or "custom"'):
        radio.AGCBlock()
    with pytest.raises(AssertionError, match='Invalid mode "medium"'):
        radio.AGCBlock("medium")                            # the mode check comes before the gain_tau check
    with pytest.raises(AssertionError, match='Missing gain_tau parameter for "custom" mode'):
        radio.AGCBlock("custom", -30, -60, {"power_tau": 0.5})
    with pytest.raises(AssertionError, match=r"Missing argument #1 \(threshold\)"):
        radio.PowerSquelchBlock()
    a = radio.AGCBlock("fast", None, None, {"gain_tau": 7.0})
    assert (a.target, a.threshold, a.gain_tau, a.power_tau) == (-35, -75, 0.1, 1.0)   # fast / slow ignore options.gain_tau
    a = radio.AGCBlock("custom", -20, -50, {"gain_tau": 0.5, "power_tau": 0.25})
    assert (a.target, a.threshold, a.gain_tau, a.power_tau) == (-20, -50, 0.5, 0.25)
    assert radio.AGCBlock("slow").gain_tau == 3.0
    # PowerSquelch: the second argument is accepted and ignored (powersquelch.lua:26 reads an undefined global)
    assert radio.PowerSquelchBlock(-40, 0.5).tau == radio.PowerSquelchBlock(-40).tau == 0.001
    for cls, args in ((radio.AGCBlock, ("slow",)), (radio.PowerSquelchBlock, (-40,))):
        b = cls(*args)
        for t in (Float32, ComplexFloat32):
            b.differentiate([t])
            assert b.get_output_type() is t


def test_glue_hooks_recorded_from_the_reference():
    with open(os.path.join(LEVEL_DIR, "level_glue_hooks.json")) as f:
        present = {(rel, needle) for rel, needles in json.load(f)["present"].items() for needle in needles}
    assert not [h for h in GLUE_RELIES_ON_LEVEL if h not in present]
    # the classes level_patch.lua patches are registered by the reference (radio/blocks/init.lua)
    with open(os.path.join(GOLDEN_DIR, "reference_glue_hooks.json")) as f:
        registered = set(json.load(f)["registered_classes"])
    with open(os.path.join(os.path.dirname(os.path.dirname(GOLDEN_DIR)), "lua", "radio_b200", "level_patch.lua")) as f:
        patched = set(re.findall(r"radio\.(\w+Block)\b", f.read()))
    assert patched == {"AGCBlock", "PowerSquelchBlock"} and patched <= registered
    # and the entry point applies the patch
    with open(os.path.join(os.path.dirname(os.path.dirname(GOLDEN_DIR)), "lua", "radio_b200", "init.lua")) as f:
        assert "require('radio_b200.level_patch')(radio)" in f.read()


# The two reference classes as the glue sees them: the fields agc.lua:41-51 / powersquelch.lua:24-26 set, the data type as
# the last constructor argument (the mock radio of tests/lua_mock/ leaves level control out).
LEVEL_MOCK = """
local block = require('radio.core.block')
local types = require('radio.types')
return function (radio)
    local F = types.Float32
    local AGC = block.factory("AGCBlock")
    function AGC:instantiate(mode, target, threshold, options, data_type)
        self.mode, self.target, self.threshold, self.options = mode, target or -35, threshold or -75, options or {}
        self.gain_tau = ({fast = 0.1, slow = 3.0})[self.mode] or self.options.gain_tau
        self.power_tau = self.options.power_tau or 1.0
        self:add_type_signature({block.Input("in", data_type or F)}, {block.Output("out", data_type or F)})
    end
    radio.AGCBlock = AGC
    local Squelch = block.factory("PowerSquelchBlock")
    function Squelch:instantiate(threshold, cutoff, data_type)
        self.threshold, self.tau = threshold, 0.001
        self:add_type_signature({block.Input("in", data_type or F)}, {block.Output("out", data_type or F)})
    end
    radio.PowerSquelchBlock = Squelch
end
"""


def level_radio(monkeypatch):
    """The mock radio with both blocks_patch.lua and level_patch.lua applied, as radio_b200/init.lua applies them."""
    from tests.test_lua_exec import patched_radio
    it, lib, types, lradio = patched_radio(monkeypatch)
    it.call(it.run(LEVEL_MOCK)[0], [lradio])
    it.call(it.require("radio_b200.level_patch"), [lradio])
    lib.calls.clear()
    return it, lib, types, lradio


def test_glue_creates_the_level_handles(monkeypatch):
    """level_patch.lua, executed with the mock library: the create call gets the dBFS values, the time constants and the
    rate (fast, slow, custom, squelch), the device form passes DEVICE, both process entry points are the shared body."""
    from tests.test_lua_exec import Handle, vec
    it, lib, types, lradio = level_radio(monkeypatch)
    C, F = types.hash["ComplexFloat32"], types.hash["Float32"]
    new = lambda cls, *a: it.call(lradio.hash[cls], list(a))[0]
    meth = lambda obj, name, *a: it.call(it.index(obj, name), [obj] + list(a))
    from tests.lua_interp import LuaTable
    cases = [
        ("AGCBlock", ("fast", None, None, None, F), "lrb200_agc_create", (-35, -75, 0.1, 1.0, 44100.0, 0)),
        ("AGCBlock", ("slow", -20, -60, LuaTable({"gain_tau": 9.0}), C), "lrb200_agc_create", (-20, -60, 3.0, 1.0, 44100.0, 1)),
        ("AGCBlock", ("custom", -30, -70, LuaTable({"gain_tau": 0.5, "power_tau": 0.25}), F), "lrb200_agc_create",
         (-30, -70, 0.5, 0.25, 44100.0, 0)),
        ("PowerSquelchBlock", (-40, 0.5, C), "lrb200_powersquelch_create", (-40, 0.001, 44100.0, 1)),
        ("PowerSquelchBlock", (-55, None, F), "lrb200_powersquelch_create", (-55, 0.001, 44100.0, 0)),
    ]
    b200 = it.require("radio_b200.platform")
    for cls, args, symbol, want in cases:
        lib.calls.clear()
        b = new(cls, *args)
        b.hash["rate"] = 44100.0
        meth(b, "initialize")
        assert lib.calls == [(symbol, want + (0,))], (cls, lib.calls)
        assert isinstance(b.hash["handle"], Handle) and b.hash["out"].hash["data_type"] is args[-1]
        assert b.hash["target" if cls == "AGCBlock" else "threshold"] == want[0]       # left in dBFS
        lib.calls.clear()
        meth(b, "make_device_handle")
        assert lib.calls == [(symbol, want + (1,))]
        lib.calls.clear()
        x = vec(types, "Float32", 8192)
        y = meth(b, "process_real", x)[0]
        assert [c[0] for c in lib.calls] == ["lrb200_block_max_output", "lrb200_block_execute"] and y.hash["length"] == 8192
        for n in ("process_real", "process_complex"):
            assert lradio.hash[cls].hash[n] is b200.hash["process"]


def rx_am_graphs():
    x = np.zeros(16, np.complex64)
    env = radio.CompositeBlock()
    env.connect(radio.ArraySource(x, 1102500.0), radio.TunerBlock(-50e3, 10e3, 25), radio.AMEnvelopeDemodulator(5e3),
                radio.AGCBlock("slow"), radio.ArraySink())
    sync = radio.CompositeBlock()
    sync.connect(radio.ArraySource(x, 1102500.0), radio.DecimatorBlock(5), radio.AMSynchronousDemodulator(50e3, 5e3),
                 radio.DownsamplerBlock(5), radio.AGCBlock("slow"), radio.ArraySink())
    for t in (env, sync):
        t._prepare_to_run(initialize=False)
    return env, sync


def test_planner_puts_both_rx_am_graphs_on_the_device():
    """rx_am.lua:51-55 (envelope) is one device chain, :66-71 (synchronous) one device DAG: no block left on the host."""
    env, sync = rx_am_graphs()
    assert env._plan_gpu_dags() == []
    runs = [[b.name for b in run] for run, _, _ in env._plan_gpu_runs()]
    assert runs == [["FrequencyTranslatorBlock", "LowpassFilterBlock", "DownsamplerBlock", "ComplexMagnitudeBlock",
                     "SinglepoleHighpassFilterBlock", "LowpassFilterBlock", "AGCBlock"]]
    dags = sync._plan_gpu_dags()
    assert len(dags) == 1
    members, ext_in, ext_out = dags[0]
    gpu = [b for b in sync._concrete_order if b.name not in ("ArraySource", "ArraySink")]
    assert set(members) == set(gpu) and members[-1].name == "AGCBlock"
    assert ext_in.owner.name == "ArraySource" and [p.owner.name for p in ext_out] == ["AGCBlock"]
    assert sync._plan_gpu_runs(set(members)) == []


def test_lua_scheduler_puts_the_envelope_graph_in_one_chain(monkeypatch):
    from tests.test_lua_exec import LUA_GPU_BASE, export_graph
    it, lib, types, lradio = level_radio(monkeypatch)
    env, _ = rx_am_graphs()
    base = dict(LUA_GPU_BASE, AGCBlock="AGCBlock", PowerSquelchBlock="PowerSquelchBlock")
    lua_gpu = {b: base[b.name] for b in env._concrete_order if b.name in base}
    assert any(b.name == "AGCBlock" for b in lua_gpu)
    lua_of, conns = export_graph(it, lradio, types, env, lua_gpu)
    it.call(it.require("radio_b200.composite_patch").hash["collapse_gpu_runs"], [conns])
    chains = {id(p.hash["owner"]): p.hash["owner"] for pair in conns.hash.items() for p in pair if "blocks" in p.hash["owner"].hash}
    got = [[b.hash["name"] for b in c.hash["blocks"].array()] for c in chains.values()]
    assert got == [[b.name for b in run] for run, _, _ in env._plan_gpu_runs()]


def _have_gpu():
    try:
        return _lib.load().lrb200_device_count() > 0
    except Exception:
        return False


def test_create_fails_without_a_device():
    if _have_gpu():
        pytest.skip("a GPU is present")
    lib = _lib.load()
    assert not lib.lrb200_agc_create(-35.0, -75.0, 3.0, 1.0, 44100.0, 1, 0)
    assert b"no CPU fallback" in lib.lrb200_last_error()
    assert not lib.lrb200_powersquelch_create(-40.0, 0.001, 44100.0, 0, 1)
    assert b"no CPU fallback" in lib.lrb200_last_error()
    for blk in (radio.AGCBlock("slow"), radio.PowerSquelchBlock(-40)):
        blk.get_rate = lambda: 44100.0
        blk.differentiate([ComplexFloat32])
        with pytest.raises(_lib.LibraryError, match="no CPU fallback"):
            blk.initialize()
