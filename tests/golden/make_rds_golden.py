#!/usr/bin/env python3
"""Golden data for BinaryPhaseCorrectorBlock, RootRaisedCosineFilterBlock and the RDS signal path, written to
tests/golden/rds/ from a luaradio checkout:

  binaryphasecorrector_spec.npz,        the reference's own spec vectors (tests/blocks/signal/*_spec.gen.lua) in
  rootraisedcosinefilter_spec.npz       make_golden.py's BlockSpec layout
  bpc_reference_executed.npz            radio/blocks/signal/binaryphasecorrector.lua executed in this repo's test interpreter
                                        (tests/lua_interp.py, tests/lua_reference_env.py: float32-faithful sample cells, Lua
                                        numbers as Python floats) for every (N, I) of BPC_CASES: the input, the output of
                                        process() over the ragged calls CALLS (state carried), and the final average
  rds_reference_executed.npz            examples/rtlsdr_rds.lua's signal path from FrequencyDiscriminatorBlock to
                                        ComplexToRealBlock at 220.5 kHz, run by the reference's CompositeBlock in the test
                                        interpreter on a synthetic FM multiplex (mono audio, 19 kHz pilot, 1187.5-baud
                                        biphase-coded BPSK on 57 kHz) in ragged vectors: the RRC, phase corrector and
                                        ComplexToReal outputs
  rrc_glue_create.npz                   rootraisedcosinefilter.lua instantiated and initialised with the glue installed
                                        (mock library): the create call it makes and the taps it passes
  digital_glue_hooks.json               which of the fields lua/radio_b200/digital_patch.lua relies on the reference files
                                        define (tests/test_rds_oracle.py GLUE_RELIES_ON_DIGITAL)

    LUARADIO_REFERENCE=<luaradio checkout> python tests/golden/make_rds_golden.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.join(ROOT, "tests", "golden", "rds")
SPECS = ("blocks/signal/binaryphasecorrector_spec", "blocks/signal/rootraisedcosinefilter_spec")
MODULES = {"BinaryPhaseCorrectorBlock": "radio.blocks.signal.binaryphasecorrector",
           "RootRaisedCosineFilterBlock": "radio.blocks.signal.rootraisedcosinefilter"}

# (N, I, stream length): the small-N streams are longer than N*I, so the window wraps
BPC_CASES = [(8000, 32, 3000), (50, 32, 4000), (17, 15, 1200), (4, 1, 600)]
CALLS = (0, 1, 7, 0, 31, 33, 100, 5)       # then the rest: empty calls, calls shorter than I, not multiples of I
RDS_RATE, RDS_N = 220500.0, 4500
RDS_SPLITS = (0, 1500, 1501, 3200, RDS_N)


def chunks(n):
    out, i = [], 0
    for c in CALLS:
        out.append((i, i + c))
        i += c
    out.append((i, n))
    return out


def bpsk_input(n, seed):
    """A BPSK-like signal whose carrier phase drifts, with noise: symbols of 8 samples."""
    rng = np.random.default_rng(seed)
    sym = np.repeat(rng.choice([-1.0, 1.0], n // 8 + 1), 8)[:n]
    phase = 0.4 + 2 * np.pi * 3e-4 * np.arange(n)
    noise = 0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return (sym * np.exp(1j * phase) + noise).astype(np.complex64)


def rds_mpx(n, rate, rng):
    """An FM-modulated broadcast multiplex: mono audio, 19 kHz pilot, and the RDS subcarrier -- biphase-coded symbols at
    1187.5 baud, DSB-SC on 57 kHz (three times the pilot, in phase with it)."""
    t = np.arange(n) / rate
    audio = 0.4 * np.sin(2 * np.pi * 700 * t) + 0.3 * np.sin(2 * np.pi * 2300 * t)
    bits = rng.integers(0, 2, int(n * 1187.5 / rate) + 2)
    tb = t * 1187.5
    k = tb.astype(int)
    chip = np.where((tb - k) < 0.5, 1.0, -1.0) * (2.0 * bits[k] - 1)       # biphase (Manchester) symbols
    rds = chip * np.sin(2 * np.pi * 57e3 * t)
    mpx = 0.8 * audio + 0.1 * np.sin(2 * np.pi * 19e3 * t) + 0.05 * rds
    phase = 2 * np.pi * 75e3 * np.cumsum(mpx) / rate
    noise = rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n)
    return (np.exp(1j * phase) + 0.001 * noise).astype(np.complex64)


RDS_LUA = """
    local radio = require('radio')
    local block = require('radio.core.block')
    local types = require('radio.types')
    local Source = block.factory("ArraySource")
    function Source:instantiate(rate, vectors)
        self.rate, self.vectors, self.k = rate, vectors, 0
        self:add_type_signature({}, {block.Output("out", types.ComplexFloat32)})
    end
    function Source:get_rate() return self.rate end
    function Source:process() self.k = self.k + 1 return self.vectors[self.k] end
    local function sink(t)
        local Sink = block.factory("CollectSink")
        function Sink:instantiate() self:add_type_signature({block.Input("in", t)}, {}) end
        function Sink:initialize() self.got = {} end
        function Sink:process(x)
            local copy = t.vector(x.length)
            for i = 0, x.length - 1 do copy.data[i] = x.data[i] end
            self.got[#self.got + 1] = copy
        end
        return Sink()
    end
    return function (rate, vectors)
        -- examples/rtlsdr_rds.lua:14-24,38-43
        local fm_demod = radio.FrequencyDiscriminatorBlock(1.25)
        local hilbert = radio.HilbertTransformBlock(129)
        local mixer_delay = radio.DelayBlock(129)
        local pilot_filter = radio.ComplexBandpassFilterBlock(129, {18e3, 20e3})
        local pll_baseband = radio.PLLBlock(1500.0, 19e3-100, 19e3+100, 3.0)
        local mixer = radio.MultiplyConjugateBlock()
        local baseband_filter = radio.LowpassFilterBlock(128, 4e3)
        local baseband_rrc = radio.RootRaisedCosineFilterBlock(101, 1, 1187.5)
        local phase_corrector = radio.BinaryPhaseCorrectorBlock(8000)
        local clock_demod = radio.ComplexToRealBlock()
        local rrc_out, bpc_out, real_out = sink(types.ComplexFloat32), sink(types.ComplexFloat32), sink(types.Float32)
        local top = radio.CompositeBlock()
        top:connect(Source(rate, vectors), fm_demod, hilbert, mixer_delay)
        top:connect(hilbert, pilot_filter, pll_baseband)
        top:connect(mixer_delay, 'out', mixer, 'in1')
        top:connect(pll_baseband, 'out', mixer, 'in2')
        top:connect(mixer, baseband_filter, baseband_rrc, phase_corrector)
        top:connect(phase_corrector, clock_demod, real_out)
        top:connect(phase_corrector, bpc_out)
        top:connect(baseband_rrc, rrc_out)
        top:start(false)
        return rrc_out.got, bpc_out.got, real_out.got
    end
"""


def register(it):
    """The two reference classes this change covers, loaded from the reference tree into the interpreter's registry."""
    it.modules["table"] = it.G.vars["table"]               # binaryphasecorrector.lua:20 requires it
    for mod in MODULES.values():
        with open(os.path.join(os.environ["LUARADIO_REFERENCE"], mod.replace(".", "/") + ".lua")) as f:
            it.modules[mod] = f.read()
    it.run("local radio = require('radio')\n" +
           "\n".join("radio.%s = require('%s')" % (cls, mod) for cls, mod in MODULES.items()))


def write_specs(ref):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import make_golden as G
    for spec in SPECS:
        block, vectors, epsilon = G.parse_block_spec(os.path.join(ref, "tests", spec + ".gen.lua"))
        arrays, man = {}, {"block": block, "epsilon": epsilon, "source": "tests/" + spec + ".gen.lua", "vectors": []}
        for i, v in enumerate(vectors):
            args = [G.jsonable_arg(a, arrays, "v%d_arg%d" % (i, k)) for k, a in enumerate(v["args"])]
            for j, a in enumerate(v["inputs"]):
                arrays["v%d_in%d" % (i, j)] = a
            for j, a in enumerate(v["outputs"]):
                arrays["v%d_out%d" % (i, j)] = a
            man["vectors"].append({"desc": v["desc"], "args": args, "n_in": len(v["inputs"]), "n_out": len(v["outputs"])})
        arrays["manifest"] = np.array(json.dumps(man))
        np.savez_compressed(os.path.join(HERE, os.path.basename(spec) + ".npz"), **arrays)
        print("%-28s %-28s %d vectors  eps=%s" % (os.path.basename(spec), block, len(vectors), epsilon))


def write_bpc_executed(E):
    out = {}
    for k, (N, I, n) in enumerate(BPC_CASES):
        it, types = E.make_env(lib=None, cuda=False)
        register(it)
        blk = it.run("""
            local radio = require('radio')
            local types = require('radio.types')
            local blk = radio.BinaryPhaseCorrectorBlock(%d, %d)
            blk:differentiate({types.ComplexFloat32})
            blk:initialize()
            return blk
        """ % (N, I))[0]
        x = bpsk_input(n, k)
        ys = []
        for a, b in chunks(n):
            ys.append(it.f32.to_numpy(it.call(it.index(blk, "process"), [blk, it.f32.vector_from_numpy(x[a:b])])[0]))
        name = "n%d_i%d" % (N, I)
        out[name + "_x"] = x
        out[name + "_y"] = np.concatenate(ys).astype(np.complex64)
        out[name + "_average"] = np.float64(blk.hash["phi_moving_average"])
        print("%-12s %d samples, average %.17g" % (name, n, blk.hash["phi_moving_average"]))
    np.savez_compressed(os.path.join(HERE, "bpc_reference_executed.npz"), **out)


def write_rds_executed(E):
    from tests.lua_interp import to_lua
    it, types = E.make_env(lib=None, cuda=False)
    register(it)
    x = rds_mpx(RDS_N, RDS_RATE, np.random.default_rng(11))
    parts = [x[a:b] for a, b in zip(RDS_SPLITS[:-1], RDS_SPLITS[1:])]
    run = it.run(RDS_LUA)[0]
    got = it.call(run, [RDS_RATE, to_lua([it.f32.vector_from_numpy(p) for p in parts])])
    rrc, bpc, real = (np.concatenate([it.f32.to_numpy(v) for v in g.array()]) for g in got)
    out = os.path.join(HERE, "rds_reference_executed.npz")
    np.savez_compressed(out, x=x, rrc=rrc, bpc=bpc, real=real, rate=np.float64(RDS_RATE), splits=np.array(RDS_SPLITS))
    print("rds path", x.shape, rrc.shape, bpc.shape, real.shape)


def write_rrc_glue(E):
    """RootRaisedCosineFilterBlock from the reference tree with the glue installed, against the mock library."""
    from tests.test_lua_exec import MockLib, make_env as mock_env
    _, mlib, _ = mock_env()
    lib = MockLib(mlib._declared)
    it, types = E.make_env(lib=lib, cuda=True)
    register(it)
    os.environ.pop("LUARADIO_DISABLE_CUDA")            # the glue's kill switch (radio_b200/platform.lua)
    blk = it.run("""
        local radio = require('radio')
        require('radio_b200.blocks_patch')(radio)        -- firfilter_patch.lua, applied to radio.FIRFilterBlock
        require('radio_b200.digital_patch')(radio)
        local types = require('radio.types')
        local blk = radio.RootRaisedCosineFilterBlock(101, 1, 1187.5)
        blk:differentiate({types.ComplexFloat32})
        blk.inputs[1].pipe = {get_rate = function () return %r end}
        blk:initialize()
        return blk
    """ % RDS_RATE)[0]
    calls = [c for c in lib.calls if c[0].startswith("lrb200_fir_create")]
    assert len(calls) == 1, lib.calls
    name, (taps, ntaps, decim, flags) = calls[0]
    data = it.index(blk, "taps").hash["data"]
    assert taps is data
    h = np.array([it.f32._fstore[(id(it.f32.get_cell(data, i)), "value")] for i in range(ntaps)], np.float32)
    np.savez_compressed(os.path.join(HERE, "rrc_glue_create.npz"), symbol=np.array(name), ntaps=ntaps, decim=decim,
                        flags=flags, taps=h, rate=np.float64(RDS_RATE))
    print("rrc glue", name, ntaps, decim, flags)


def write_hooks(ref):
    from tests.test_rds_oracle import GLUE_RELIES_ON_DIGITAL
    found = {}
    for rel, needle in sorted(GLUE_RELIES_ON_DIGITAL):
        if needle in open(os.path.join(ref, rel)).read():
            found.setdefault(rel, []).append(needle)
    with open(os.path.join(HERE, "digital_glue_hooks.json"), "w") as f:
        json.dump({"present": found}, f, separators=(",", ":"))


def main():
    os.environ["LUARADIO_DISABLE_CUDA"] = "1"
    from tests import lua_reference_env as E
    if not E.available():
        sys.exit("set LUARADIO_REFERENCE to a luaradio checkout")
    os.makedirs(HERE, exist_ok=True)
    only = sys.argv[1:]
    for name, fn, arg in (("specs", write_specs, E.REF), ("bpc", write_bpc_executed, E), ("rds", write_rds_executed, E),
                          ("glue", write_rrc_glue, E), ("hooks", write_hooks, E.REF)):
        if not only or name in only:
            fn(arg)
    print("wrote", HERE)


if __name__ == "__main__":
    main()
