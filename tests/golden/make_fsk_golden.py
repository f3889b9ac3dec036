#!/usr/bin/env python3
"""Golden vectors for the POCSAG and AX.25 receivers' signal paths, produced by the reference itself: the example graphs
(examples/rtlsdr_pocsag.lua, examples/rtlsdr_ax25.lua) truncated after the data filter that feeds the clock recoverer, with
the RTL-SDR source replaced by ragged vectors of a synthetic 1 MS/s capture (tests/fsk_ref.py).  The reference's block
files and CompositeBlock run loop execute in this repo's test interpreter on float32-faithful sample cells
(tests/lua_interp.py, tests/lua_reference_env.py), as tests/golden/make_composite_goldens.py does.

    pocsag:  TunerBlock(-100e3, 12e3, 80) -> ComplexBandpassFilterBlock(129, {3500, 5500}) -> ComplexMagnitudeBlock (space)
                                          -> ComplexBandpassFilterBlock(129, {-5500, -3500}) -> ComplexMagnitudeBlock (mark)
             mark -> SubtractBlock in1, space -> in2 -> LowpassFilterBlock(128, 1200)
    ax25:    TunerBlock(-100e3, 12e3, 80) -> NBFMDemodulator(3e3, 3e3) -> HilbertTransformBlock(129)
             -> FrequencyTranslatorBlock(-1700) -> LowpassFilterBlock(128, 750) -> FrequencyDiscriminatorBlock(1.25)
             -> LowpassFilterBlock(128, 1200)

    LUARADIO_REFERENCE=<luaradio checkout> python tests/golden/make_fsk_golden.py [pocsag] [ax25]
        # writes tests/golden/fsk/{pocsag,ax25}_reference_executed.npz (about ten minutes each)
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

LUA = """
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
    local Sink = block.factory("CollectSink")
    function Sink:instantiate() self:add_type_signature({block.Input("in", types.Float32)}, {}) end
    function Sink:initialize() self.got = {} end
    function Sink:process(x)
        local copy = types.Float32.vector(x.length)
        for i = 0, x.length - 1 do copy.data[i] = x.data[i] end
        self.got[#self.got + 1] = copy
    end
    local graphs = {
        pocsag = function (top, source, sink)
            local tuner = radio.TunerBlock(-100e3, 12e3, 80)
            local space_filter = radio.ComplexBandpassFilterBlock(129, {3500, 5500})
            local space_magnitude = radio.ComplexMagnitudeBlock()
            local mark_filter = radio.ComplexBandpassFilterBlock(129, {-5500, -3500})
            local mark_magnitude = radio.ComplexMagnitudeBlock()
            local subtractor = radio.SubtractBlock()
            local data_filter = radio.LowpassFilterBlock(128, 1200)
            top:connect(source, tuner)
            top:connect(tuner, space_filter, space_magnitude)
            top:connect(tuner, mark_filter, mark_magnitude)
            top:connect(mark_magnitude, 'out', subtractor, 'in1')
            top:connect(space_magnitude, 'out', subtractor, 'in2')
            top:connect(subtractor, data_filter, sink)
        end,
    }
    graphs.ax25 = function (top, source, sink)
        local tuner = radio.TunerBlock(-100e3, 12e3, 80)
        local nbfm_demod = radio.NBFMDemodulator(3e3, 3e3)
        local hilbert = radio.HilbertTransformBlock(129)
        local translator = radio.FrequencyTranslatorBlock(-1700)
        local afsk_filter = radio.LowpassFilterBlock(128, 750)
        local afsk_demod = radio.FrequencyDiscriminatorBlock(1.25)
        local data_filter = radio.LowpassFilterBlock(128, 1200)
        top:connect(source, tuner, nbfm_demod)
        top:connect(nbfm_demod, hilbert, translator, afsk_filter, afsk_demod, data_filter, sink)
    end
    return function (name, rate, vectors)
        local sink = Sink()
        local top = radio.CompositeBlock()
        graphs[name](top, Source(rate, vectors), sink)
        top:start(false)
        return sink.got
    end
"""


def main():
    os.environ["LUARADIO_DISABLE_CUDA"] = "1"
    from tests import fsk_ref as K
    from tests import lua_reference_env as E
    from tests.lua_interp import to_lua
    names = sys.argv[1:] or ["pocsag", "ax25"]
    n = K.GOLDEN_N
    it, _ = E.make_env(lib=None, cuda=False)
    run = it.run(LUA)[0]
    for name, gen in (("pocsag", K.fsk_iq), ("ax25", K.afsk_nbfm_iq)):
        if name not in names:
            continue
        x = gen(n, K.GOLDEN_SEED[name])
        splits = K.golden_splits(n)
        parts = [x[a:b] for a, b in zip(splits[:-1], splits[1:])]
        t0 = time.time()
        got = it.call(run, [name, K.CAPTURE_RATE, to_lua([it.f32.vector_from_numpy(p) for p in parts])])[0]
        y = np.concatenate([it.f32.to_numpy(v) for v in got.array()])
        path = os.path.join(ROOT, "tests", "golden", "fsk", name + "_reference_executed.npz")
        np.savez_compressed(path, x=x, y=y, rate=np.float64(K.CAPTURE_RATE), splits=np.array(splits))
        print(name, x.shape, "->", y.shape, "%.1f s" % (time.time() - t0), flush=True)


if __name__ == "__main__":
    main()
