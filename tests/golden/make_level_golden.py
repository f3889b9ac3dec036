#!/usr/bin/env python3
"""Golden data for AGCBlock and PowerSquelchBlock, written to tests/golden/level/ from a luaradio checkout:

  agc_spec.npz, powersquelch_spec.npz   the reference's own spec vectors (tests/blocks/signal/{agc,powersquelch}_spec.gen.lua)
                                        in make_golden.py's BlockSpec layout
  level_reference_executed.npz          radio/blocks/signal/agc.lua and powersquelch.lua executed in this repo's test
                                        interpreter (tests/lua_interp.py, tests/lua_reference_env.py: float32-faithful
                                        sample cells, Lua numbers as Python floats): for every case in CASES the input,
                                        the output of process() over ragged calls (state carried), the constants
                                        initialize() linearised and the state after the last call
  level_glue_hooks.json                 which of the fields lua/radio_b200/level_patch.lua relies on the reference files
                                        define (tests/test_level_oracle.py GLUE_RELIES_ON_LEVEL)

At 1 kHz the time constants play out within a few thousand samples; the input is a noise floor with two tone bursts, so
the gate opens and closes inside the run.

    LUARADIO_REFERENCE=<luaradio checkout> python tests/golden/make_level_golden.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.join(ROOT, "tests", "golden", "level")
SPECS = ("blocks/signal/agc_spec", "blocks/signal/powersquelch_spec")
MODULES = {"AGCBlock": "radio.blocks.signal.agc", "PowerSquelchBlock": "radio.blocks.signal.powersquelch"}

RATE, N = 1000.0, 3000
CALLS = (1, 7, 256, 1000)          # then the rest: ragged process() calls
# (name, Lua constructor, complex input, fields initialize() sets)
AGC_FIELDS = ("power_alpha", "gain_alpha", "target", "threshold", "gain_tau", "power_tau", "average_power", "gain")
SQ_FIELDS = ("alpha", "threshold", "tau", "average_power")
CASES = [
    ("agc_fast_real", "AGCBlock('fast', -20, -45, {gain_tau = 7, power_tau = 0.05})", False, AGC_FIELDS),
    ("agc_slow_complex", "AGCBlock('slow', nil, -45, {power_tau = 0.05})", True, AGC_FIELDS),
    ("agc_custom_real", "AGCBlock('custom', -30, -40, {gain_tau = 0.02, power_tau = 0.1})", False, AGC_FIELDS),
    ("agc_custom_complex", "AGCBlock('custom', -10, nil, {gain_tau = 0.05})", True, AGC_FIELDS),
    ("squelch_real", "PowerSquelchBlock(-40, 123)", False, SQ_FIELDS),
    ("squelch_complex", "PowerSquelchBlock(-30)", True, SQ_FIELDS),
]


def level_input(cplx, seed):
    """-60 dBFS noise floor, 0.1-amplitude tone bursts at samples [500, 1200) and [2000, 2400)."""
    rng = np.random.default_rng(seed)
    t = np.arange(N)
    burst = ((t >= 500) & (t < 1200)) | ((t >= 2000) & (t < 2400))
    if cplx:
        x = 1e-3 * (rng.standard_normal(N) + 1j * rng.standard_normal(N)) / np.sqrt(2) + 0.1 * burst * np.exp(2j * np.pi * 0.05 * t)
        return x.astype(np.complex64)
    return (1e-3 * rng.standard_normal(N) + 0.1 * burst * np.cos(2 * np.pi * 0.05 * t)).astype(np.float32)


def chunks(n):
    out, i = [], 0
    for c in CALLS:
        out.append((i, i + c))
        i += c
    out.append((i, n))
    return out


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
        print("%-20s %-18s %d vectors  eps=%s" % (os.path.basename(spec), block, len(vectors), epsilon))


def write_executed(E):
    out = {}
    for k, (name, ctor, cplx, fields) in enumerate(CASES):
        it, types = E.make_env(lib=None, cuda=False)
        for mod in MODULES.values():
            with open(os.path.join(E.REF, mod.replace(".", "/") + ".lua")) as f:
                it.modules[mod] = f.read()
        cls = ctor.split("(", 1)[0]
        blk = it.run("""
            local %s = require('%s')
            local types = require('radio.types')
            local blk = %s
            blk:differentiate({%s})
            blk.inputs[1].pipe = {get_rate = function () return %r end}
            blk:initialize()
            return blk
        """ % (cls, MODULES[cls], ctor, "types.ComplexFloat32" if cplx else "types.Float32", RATE))[0]
        x = level_input(cplx, k)
        ys = []
        for a, b in chunks(N):
            ys.append(it.f32.to_numpy(it.call(it.index(blk, "process"), [blk, it.f32.vector_from_numpy(x[a:b])])[0]))
        out[name + "_x"] = x
        out[name + "_y"] = np.concatenate(ys).astype(x.dtype)
        for f in fields:
            out["%s_%s" % (name, f)] = np.float64(blk.hash[f])
        print("%-20s %s" % (name, " ".join("%s=%.17g" % (f, blk.hash[f]) for f in fields)))
    np.savez_compressed(os.path.join(HERE, "level_reference_executed.npz"), **out)


def write_hooks(ref):
    from tests.test_level_oracle import GLUE_RELIES_ON_LEVEL
    found = {}
    for rel, needle in sorted(GLUE_RELIES_ON_LEVEL):
        if needle in open(os.path.join(ref, rel)).read():
            found.setdefault(rel, []).append(needle)
    with open(os.path.join(HERE, "level_glue_hooks.json"), "w") as f:
        json.dump({"present": found}, f, separators=(",", ":"))


def main():
    os.environ["LUARADIO_DISABLE_CUDA"] = "1"
    from tests import lua_reference_env as E
    if not E.available():
        sys.exit("set LUARADIO_REFERENCE to a luaradio checkout")
    os.makedirs(HERE, exist_ok=True)
    write_specs(E.REF)
    write_executed(E)
    write_hooks(E.REF)
    print("wrote", HERE)


if __name__ == "__main__":
    main()
