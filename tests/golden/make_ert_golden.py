#!/usr/bin/env python3
"""Golden data for ManchesterMatchedFilterBlock, written to tests/golden/ert/ from a luaradio checkout: the reference's
own spec vectors (tests/blocks/signal/manchestermatchedfilter_spec.gen.lua) in make_golden.py's BlockSpec layout.  They
live in a sub-directory of their own, as the RDS and level-control vectors do, and are pinned by tests/test_ert_ref.py.

    LUARADIO_REFERENCE=<luaradio checkout> python tests/golden/make_ert_golden.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

OUT = os.path.join(HERE, "ert")
SPECS = ("blocks/signal/manchestermatchedfilter_spec",)


def main():
    os.makedirs(OUT, exist_ok=True)
    for spec in SPECS:
        block, vectors, epsilon = mg.parse_block_spec(os.path.join(mg.REF, "tests", spec + ".gen.lua"))
        arrays, man = {}, {"block": block, "epsilon": epsilon, "source": "tests/" + spec + ".gen.lua", "vectors": []}
        for i, v in enumerate(vectors):
            args = [mg.jsonable_arg(a, arrays, "v%d_arg%d" % (i, k)) for k, a in enumerate(v["args"])]
            for j, a in enumerate(v["inputs"]):
                arrays["v%d_in%d" % (i, j)] = a
            for j, a in enumerate(v["outputs"]):
                arrays["v%d_out%d" % (i, j)] = a
            man["vectors"].append({"desc": v["desc"], "args": args, "n_in": len(v["inputs"]), "n_out": len(v["outputs"])})
        arrays["manifest"] = np.array(json.dumps(man))
        np.savez_compressed(os.path.join(OUT, os.path.basename(spec) + ".npz"), **arrays)
        print("%-34s %-30s %3d vectors  eps=%s" % (os.path.basename(spec), block, len(vectors), epsilon))


if __name__ == "__main__":
    sys.exit(main())
