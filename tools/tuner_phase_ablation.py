#!/usr/bin/env python3
"""Which phase of the tuner+discriminator kernel (luaradio_b200/csrc/tuner.cu, the interior kernel of the WBFM-mono chain's
first stage) is exposed: the chain timed by `bench.py --profile --no-check` on this code and on timing-only builds of it
(LRB_PT_EXPERIMENT, each built with LRB200_NVCC_EXTRA in a temporary copy of the package; their outputs are wrong):

  no_wait              after a CTA's first tile no copy is issued or waited for: later tiles compute on stale shared memory
  no_rotation_math     the tile is copied, waited for, loaded and stored as before, without the translator's complex multiplies
  no_discrim_epilogue  the imaginary part of y[m] conj(y[m-1]) is stored instead of its angle (no atan2)
  no_mac               the MAC loop is skipped

The builds run alternately, `--repeats` rounds of all of them in one call; every record carries the card's name, power
limit and SM clocks as read right after the run.  One JSON object on stdout.  Needs a GPU.

    python tools/tuner_phase_ablation.py > profiles/h100_700w_tuner_phase_ablation.json
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

VARIANTS = {
    "this_code": "",
    "no_wait": "-DLRB_PT_EXPERIMENT=3",
    "no_rotation_math": "-DLRB_PT_EXPERIMENT=4",
    "no_discrim_epilogue": "-DLRB_PT_EXPERIMENT=5",
    "no_mac": "-DLRB_PT_EXPERIMENT=2",
}
STAGE = "tuner+discrim(128,/5)"


def build_variant(name, flags, tmp):
    d = os.path.join(tmp, name)
    shutil.copytree(os.path.join(ROOT, "luaradio_b200"), os.path.join(d, "luaradio_b200"),
                    ignore=shutil.ignore_patterns("__pycache__", "*.so", "_build"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(d, "include"))
    env = dict(os.environ, PYTHONPATH=d, LRB200_NVCC_EXTRA=flags)
    out = subprocess.run([sys.executable, "-m", "luaradio_b200.build"], cwd=d, env=env, check=True,
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[-1]


def run_bench(lib, args):
    from tools.aux_bench import card
    env = dict(os.environ, LRB200_LIB=lib)
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup),
           "--profile", "--no-check"]
    out = subprocess.run(cmd, cwd=ROOT, env=env, check=True, capture_output=True, text=True)
    rec = json.loads(out.stdout.strip().splitlines()[-1])
    return {"ms_per_step": round(rec["ms_per_step"], 4), "stage_ms": round(rec["stages_ms"][STAGE], 4),
            "stages_ms": {k: round(v, 4) for k, v in rec["stages_ms"].items()}, "card": card()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    names = list(VARIANTS)
    result = {"command": "python tools/tuner_phase_ablation.py", "bench": "bench.py --gpus 1 --steps %d --warmup %d --profile --no-check"
              % (args.steps, args.warmup), "flags": {n: VARIANTS[n] for n in names}, "runs": {n: [] for n in names}}
    with tempfile.TemporaryDirectory() as tmp:
        libs = {n: build_variant(n, VARIANTS[n], tmp) for n in names}
        for _ in range(args.repeats):
            for n in names:
                result["runs"][n].append(run_bench(libs[n], args))
    result["stage_ms_mean"] = {n: round(sum(r["stage_ms"] for r in rs) / len(rs), 4) for n, rs in result["runs"].items()}
    result["step_ms_mean"] = {n: round(sum(r["ms_per_step"] for r in rs) / len(rs), 4) for n, rs in result["runs"].items()}
    print(json.dumps(result))


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()
