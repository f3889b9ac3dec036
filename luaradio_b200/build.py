"""Build libluaradio_b200.so in-tree with nvcc for sm_90a / H100 (cross-compiles without a GPU).

    python -m luaradio_b200.build [--force]

The .so and the objects under _build/ are build products (git-ignored).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libluaradio_b200.so")
SOURCES = ["capi.cu", "graph.cu", "fir_direct.cu", "fir_fft.cu", "tuner.cu", "elementwise.cu", "iir.cu", "synth.cu", "iqconv.cu", "resample.cu", "aux_blocks.cu", "psd_long.cu", "poly_generic.cu", "level.cu", "phasecorr.cu", "iir_order.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# --split-compile 0: the fully unrolled tuner / FFT kernels are dozens of large kernels per file; let ptxas use every core.
# With it the generated SASS depends on thread scheduling (two variants per file have been seen); LRB200_DETERMINISTIC=1 compiles single-threaded instead: reproducible, ~3x the build time.
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "--split-compile", "1" if os.environ.get("LRB200_DETERMINISTIC") else "0"]
FLAGS += os.environ.get("LRB200_NVCC_EXTRA", "").split()


def _deps():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hdrs.append(os.path.join(os.path.dirname(HERE), "include", "lrb200.h"))
    return hdrs


def _stale(target, srcs):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in srcs)


def build(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    # objects compiled with other flags (another architecture, LRB200_NVCC_EXTRA) are stale whatever their mtimes say
    stamp, flags = os.path.join(BUILD, "flags"), "\n".join([NVCC] + FLAGS) + "\n"
    if not os.path.exists(stamp) or open(stamp).read() != flags:
        force = True
    hdrs = _deps()
    jobs = []
    objs = []
    for src in SOURCES:
        sp = os.path.join(CSRC, src)
        obj = os.path.join(BUILD, src[:-3] + ".o")
        objs.append(obj)
        if force or _stale(obj, [sp] + hdrs):
            cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", sp, "-o", obj]
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        return cmd, r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for cmd, r in ex.map(run, jobs):
                if verbose or r.returncode != 0:
                    sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
                if r.returncode != 0:
                    raise RuntimeError("nvcc failed for " + cmd[-3])
    if jobs or force or _stale(LIB, objs + [os.path.join(CSRC, "exports.map")]):
        # only the C ABI (include/lrb200.h) is exported; the internal lrb:: symbols stay local
        cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs + \
              ["-Xlinker", "--version-script=" + os.path.join(CSRC, "exports.map"), "-lcudart_static", "-lpthread", "-ldl", "-lrt"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    with open(stamp, "w") as f:
        f.write(flags)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
