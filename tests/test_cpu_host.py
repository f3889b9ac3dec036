"""CPU-side tests (no GPU): the C-ABI library loads and exports every declared symbol, product tap
design matches the reference's golden vectors, flow-graph construction follows the reference's rules,
and every compute entry point fails LOUDLY without a CUDA device (no CPU fallback)."""
import os
import re

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from luaradio_b200.types import ComplexFloat32, Float32, Vector
from tests.golden_util import GOLDEN_DIR, epsilon_ok

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _have_gpu():
    try:
        return _lib.load().lrb200_device_count() > 0
    except Exception:
        return False


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "lrb200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = sorted(set(re.findall(r"\b(lrb200_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) > 40
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), "declared in include/lrb200.h but not exported: " + name
    assert set(declared) == set(_lib.EXPORTED_SYMBOLS), set(declared) ^ set(_lib.EXPORTED_SYMBOLS)
    assert b"sm_90a" in lib.lrb200_version()


def test_every_block_create_function_is_in_the_bounds_harness():
    """Every lrb200_*_create entry point of the header is a case of tests/test_gpu_bounds.py (guard bands, poison,
    unaligned placements) or is named in its commented exclusion list: a new block cannot skip the harness."""
    from tests import test_gpu_bounds as bounds
    hdr = open(os.path.join(ROOT, "include", "lrb200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(lrb200_[a-z0-9_]*_create[a-z0-9_]*)\s*\(", hdr))
    assert len(declared) > 20
    covered = bounds.covered_create_functions()
    assert not covered & bounds.BOUNDS_EXCLUDED_CREATE
    missing = declared - covered - bounds.BOUNDS_EXCLUDED_CREATE
    assert not missing, "create entry points without a buffer-boundary case: %s" % sorted(missing)
    assert covered | bounds.BOUNDS_EXCLUDED_CREATE <= declared, sorted((covered | bounds.BOUNDS_EXCLUDED_CREATE) - declared)


def test_no_cpu_fallback_without_device():
    if _have_gpu():
        pytest.skip("a GPU is present")
    lib = _lib.load()
    assert lib.lrb200_init(0) != 0
    assert b"no CPU fallback" in lib.lrb200_last_error()
    taps = np.ones(4, np.float32)
    assert not lib.lrb200_fir_create_crcf(taps.ctypes.data, 4, 1, 0)
    assert not lib.lrb200_graph_create()
    blk = radio.LowpassFilterBlock(128, 0.2)
    blk.get_rate = lambda: 2.0
    blk.differentiate([ComplexFloat32])
    with pytest.raises(_lib.LibraryError):
        blk.initialize()


def test_product_tap_design_matches_reference_vectors():
    fu = radio.filter_utils
    z = np.load(GOLDEN_DIR + "/filter_utils_vectors.npz")
    cases = {
        "firwin_lowpass": fu.firwin_lowpass(128, 0.5), "firwin_highpass": fu.firwin_highpass(129, 0.5),
        "firwin_bandpass": fu.firwin_bandpass(129, [0.4, 0.6]), "firwin_bandstop": fu.firwin_bandstop(129, [0.4, 0.6]),
        "firwin_complex_bandpass_positive": fu.firwin_complex_bandpass(129, [0.1, 0.3]),
        "firwin_complex_bandpass_negative": fu.firwin_complex_bandpass(129, [-0.1, -0.3]),
        "firwin_complex_bandpass_zero": fu.firwin_complex_bandpass(129, [-0.2, 0.2]),
        "firwin_complex_bandstop_positive": fu.firwin_complex_bandstop(129, [0.1, 0.3]),
        "firwin_complex_bandstop_negative": fu.firwin_complex_bandstop(129, [-0.1, -0.3]),
        "firwin_complex_bandstop_zero": fu.firwin_complex_bandstop(129, [-0.2, 0.2]),
        "fir_hilbert_transform": fu.fir_hilbert_transform(129),
    }
    for k, h in cases.items():
        h = np.asarray(h)
        h = h.astype(np.complex64 if np.iscomplexobj(h) else np.float32)
        ok, msg = epsilon_ok(h, z[k], 1e-6)
        assert ok, "%s: %s" % (k, msg)
    w = np.load(GOLDEN_DIR + "/window_utils_vectors.npz")
    for name in ("rectangular", "hamming", "hanning", "bartlett", "blackman"):
        for per in (False, True):
            key = "window_" + name + ("_periodic" if per else "")
            ok, msg = epsilon_ok(np.array(radio.window_utils.window(len(w[key]), name, per), np.float32), w[key], 1e-6)
            assert ok, "%s: %s" % (key, msg)


def test_type_signatures_and_differentiate():
    f = radio.FIRFilterBlock([0.2] * 5)
    f.differentiate([Float32])
    assert f.get_output_type() is Float32
    f = radio.FIRFilterBlock([0.2] * 5)
    f.differentiate([ComplexFloat32])
    assert f.get_output_type() is ComplexFloat32
    f = radio.FIRFilterBlock(ComplexFloat32.vector_from_array([1 + 1j, 0.5]))
    with pytest.raises(AssertionError):
        f.differentiate([Float32])            # complex taps have no real-input signature (firfilter.lua:68-73)
    d = radio.FrequencyDiscriminatorBlock(1.25)
    d.differentiate([ComplexFloat32])
    assert d.get_output_type() is Float32
    with pytest.raises(AssertionError):
        radio.HilbertTransformBlock(128)      # even tap count
    with pytest.raises(AssertionError):
        radio.FrequencyTranslatorBlock(None)


def test_composite_graph_building_and_rates():
    src = radio.ArraySource(np.zeros(100, np.complex64), 1102500.0)
    snk = radio.ArraySink()
    top = radio.CompositeBlock()
    tuner = radio.TunerBlock(-250e3, 200e3, 5)
    ds = radio.DownsamplerBlock(5)
    top.connect(src, tuner, radio.FrequencyDiscriminatorBlock(1.25), radio.LowpassFilterBlock(128, 15e3),
                radio.FMDeemphasisFilterBlock(75e-6), ds, snk)
    top._validate_inputs()
    top._differentiate()
    conns = top._crawl_connections()
    # hierarchical tuner flattened to its three concrete blocks: 7 blocks + sink input => 8 edges
    assert len(conns) == 8
    for inp, outp in conns.items():
        p = radio.block.Pipe(outp, inp)
        outp.pipes.append(p)
        inp.pipe = p
    assert snk.get_rate() == pytest.approx(1102500.0 / 25)
    assert ds.inputs[0].pipe.get_rate() == pytest.approx(220500.0)
    # an unconnected input is an error (composite.lua:302-312)
    top2 = radio.CompositeBlock()
    a, b = radio.FrequencyTranslatorBlock(1.0), radio.ComplexMagnitudeBlock()
    top2.connect(a, b)
    with pytest.raises(AssertionError):
        top2._validate_inputs()
    # an input can only be driven once
    with pytest.raises(AssertionError):
        top2.connect(radio.FrequencyTranslatorBlock(2.0), "out", b, "in")


def test_vector_semantics():
    v = ComplexFloat32.vector(4)
    assert v.length == 4 and v.size == 32 and np.all(v.data == 0)
    v.resize(2)
    assert v.length == 2
    v.resize(6)
    assert v.length == 6 and v.data.dtype == np.complex64
    f = Float32.vector_from_array([1, 2, 3])
    assert f.size == 12
    c = Vector.cast(np.arange(4, dtype=np.float32))
    assert c.data_type is Float32 and c.length == 4


def test_file_block_host_logic_without_gpu(tmp_path):
    """The parts of the file sources/sinks that are plain host I/O: raw-chunk reading (whole samples, EOF, repeat),
    RawFileSource/RawFileSink round trip, WAV header bytes, argument errors.  (The format conversion itself needs the GPU.)"""
    import io
    import numpy as np
    import luaradio_b200 as radio
    from luaradio_b200.types import ComplexFloat32, Float32, Vector
    from oracle import lr_oracle as O
    # IQFileSource.read_raw: 10 s16 I/Q samples + 3 stray bytes, chunks of 4 samples
    raw = bytes(range(43))
    src = radio.IQFileSource(raw, "s16le", 1000, chunk=4)
    src.differentiate([])
    src.initialize()
    got = []
    while True:
        c = src.read_raw()
        if c is None:
            break
        got.append(bytes(c))
    assert [len(c) for c in got] == [16, 16, 8] and b"".join(got) == raw[:40]
    assert src.get_rate() == 1000 and src.sample_bytes == 4
    rep = radio.RealFileSource(bytes(range(6)), "u16be", 1, repeat_on_eof=True, chunk=2)
    rep.differentiate([])
    rep.initialize()
    assert [bytes(rep.read_raw()) for _ in range(4)] == [bytes([0, 1, 2, 3]), bytes([4, 5]), bytes([0, 1, 2, 3]), bytes([4, 5])]
    with pytest.raises(AssertionError):
        radio.IQFileSource(raw, "u12", 1)
    with pytest.raises(AssertionError):
        radio.IQFileSink(io.BytesIO(), "s24le")
    # RawFileSink -> RawFileSource round trip through a real file
    x = (np.arange(1000) + 1j * np.arange(1000, 2000)).astype(np.complex64)
    path = str(tmp_path / "raw.bin")
    snk = radio.RawFileSink(path)
    snk.differentiate([ComplexFloat32])
    snk.initialize()
    snk.process(Vector.cast(x[:600]))
    snk.process(Vector.cast(x[600:]))
    snk.cleanup()
    rsrc = radio.RawFileSource(path, ComplexFloat32, 48000, chunk=256)
    rsrc.differentiate([])
    rsrc.initialize()
    outs = []
    while True:
        v = rsrc.process()
        if v is None:
            break
        outs.append(np.array(v.data, copy=True))
    assert [len(o) for o in outs] == [256, 256, 256, 232] and np.array_equal(np.concatenate(outs), x)
    # WAV header for every (bits, channels) of the reference's sink spec, from the sink's own header()
    from tests.test_oracle_golden import WAV_HEADERS
    for (bits, ch), hexs in WAV_HEADERS.items():
        w = radio.WAVFileSink(io.BytesIO(), ch, bits)
        w.get_rate = lambda: 44100
        w.count = 256
        assert w.header() == bytes.fromhex(hexs.replace(" ", "")) == O.wav_header(256, ch, bits, 44100)
        assert w.raw_sink == (ch == 1)


def test_public_header_is_plain_c(tmp_path):
    """include/lrb200.h is the drop-in boundary: it must compile as C99 and as C++ on its own (plain pointers and sizes,
    no CUDA / torch types), and a C program must link against the library using only that header."""
    import os
    import shutil
    import subprocess
    from luaradio_b200 import _lib
    if not shutil.which("gcc"):
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "use.c"
    src.write_text('#include "lrb200.h"\n#include <stdio.h>\n'
                   'int main(void) {\n'
                   '    float32_t taps[3] = {{0.25f}, {0.5f}, {0.25f}};\n'
                   '    lrb200_block_t *q = lrb200_fir_create_crcf(taps, 3, 1, LRB200_HOST);\n'
                   '    if (!q) { printf("%s\\n", lrb200_last_error()); return lrb200_device_count() > 0; }\n'
                   '    lrb200_block_destroy(q);\n    return 0;\n}\n')
    inc = os.path.join(root, "include")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", inc, "-fsyntax-only", str(src)], check=True)
    subprocess.run(["g++", "-std=c++11", "-Wall", "-Werror", "-I", inc, "-fsyntax-only", "-x", "c++", str(src)], check=True)
    libpath = _lib.LIB_PATH
    exe = tmp_path / "use"
    subprocess.run(["gcc", "-std=c99", "-I", inc, str(src), "-o", str(exe), libpath, "-Wl,-rpath," + os.path.dirname(libpath)], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    # on a box without a GPU the create call fails loudly with the library's own message and the program exits 0
    assert r.returncode == 0, r.stdout + r.stderr


def test_scheduler_plans_maximal_gpu_runs_in_a_dag():
    """CompositeBlock._plan_gpu_runs (the pure planning half of the GPU scheduler; its Lua twin is
    lua/radio_b200/composite_patch.lua: collapse_gpu_runs): linear chain, fan-out, a two-input junction, a host block in the
    middle, and the WBFM-stereo composite -- no device needed, nothing is initialised."""
    import luaradio_b200 as radio
    from luaradio_b200.block import Block, Input, Output
    from luaradio_b200.types import ComplexFloat32

    def plan(top):
        top._prepare_to_run(initialize=False)
        return [[b.name for b in run] for run, _, _ in top._plan_gpu_runs()]

    x = np.zeros(16, np.complex64)
    # 1. the mono chain: one run of all seven concrete blocks
    top = radio.CompositeBlock()
    top.connect(radio.ArraySource(x, 1102500.0), radio.TunerBlock(-250e3, 200e3, 5), radio.FrequencyDiscriminatorBlock(1.25),
                radio.LowpassFilterBlock(128, 15e3), radio.FMDeemphasisFilterBlock(75e-6), radio.DownsamplerBlock(5), radio.ArraySink())
    assert plan(top) == [["FrequencyTranslatorBlock", "LowpassFilterBlock", "DownsamplerBlock", "FrequencyDiscriminatorBlock",
                          "LowpassFilterBlock", "FMDeemphasisFilterBlock", "DownsamplerBlock"]]

    # 2. a host block splits the graph into two runs; a fan-out ends a run; single blocks stay on their own handle
    class Host(Block):
        name = "Host"

        def instantiate(self):
            self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])

    top = radio.CompositeBlock()
    a1, a2, host, b1, b2, c1 = radio.FrequencyTranslatorBlock(1e5), radio.LowpassFilterBlock(64, 2e5), Host(), radio.DownsamplerBlock(2), \
        radio.ComplexMagnitudeBlock(), radio.ComplexToRealBlock()
    top.connect(radio.ArraySource(x, 1e6), a1, a2, host, b1)
    top.connect(b1, b2, radio.ArraySink())
    top.connect(b1, c1, radio.ArraySink())
    assert plan(top) == [["FrequencyTranslatorBlock", "LowpassFilterBlock"]]

    # 3. tests/top_spec.lua topology: two sources into a two-input block, then one run
    top = radio.CompositeBlock()
    mixer = radio.MultiplyConjugateBlock()
    top.connect(radio.ArraySource(x, 1e6), "out", mixer, "in1")
    top.connect(radio.ArraySource(x, 1e6), "out", mixer, "in2")
    top.connect(mixer, radio.LowpassFilterBlock(16, 100e3), radio.FrequencyDiscriminatorBlock(5), radio.DecimatorBlock(25, {"num_taps": 16}),
                radio.ArraySink())
    assert plan(top) == [["LowpassFilterBlock", "FrequencyDiscriminatorBlock", "LowpassFilterBlock", "DownsamplerBlock"]]

    # 4. WBFM stereo: discriminator -> hilbert, and the two lowpass -> complex-to-real arms
    top = radio.CompositeBlock()
    demod = radio.WBFMStereoDemodulator()
    top.connect(radio.ArraySource(x, 220500.0), demod)
    top.connect(demod, "left", radio.ArraySink(), "in")
    top.connect(demod, "right", radio.ArraySink(), "in")
    runs = plan(top)
    assert ["FrequencyDiscriminatorBlock", "HilbertTransformBlock"] in runs
    assert runs.count(["LowpassFilterBlock", "ComplexToRealBlock"]) == 2
    assert all(len(r) >= 2 for r in runs)
    # ... and as a whole it is ONE device DAG: a single external input (the source), two outputs (left, right)
    dags = top._plan_gpu_dags()
    assert len(dags) == 1
    members, ext_in, ext_out = dags[0]
    assert len(members) == 14 and ext_in.owner.name == "ArraySource"
    assert [p.owner.name for p in ext_out] == ["FMDeemphasisFilterBlock", "FMDeemphasisFilterBlock"]
    assert top._plan_gpu_runs({m for m in members}) == []
    # a straight line is no DAG candidate; two external feeds (top_spec topology) keep the set on the host scheduler
    for t in (radio.CompositeBlock(),):
        t.connect(radio.ArraySource(x, 1102500.0), radio.TunerBlock(-250e3, 200e3, 5), radio.FrequencyDiscriminatorBlock(1.25), radio.ArraySink())
        t._prepare_to_run(initialize=False)
        assert t._plan_gpu_dags() == []
    t = radio.CompositeBlock()
    mixer = radio.MultiplyConjugateBlock()
    t.connect(radio.ArraySource(x, 1e6), "out", mixer, "in1")
    t.connect(radio.ArraySource(x, 1e6), "out", mixer, "in2")
    t.connect(mixer, radio.LowpassFilterBlock(16, 100e3), radio.ArraySink())
    t._prepare_to_run(initialize=False)
    assert t._plan_gpu_dags() == []


def test_bench_clock_sampler_with_a_fake_nvidia_smi(tmp_path, monkeypatch):
    """bench.ClockSampler against a stand-in `nvidia-smi` on PATH: it must wait for the first line, keep the load loop going
    until enough samples were taken under load (the timed region is shorter than one sampling period), split the samples
    into timed-region / load, and report throttle reasons."""
    import stat
    import sys
    import time
    fake = tmp_path / "nvidia-smi"
    fake.write_text("#!/bin/sh\nsleep 0.3\nwhile true; do echo '1965, 1965, Not Active, Not Active, Not Active, Active'; sleep 0.02; done\n")
    fake.chmod(fake.stat().st_mode | stat.S_IEXEC)
    monkeypatch.setenv("PATH", str(tmp_path) + os.pathsep + os.environ["PATH"])
    sys.path.insert(0, ROOT)
    import bench
    s = bench.ClockSampler(0)
    s.start()
    t0 = time.monotonic()
    assert s.wait_ready() and time.monotonic() - t0 >= 0.25           # blocked through the slow start-up
    s.load_begin()
    steps = []
    th0 = time.monotonic()
    time.sleep(0.005)                                                  # a "timed region" far shorter than a period
    s.mark(th0, time.monotonic())
    s.continue_load(lambda: steps.append(1), lambda: time.sleep(0.01))
    c = s.stop()
    assert c["samples"] >= bench.ClockSampler.MIN_LOAD and len(steps) >= 8
    assert c["sm_mhz"] == 1965.0 and c["sm_max_mhz"] == 1965.0 and c["reasons"] == ["sw_power_cap"]
    assert c["samples_in_timed_region"] <= 1
    # no nvidia-smi at all: an explicit reason, never a silent empty record
    monkeypatch.setenv("PATH", str(tmp_path / "nowhere"))
    s = bench.ClockSampler(0)
    s.start()
    assert not s.wait_ready(timeout=0.2)
    assert s.stop()["reasons"] == ["nvidia-smi unavailable"]
