"""The POCSAG and AX.25 receivers' signal paths on the GPU, up to their data filters (examples/rtlsdr_pocsag.lua,
rtlsdr_ax25.lua), and the device DAG's FSK-detector rewrite (graph.cu fuse_fsk_detector, FskDetectBlock):

  * the POCSAG graph's diamond is one node `fsk_detect(129)[fused x5]`, five blocks with fuse=False;
  * fused == unfused bit for bit: 8192-sample vectors, ragged calls, super-chunks of 2^20, an absorbed u8 IQFileSource,
    lrb200_dag_execute_device; calls of 1, 8 L - 1, 8 L samples and across a block boundary (both sides of the short-call
    policy, FskDetectBlock::fused);
  * a 2^24-sample capture through the detector alone within tests/fsk_ref.py's per-output bound;
  * shapes the rule leaves alone: unequal tap counts, real taps, a decimating FIR, a fused translator, an intermediate
    that is a DAG output or has a second reader in the DAG, Add for Subtract;
  * the fused node in poisoned guard bands at unaligned offsets and tile-boundary lengths;
  * halo and shards at worlds 2 and 4; reset;
  * both example graphs against the reference's own output (tests/golden/fsk/) and against float64 oracle chains; the
    AX.25 chain as one device chain."""
import contextlib
import ctypes
import os
import tempfile

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from luaradio_b200.composite import GPUDagBlock
from tests import fsk_ref as K
from tests import test_gpu_dag_boundary as B
from tests import test_gpu_dag_shard as SH
from tests.test_gpu_bounds import GUARD, POISON_A, SENTINELS, Guarded

pytestmark = pytest.mark.gpu

VECTOR = 8192
N = 1 << 22                                  # capture samples: 52 428 at the detector
L = 1024 - (K.M - 1)                         # the overlap-save block at M = 129
RAGGED = (1, 8192, 100003, 5, 3 * 65536 + 7, 0, 777777, 2, 1 << 20)


def capture(n=N, seed=41):
    return K.fsk_iq(n, seed)


def detector(src, top, in1=None, in2=None, mag_taps=(K.M, K.M), first=None):
    """The POCSAG receiver's mark/space detector fed by `src`, returning the Subtract (mark into in1, space into in2)."""
    bp1 = first or radio.ComplexBandpassFilterBlock(mag_taps[0], K.MARK)
    bp2 = radio.ComplexBandpassFilterBlock(mag_taps[1], K.SPACE)
    m1, m2 = radio.ComplexMagnitudeBlock(), radio.ComplexMagnitudeBlock()
    sub = radio.SubtractBlock()
    top.connect(src, "out", bp1, "in")
    top.connect(src, "out", bp2, "in")
    top.connect(bp1, m1)
    top.connect(bp2, m2)
    top.connect(m1, "out", sub, "in1")
    top.connect(m2, "out", sub, "in2")
    return sub


def pocsag_top(x, chunk=VECTOR, src=None):
    src = src if src is not None else radio.ArraySource(x, K.CAPTURE_RATE, chunk)
    tuner, snk, top = radio.TunerBlock(K.OFFSET, 12e3, K.DECIM), radio.ArraySink(), radio.CompositeBlock()
    top.connect(src, tuner)
    top.connect(detector(tuner, top), radio.LowpassFilterBlock(128, 1200.0), snk)
    return top, [snk]


class _Vectors(radio.ArraySource):
    """The capture handed out in the ragged vectors [splits[k], splits[k + 1])."""

    def instantiate(self, array, splits):
        radio.ArraySource.instantiate(self, array, K.CAPTURE_RATE)
        self.bounds = list(splits[1:])

    def process(self):
        if not self.bounds:
            return None
        end = self.bounds.pop(0)
        v = radio.Vector.cast(self.array[self.pos:end])
        self.pos = end
        return v


def ax25_top(x, chunk=VECTOR, src=None):
    src = src if src is not None else radio.ArraySource(x, K.CAPTURE_RATE, chunk)
    snk, top = radio.ArraySink(), radio.CompositeBlock()
    top.connect(src, radio.TunerBlock(K.OFFSET, 12e3, K.DECIM),
                radio.NBFMDemodulator(3e3, 3e3), radio.HilbertTransformBlock(129), radio.FrequencyTranslatorBlock(-1700.0),
                radio.LowpassFilterBlock(128, 750.0), radio.FrequencyDiscriminatorBlock(1.25),
                radio.LowpassFilterBlock(128, 1200.0), snk)
    return top, [snk]


@contextlib.contextmanager
def dag_rewrites(on):
    """Device DAGs committed with their rewrites on or off, linear graphs fused either way: the fused detector is then the
    only difference between two runs (fuse=False would also unfuse the tuner, which changes its bits)."""
    lib = _lib.load()
    real = lib.lrb200_dag_set_outputs

    def set_outputs(d, outs, n):
        rc = real(d, outs, n)
        return rc if rc != 0 else lib.lrb200_dag_commit(d, 0)
    if not on:
        lib.lrb200_dag_set_outputs = set_outputs
    try:
        yield
    finally:
        lib.lrb200_dag_set_outputs = real


def run(make, x, rewrite=True, superchunk=0, fuse=True, **kw):
    top, sinks = make(x, **kw)
    with dag_rewrites(rewrite):
        top.run(fuse=fuse, superchunk=superchunk)
    return top.describe_gpu_graph(), [s.result() for s in sinks]


def same(a, b, what):
    assert len(a) == len(b), "%s: %d outputs, unfused %d" % (what, len(a), len(b))
    assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)), \
        "%s: differs from the unfused DAG at %d places" % (what, int(np.sum(np.asarray(a) != np.asarray(b))))


def dag_of(make, x, rewrite):
    """The scheduler's GPUDagBlock of `make`'s graph, initialised with the DAG rewrites on or off."""
    top, _ = make(x)
    top._prepare_to_run()
    with dag_rewrites(rewrite):
        top._collapse_gpu_runs(True, 0)
    dags = [c for c in top._chains if isinstance(c, GPUDagBlock)]
    assert len(dags) == 1
    return top, dags[0]


# ---- the rewrite and its description ------------------------------------------------------------------------------------
def test_description_names_the_fused_node():
    x = capture(1 << 16)
    fused, _ = run(pocsag_top, x)
    plain, _ = run(pocsag_top, x, fuse=False)
    off, _ = run(pocsag_top, x, rewrite=False)
    assert "fsk_detect" not in off and "rot+fir_crcf[fused x3]" in off, off
    assert "fsk_detect(129)[fused x5]" in fused, fused
    assert "fsk_detect" not in plain and plain.count("cmag") == 2 and "subtract_rr" in plain, plain


@pytest.mark.parametrize("mode", ["vectors", "superchunk"])
def test_fused_equals_unfused(mode):
    x = capture()
    sc = (1 << 20) if mode == "superchunk" else 0
    _, a = run(pocsag_top, x, superchunk=sc)
    _, b = run(pocsag_top, x, rewrite=False, superchunk=sc)
    same(a[0], b[0], mode)
    assert len(a[0]) == -(-N // K.DECIM)


def _ragged(make, x, fuse):
    lib = _lib.require_device()
    top, dag = dag_of(make, x, fuse)
    try:
        out, pos = [], 0
        for n in RAGGED:
            out.append(B.host_execute(lib, dag, np.ascontiguousarray(x[pos:pos + n]))[0])
            pos += n
        return np.concatenate(out), dag.desc
    finally:
        B.release(top)


def test_fused_equals_unfused_ragged_calls():
    x = capture(sum(RAGGED))
    a, da = _ragged(pocsag_top, x, True)
    b, db = _ragged(pocsag_top, x, False)
    assert "fsk_detect" in da and "fsk_detect" not in db
    same(a, b, "ragged")


def test_fused_equals_unfused_absorbed_u8_file():
    x = capture()
    raw = np.clip(np.round(np.stack([x.real, x.imag], 1).reshape(-1) * 127.5 + 127.5), 0, 255).astype(np.uint8)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "capture.u8")
        raw.tofile(path)
        res = []
        for rewrite in (True, False):
            top, sinks = pocsag_top(None, src=radio.IQFileSource(path, "u8", K.CAPTURE_RATE))
            with dag_rewrites(rewrite):
                top.run()
            desc = top.describe_gpu_graph()
            assert "iqconv" in desc or "u8" in desc, desc
            res.append(sinks[0].result())
    same(res[0], res[1], "u8 file")
    assert len(res[0]) == -(-N // K.DECIM)


def _device(dag, lib, x, calls):
    dx = lib.lrb200_malloc(max(calls) * 8)
    dy = lib.lrb200_malloc(max(calls) * 4)
    out = []
    try:
        pos = 0
        for n in calls:
            xs = np.ascontiguousarray(x[pos:pos + n])
            pos += n
            _lib.check(lib.lrb200_memcpy_h2d(dx, xs.ctypes.data, n * 8), "h2d")
            n_out = (ctypes.c_size_t * 1)()
            _lib.check(lib.lrb200_dag_execute_device(dag.dag, dx, n, (ctypes.c_void_p * 1)(dy), n_out), "execute_device")
            h = np.zeros(n_out[0], np.float32)
            _lib.check(lib.lrb200_memcpy_d2h(h.ctypes.data, dy, h.nbytes), "d2h")
            _lib.check(lib.lrb200_sync(), "sync")
            out.append(h)
    finally:
        lib.lrb200_free(dx)
        lib.lrb200_free(dy)
    return np.concatenate(out)


def detector_top(x, chunk=VECTOR, **kw):
    """The detector alone on a baseband stream at the detector's rate."""
    src, snk, top = radio.ArraySource(x, K.RATE, chunk), radio.ArraySink(), radio.CompositeBlock()
    top.connect(detector(src, top, **kw), snk)
    return top, [snk]


CALLS = (1, 8 * L - 1, 8 * L, L + 3, 2 * L - 5, 8 * L + L + 1, 5, 100003, 8 * L - 1, 1 << 18)


@pytest.mark.parametrize("what", ["detector", "pocsag"])
def test_fused_equals_unfused_execute_device(what):
    """Device-mode calls of 1, 8 L - 1 and 8 L detector inputs and calls across block boundaries: the short calls run the
    members' direct kernels, the others the fused kernel; both equal the unfused DAG."""
    lib = _lib.require_device()
    make = detector_top if what == "detector" else pocsag_top
    calls = CALLS if what == "detector" else tuple(c * K.DECIM for c in CALLS[:8])
    x = K.fsk_iq(sum(calls), 42, offset=0.0, rate=K.RATE) if what == "detector" else capture(sum(calls))
    res = []
    for fuse in (True, False):
        top, dag = dag_of(make, x, fuse)
        try:
            assert ("fsk_detect(129)[fused x5]" in dag.desc) == fuse, dag.desc
            res.append(_device(dag, lib, x, calls))
        finally:
            B.release(top)
    same(res[0], res[1], what)


def test_long_capture_within_the_bound():
    """2^24 detector inputs in one device call (the fused kernel throughout), every output within its bound."""
    lib = _lib.require_device()
    n = 1 << 24
    x = K.fsk_iq(n, 43, offset=0.0, rate=K.RATE)
    top, dag = dag_of(detector_top, x, True)
    try:
        got = _device(dag, lib, x, [n])
    finally:
        B.release(top)
    ha, hb = K.detector_taps()
    ref, bound = K.detector_bound(ha, hb, x)
    r = np.abs(got.astype(np.float64) - ref) / bound
    i = int(np.argmax(r))
    print("\n2^24 samples: at %.3g of the bound (output %d)" % (r[i], i))
    assert r[i] <= 1.0, "output %d off by %.3g, bound %.3g" % (i, abs(got[i] - ref[i]), bound[i])


# ---- shapes the rule leaves alone ---------------------------------------------------------------------------------------
def _nonmatch(kind):
    def make(x, chunk=VECTOR):
        src, snk, top = radio.ArraySource(x, K.RATE, chunk), radio.ArraySink(), radio.CompositeBlock()
        if kind == "unequal":
            out = detector(src, top, mag_taps=(K.M, 65))
        elif kind == "real_taps":
            out = detector(src, top, first=radio.LowpassFilterBlock(K.M, 2000.0))
        elif kind == "translator":
            tr = radio.FrequencyTranslatorBlock(1000.0)
            bp1 = radio.ComplexBandpassFilterBlock(K.M, K.MARK)
            top.connect(tr, bp1)
            top.connect(src, "out", tr, "in")
            out = _detector_from(src, top, tr_first=(tr, bp1))
        elif kind == "decimating":
            out = _detector_from(src, top, decimate=True)
        elif kind == "second_consumer":
            extra = radio.ArraySink()
            top.connect(_detector_from(src, top, extra_sink=extra), snk)
            return top, [snk, extra]
        elif kind == "second_reader":
            extra, scale = radio.ArraySink(), radio.MultiplyConstantBlock(2.0)
            top.connect(_detector_from(src, top, extra_sink=scale), snk)
            top.connect(scale, extra)
            return top, [snk, extra]
        else:                                           # "add"
            out = _detector_from(src, top, add=True)
        top.connect(out, snk)
        return top, [snk]
    return make


def _detector_from(src, top, tr_first=None, decimate=False, add=False, extra_sink=None):
    """The detector with one change: a translator in front of the first FIR, a Downsampler(2) behind each FIR, Add, or
    the first magnitude also read by extra_sink (a sink: a second DAG output; a GPU block: a second reader inside the DAG)."""
    if tr_first:
        tr, bp1 = tr_first
        first = bp1
    else:
        bp1 = radio.ComplexBandpassFilterBlock(K.M, K.MARK)
        top.connect(src, "out", bp1, "in")
        first = bp1
    bp2 = radio.ComplexBandpassFilterBlock(K.M, K.SPACE)
    top.connect(src, "out", bp2, "in")
    m1, m2 = radio.ComplexMagnitudeBlock(), radio.ComplexMagnitudeBlock()
    sub = radio.AddBlock() if add else radio.SubtractBlock()
    if decimate:
        d1, d2 = radio.DownsamplerBlock(2), radio.DownsamplerBlock(2)
        top.connect(first, d1, m1)
        top.connect(bp2, d2, m2)
    else:
        top.connect(first, m1)
        top.connect(bp2, m2)
    top.connect(m1, "out", sub, "in1")
    top.connect(m2, "out", sub, "in2")
    if extra_sink is not None:
        top.connect(m1, "out", extra_sink, "in")
    return sub


@pytest.mark.parametrize("kind", ["unequal", "real_taps", "translator", "decimating", "second_consumer", "second_reader", "add"])
def test_rule_leaves_other_shapes_alone(kind):
    x = K.fsk_iq(300000, 44, offset=0.0, rate=K.RATE)
    da, a = run(_nonmatch(kind), x)
    db, b = run(_nonmatch(kind), x, rewrite=False)
    assert "fsk_detect" not in da, da
    assert da.count("cmag") == 2 or kind == "real_taps", da
    for k in range(len(a)):
        same(a[k], b[k], "%s port %d" % (kind, k))


# ---- guard bands, shards, reset -----------------------------------------------------------------------------------------
GUARD_CALLS = (1, 2, 8 * L - 1, 8 * L, 8 * L + 1, 3 * L + 17, 100003)


def test_fused_node_in_guard_bands():
    """Input and output in guard-banded allocations at unaligned offsets, the input's surroundings poisoned, the output's
    filled with a sentinel: the outputs equal the ones from plain buffers and nothing outside the output is written."""
    lib = _lib.require_device()
    x = K.fsk_iq(sum(GUARD_CALLS), 45, offset=0.0, rate=K.RATE)
    top_r, dag_r = dag_of(detector_top, x, True)
    top_g, dag_g = dag_of(detector_top, x, True)
    try:
        want = _device(dag_r, lib, x, GUARD_CALLS)
        pos, got = 0, []
        for k, n in enumerate(GUARD_CALLS):
            xin = np.ascontiguousarray(x[pos:pos + n])
            pos += n
            ioff, ooff = (8 if k % 2 else 16), (4 if k % 2 else 12)
            gi, go = Guarded(lib, n * 8 + 32), Guarded(lib, n * 4 + 32)
            try:
                img = np.tile(np.array([POISON_A], "<u4").view(np.uint8), gi.size // 4)
                img[GUARD + ioff:GUARD + ioff + n * 8] = xin.view(np.uint8)
                gi.load(img)
                sent = np.tile(np.array([SENTINELS[k % 2]], "<u4").view(np.uint8), go.size // 4)
                go.load(sent)
                n_out = (ctypes.c_size_t * 1)()
                _lib.check(lib.lrb200_dag_execute_device(dag_g.dag, gi.ptr + GUARD + ioff, n,
                                                         (ctypes.c_void_p * 1)(go.ptr + GUARD + ooff), n_out), "execute_device")
                _lib.check(lib.lrb200_sync(), "sync")
                assert n_out[0] == n
                after = go.read()
                lo, hi = GUARD + ooff, GUARD + ooff + n * 4
                assert np.array_equal(after[:lo], sent[:lo]) and np.array_equal(after[hi:], sent[hi:]), "n=%d: written outside" % n
                got.append(after[lo:hi].view(np.float32).copy())
            finally:
                gi.free()
                go.free()
        same(np.concatenate(got), want, "guarded")
    finally:
        B.release(top_r)
        B.release(top_g)


def test_halo_equals_the_unfused_dags():
    lib = _lib.require_device()
    x = capture(1 << 16)
    halos = []
    for fuse in (True, False):
        top, dag = dag_of(pocsag_top, x, fuse)
        try:
            halos.append(lib.lrb200_dag_halo(dag.dag))
        finally:
            B.release(top)
    assert halos[0] == halos[1] > 0, halos


@pytest.mark.parametrize("world", [2, 4])
def test_shards_equal_the_stream(world, monkeypatch):
    lib = _lib.require_device()
    monkeypatch.setitem(B.CASES, "fsk", (pocsag_top, capture, None, None))
    x = capture(1 << 21)
    res = []
    for rewrite in (True, False):
        with dag_rewrites(rewrite):
            ranks = SH.Ranks(lib, "fsk", x, world, 0)
        try:
            assert ("fsk_detect" in ranks.dags[0].desc) == rewrite
            got, _, reruns, _ = ranks.run()
        finally:
            ranks.close()
        assert not any(reruns)
        res.append(got[0])
    want = SH.single(lib, "fsk", x, 0)
    # the fused shards are the unfused DAG's shards bit for bit; a shard starts cold one halo early, so its blocks fall
    # elsewhere than the stream's: equal to it within the fan-out DAG's comparison (tests/test_gpu_dag_shard.py)
    same(res[0], res[1], "world %d shards" % world)
    B.cmp_rel(2e-6)(res[0], want[0], "world %d" % world)


def test_reset_repeats_the_outputs():
    lib = _lib.require_device()
    x = capture(1 << 20)
    top, dag = dag_of(pocsag_top, x, True)
    try:
        a = B.host_execute(lib, dag, x)[0].copy()
        _lib.check(lib.lrb200_dag_reset(dag.dag), "reset")
        b = B.host_execute(lib, dag, x)[0]
    finally:
        B.release(top)
    same(a, b, "after reset")


# ---- the receivers against the float64 oracle chains --------------------------------------------------------------------
def _cmp(got, ref, rel, what):
    tol = rel * max(1.0, float(np.max(np.abs(ref))))
    err = float(np.max(np.abs(got.astype(np.float64) - ref)))
    print("\n%s: max abs err %.3g (tolerance %.3g)" % (what, err, tol))
    assert err <= tol, "%s: max abs err %.3g > %.3g" % (what, err, tol)


def test_pocsag_receiver_against_the_oracle():
    x = capture()
    desc, got = run(pocsag_top, x)
    _cmp(got[0], K.pocsag_oracle(x), 1e-5, "pocsag")


def test_ax25_receiver_stays_on_the_device_and_matches_the_oracle():
    x = K.afsk_nbfm_iq(N, 46)
    top, sinks = ax25_top(x)
    top.run()
    desc = top.describe_gpu_graph()
    # one device chain from the source to the sink: no block of the chain ran on the host
    assert len(top._chains) == 1 and "hilbert" in desc and desc.count("discrim") >= 2, desc
    got, ref = sinks[0].result(), K.ax25_oracle(x)
    assert len(got) == len(ref)
    _cmp(got[K.AX25_SETTLE:], ref[K.AX25_SETTLE:], 1e-5, "ax25")


@pytest.mark.parametrize("name", ["pocsag", "ax25"])
def test_receivers_match_the_reference_golden(name):
    """The example graph through CompositeBlock.run against the reference's own output (tests/golden/fsk/), fed in the
    golden's ragged vectors, at the tolerance of the tuner's goldens (1e-5); AX.25 from fsk_ref.AX25_SETTLE on."""
    x, ref, splits = K.load_golden(name)
    src = _Vectors(x, splits)
    top, sinks = (pocsag_top(None, src=src) if name == "pocsag" else ax25_top(None, src=src))
    top.run()
    assert ("fsk_detect(129)[fused x5]" in top.describe_gpu_graph()) == (name == "pocsag")
    got = sinks[0].result()
    assert len(got) == len(ref)
    skip = K.AX25_SETTLE if name == "ax25" else 0
    _cmp(got[skip:], ref[skip:].astype(np.float64), 1e-5, name + " golden")
