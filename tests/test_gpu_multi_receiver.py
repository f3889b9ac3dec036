"""Receivers that share one source, run as ONE device DAG (the planner merges them): three NBFM receivers and one
WBFM-mono receiver on a 2.4 MS/s capture.

  * the merged DAG computes bit for bit what the per-receiver chains (run(device_dag=False)) compute from the same
    8192-sample vectors, and in super-chunks what the chains compute in super-chunks of the same size; against the
    8192-sample stream the super-chunks agree within the stream tolerance of tests/test_gpu_dag_boundary.py;
  * from a u8 IQFileSource the converter is the DAG's first node and only the DAG reads the file;
  * a WBFM-stereo receiver next to a mono one keeps the stereo DAG's outputs;
  * lrb200_dag_execute_device equals lrb200_dag_execute bit for bit;
  * the merged DAG's halo is the largest of the receivers' own, and its shards match the stream;
  * a reset DAG, and a second run() of the same top block, repeat the outputs."""
import ctypes

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from luaradio_b200.composite import GPUDagBlock
from oracle import lr_oracle as O
from tests.test_gpu_dag import rnd_c
from tests.test_gpu_dag_boundary import (CASES, VECTOR, cmp_rel, cmp_stereo, counting, host_execute, planned_dag, release,
                                         stereo_input, stereo_top)
from tests.test_gpu_dag_shard import Ranks, single

pytestmark = pytest.mark.gpu

RATE = 2.4e6
N = 1 << 22
NBFM_OFFSETS = (-600e3, -200e3, 300e3)
WBFM_OFFSET = 700e3
DECIMATION = 10                       # every receiver at 240 kHz: one output period, so the halos compare directly


def capture(n, seed):
    """Three narrowband FM carriers and one broadcast FM carrier at the receivers' offsets, plus noise, within [-1, 1]."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / RATE
    x = np.zeros(n, np.complex128)
    for k, f in enumerate(NBFM_OFFSETS):
        tone = np.sin(2 * np.pi * (700 + 400 * k) * t)
        x += 0.2 * np.exp(1j * (2 * np.pi * f * t + 2 * np.pi * 3e3 * np.cumsum(tone) / RATE))
    tone = 0.5 * np.sin(2 * np.pi * 1000 * t) + 0.4 * np.sin(2 * np.pi * 3100 * t)
    x += 0.2 * np.exp(1j * (2 * np.pi * WBFM_OFFSET * t + 2 * np.pi * 75e3 * np.cumsum(tone) / RATE))
    return (x + 0.01 * rnd_c(rng, n)).astype(np.complex64)


def receivers_top(x, chunk=VECTOR, src=None):
    src = src if src is not None else radio.ArraySource(x, RATE, chunk)
    top, sinks = radio.CompositeBlock(), []
    for f in NBFM_OFFSETS:
        sinks.append(radio.ArraySink())
        top.connect(src, radio.TunerBlock(f, 25e3, DECIMATION), radio.NBFMDemodulator(5e3, 4e3), sinks[-1])
    sinks.append(radio.ArraySink())
    top.connect(src, radio.TunerBlock(WBFM_OFFSET, 200e3, DECIMATION), radio.WBFMMonoDemodulator(), sinks[-1])
    return top, sinks


def run(make, x, **kw):
    top, sinks = make(x)
    top.run(**kw)
    return top, [s.result() for s in sinks]


def same_bits(got, ref, what):
    assert len(got) == len(ref), what
    for k, (g, r) in enumerate(zip(got, ref)):
        assert len(g) == len(r) > 0, "%s port %d: %d samples, %d expected" % (what, k, len(g), len(r))
        assert np.array_equal(g.view(np.uint8), r.view(np.uint8)), "%s port %d differs" % (what, k)


@pytest.fixture(scope="module")
def x():
    return capture(N, 41)


@pytest.fixture(scope="module")
def per_chain(x):
    top, outs = run(receivers_top, x, device_dag=False)
    desc = top.describe_gpu_graph()
    assert "dag{" not in desc and len(top._chains) == 4, desc
    return outs


def test_merged_dag_equals_the_per_receiver_chains(x, per_chain):
    top, outs = run(receivers_top, x)
    desc = top.describe_gpu_graph()
    assert desc.startswith("dag{") and desc.count("dag{") == 1 and len(top._chains) == 1, desc
    assert len(top._chains[0].ext_out) == 4
    same_bits(outs, per_chain, "8192-sample vectors")


def test_merged_dag_in_superchunks(x, per_chain):
    S = 1 << 20
    _, outs = run(receivers_top, x, superchunk=S)
    _, chains = run(receivers_top, x, superchunk=S, device_dag=False)
    same_bits(outs, chains, "super-chunks of %d" % S)
    for k, (g, r) in enumerate(zip(outs, per_chain)):
        assert len(g) == len(r)
        cmp_rel(1e-5)(g, r, "super-chunk port %d" % k)


def test_u8_file_source_is_absorbed_into_the_merged_dag(x):
    raw = np.clip(np.round(np.stack([x.real, x.imag], 1).reshape(-1) * 127.5 + 127.5), 0, 255).astype(np.uint8)
    conv = O.iq_file_convert(raw, "u8")
    for sc in (0, 1 << 20):
        src = radio.IQFileSource(raw.tobytes(), "u8", RATE)
        calls = counting(src)
        top, sinks = receivers_top(None, src=src)
        top.run(superchunk=sc)
        desc = top.describe_gpu_graph()
        assert desc.startswith("dag{iqconv(u8) ; ") and desc.count("dag{") == 1 and len(top._chains) == 1, desc
        read = GPUDagBlock.RAW_READ
        assert calls == [read] * (-(-len(conv) // read) + 1) and src._handle is None
        # the same calls on the host-converted samples, per receiver
        _, ref = run(lambda y: receivers_top(y, chunk=read), conv, superchunk=sc, device_dag=False)
        for k, s in enumerate(sinks):
            assert len(s.result()) == len(ref[k]) == -(-len(conv) // DECIMATION)
            cmp_rel(1e-5)(s.result(), ref[k], "sc=%d port %d" % (sc, k))


def test_stereo_next_to_a_mono_receiver():
    y = stereo_input(N, 42)

    def both(z):
        src = radio.ArraySource(z, 1102500.0, VECTOR)
        top, sinks = stereo_top(None, src=src)
        mono = radio.ArraySink()
        top.connect(src, radio.TunerBlock(-250e3, 200e3, 5), radio.WBFMMonoDemodulator(), mono)
        return top, sinks + [mono]

    top, outs = run(both, y)
    assert top.describe_gpu_graph().count("dag{") == 1 and len(top._chains) == 1
    _, alone = run(stereo_top, y)
    for k in range(2):
        assert len(outs[k]) == len(alone[k])
        cmp_stereo(outs[k], alone[k], "stereo port %d next to a mono receiver" % k)

    def mono_only(z):
        top, mono = radio.CompositeBlock(), radio.ArraySink()
        top.connect(radio.ArraySource(z, 1102500.0, VECTOR), radio.TunerBlock(-250e3, 200e3, 5), radio.WBFMMonoDemodulator(), mono)
        return top, [mono]
    _, mono = run(mono_only, y)
    same_bits(outs[2:], mono, "mono receiver next to the stereo one")


RAGGED = (0, 1, 8192, 100003, 5, 3 * 65536 + 7, 0, 333333, 2)


def test_execute_device_equals_execute(x):
    lib = _lib.require_device()
    xs_all = x[:sum(RAGGED)]
    top_h, dag_h = planned_dag(receivers_top, xs_all)
    top_d, dag_d = planned_dag(receivers_top, xs_all)
    maxn = max(RAGGED)
    sizes = [p.data_type.dtype.itemsize for p in dag_d.ext_out]
    dx = lib.lrb200_malloc(maxn * 8)
    dys = [lib.lrb200_malloc(max(1, lib.lrb200_dag_max_output(dag_d.dag, k, maxn)) * s) for k, s in enumerate(sizes)]
    try:
        pos = 0
        for n in RAGGED:
            xs = np.ascontiguousarray(xs_all[pos:pos + n])
            pos += n
            want = host_execute(lib, dag_h, xs)
            if n:
                _lib.check(lib.lrb200_memcpy_h2d(dx, xs.ctypes.data, n * 8), "h2d")
            n_out = (ctypes.c_size_t * len(dys))()
            _lib.check(lib.lrb200_dag_execute_device(dag_d.dag, dx, n, (ctypes.c_void_p * len(dys))(*dys), n_out), "execute_device")
            _lib.check(lib.lrb200_sync(), "sync")
            for k, w in enumerate(want):
                assert n_out[k] == len(w), "n=%d port %d: %d outputs, host mode %d" % (n, k, n_out[k], len(w))
                got = np.zeros(len(w), w.dtype)
                if len(w):
                    _lib.check(lib.lrb200_memcpy_d2h(got.ctypes.data, dys[k], len(w) * sizes[k]), "d2h")
                assert np.array_equal(got.view(np.uint8), w.view(np.uint8)), "n=%d port %d differs from host mode" % (n, k)
    finally:
        lib.lrb200_free(dx)
        for d in dys:
            lib.lrb200_free(d)
        release(top_h)
        release(top_d)


def receiver_halo(lib, top, k):
    """The halo of receiver k's own device DAG (one linear graph node), built from the prepared top block."""
    conns = top._all_connections
    src_port = next(p for p in conns.values() if p.owner.name == "ArraySource")
    consumers = {}
    for i, o in conns.items():
        consumers.setdefault(o.owner, []).append(i.owner)
    chain, b = [], consumers[src_port.owner][k]
    while b.name != "ArraySink":
        chain.append(b)
        b = consumers[b][0]
    dag = GPUDagBlock(chain, src_port, [chain[-1].outputs[0]], conns)
    dag.initialize()
    try:
        return lib.lrb200_dag_halo(dag.dag)
    finally:
        dag.cleanup()


def test_halo_and_shards_of_the_merged_dag(x, monkeypatch):
    lib = _lib.require_device()
    top, dag = planned_dag(receivers_top, x)
    try:
        halo = lib.lrb200_dag_halo(dag.dag)
        own = [receiver_halo(lib, top, k) for k in range(4)]
        print("merged halo", halo, "receivers", own)
        assert halo > 0 and halo == max(own)
    finally:
        release(top)
    # a first and a second shard on one device against the stream (lrb200_dag_execute_device of all of it)
    monkeypatch.setitem(CASES, "receivers", (receivers_top, lambda: x, cmp_rel(1e-5), cmp_rel(1e-5)))
    ref = single(lib, "receivers", x, 0)
    ranks = Ranks(lib, "receivers", x, 2, 0)
    try:
        got, per_rank, reruns, _ = ranks.run()
        assert ranks.halo == halo and ranks.nb == 0 and reruns == [0, 0]
        for k in range(len(ref)):
            assert got[k].shape == ref[k].shape, "port %d: %d outputs, the stream %d" % (k, len(got[k]), len(ref[k]))
            err = float(np.max(np.abs(got[k].astype(np.float64) - ref[k]), initial=0))
            print("port %d: shards vs stream max abs err %.3g" % (k, err))
            cmp_rel(1e-5)(got[k], ref[k], "shards port %d" % k)
        r0 = single(lib, "receivers", x, 0, ranks.counts[0])
        for k in range(len(ref)):
            assert np.array_equal(per_rank[k][0].view(np.uint8), r0[k].view(np.uint8)), "rank 0 port %d" % k
    finally:
        ranks.close()


def test_reset_and_second_run_repeat_the_outputs(x):
    lib = _lib.require_device()
    y = x[:1 << 20]
    top, dag = planned_dag(receivers_top, y)
    try:
        first = [np.concatenate(o) for o in zip(*[host_execute(lib, dag, np.ascontiguousarray(y[i:i + 65536]))
                                                  for i in range(0, len(y), 65536)])]
        _lib.check(lib.lrb200_dag_reset(dag.dag), "reset")
        again = [np.concatenate(o) for o in zip(*[host_execute(lib, dag, np.ascontiguousarray(y[i:i + 65536]))
                                                  for i in range(0, len(y), 65536)])]
        same_bits(again, first, "after lrb200_dag_reset")
    finally:
        release(top)
    src = radio.ArraySource(y, RATE, VECTOR)
    top, sinks = receivers_top(None, src=src)
    top.run()
    a = [s.result() for s in sinks]
    for s in sinks:
        s.chunks = []
    src.pos = 0
    top.run()
    same_bits([s.result() for s in sinks], a, "second run()")
