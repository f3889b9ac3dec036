"""The host <-> device boundary that linear graphs, device DAGs and host-mode blocks share (graph.cu, HostBoundary).

  * a graph reset with super-chunks pending drops them: what the graph hands back afterwards is a fresh graph's stream;
  * a graph's DEVICE-mode and shard runs are refused in super-chunk mode, with the DAG's words, and run once it is off;
  * the split points of a host call stay where they were: a graph's call is cut every 2^23 input samples, a host-mode
    block's every 2^24 (MultiplyConjugate with two inputs, the chunk-parallel PLL with two outputs), and a DAG's call is
    never cut.  Where a stream is cut changes output bits (the chunk-parallel PLL engages by call length, the IIR scan
    restarts its warm-up from a call's start, the FIR's AUTO path depends on n), so these compare bit for bit."""
import ctypes

import numpy as np
import pytest

from luaradio_b200 import _lib
from oracle import lr_oracle as O
from tests.test_gpu_bounds import PLL_ARGS
from tests.test_gpu_dag import rnd_c
from tests.test_gpu_dag_boundary import host_execute, planned_dag, release, stereo_input, stereo_top

pytestmark = pytest.mark.gpu

VEC = 8192                     # the reference's source vectors (zero.lua:30)
S = 1 << 16                    # super-chunk slots of 8 vectors
GRAPH_CHUNK = 1 << 23
BLOCK_CHUNK = 1 << 24
DIRECTLY = "runs the stream directly; switch super-chunk mode off first (set_superchunk 0)"


@pytest.fixture
def lib():
    return _lib.require_device()


@pytest.fixture
def chain(lib):
    """A factory of the rtlsdr_wbfm_mono.lua chain as a committed graph (fused, or not), destroyed after the test."""
    import bench
    made = []

    def make(fuse=1):
        g = bench.build_chain_graph(lib, _lib)
        if not fuse:
            _lib.check(lib.lrb200_graph_commit(g, 0), "commit")
        made.append(g)
        return g
    yield make
    for g in made:
        lib.lrb200_graph_destroy(g)


def graph_calls(lib, g, x, lengths, flush=False):
    """x through lrb200_graph_execute in calls of `lengths` (then lrb200_graph_flush): everything handed back."""
    outs, pos, no = [], 0, ctypes.c_size_t()
    for n in lengths:
        seg = np.ascontiguousarray(x[pos:pos + n])
        y = np.zeros(lib.lrb200_graph_max_output(g, n) + 16, np.float32)
        _lib.check(lib.lrb200_graph_execute(g, seg.ctypes.data, n, y.ctypes.data, ctypes.byref(no)), "graph_execute")
        outs.append(y[:no.value].copy())
        pos += n
    if flush:
        y = np.zeros(lib.lrb200_graph_max_output(g, 0) + 16, np.float32)
        _lib.check(lib.lrb200_graph_flush(g, y.ctypes.data, ctypes.byref(no)), "graph_flush")
        outs.append(y[:no.value].copy())
    return np.concatenate(outs)


def vectors(n):
    return [VEC] * (n // VEC) + ([n % VEC] if n % VEC else [])


def same_bits(a, b, what):
    assert a.shape == b.shape, "%s: %s samples, expected %s" % (what, a.shape, b.shape)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "%s: differs" % what


def test_graph_reset_drops_pending_superchunks(lib, chain):
    """37 vectors and a bit leave slots in flight and one partly filled; after the reset the graph hands back exactly
    what a fresh graph with the same slots does for the next stream."""
    g, fresh = chain(), chain()
    for h in (g, fresh):
        _lib.check(lib.lrb200_graph_set_superchunk(h, S), "set_superchunk")
    before = rnd_c(np.random.default_rng(41), 37 * VEC + 100)
    graph_calls(lib, g, before, vectors(len(before)))
    _lib.check(lib.lrb200_graph_reset(g), "reset")
    x = O.synth_fm_iq(1, 600000)
    got, want = graph_calls(lib, g, x, vectors(len(x)), flush=True), graph_calls(lib, fresh, x, vectors(len(x)), flush=True)
    assert len(want) == -(-len(x) // 25)
    same_bits(got, want, "after the reset")


def test_graph_direct_runs_refused_in_superchunk_mode(lib, chain):
    g = chain()
    halo, per = lib.lrb200_graph_halo(g), 25 * 4096
    assert 0 < halo < per
    dx, dy = lib.lrb200_malloc((halo + per) * 8), lib.lrb200_malloc((per // 25 + 16) * 4)
    no = ctypes.c_size_t()
    runs = {
        "execute_device": lambda: lib.lrb200_graph_execute_device(g, dx, per, dy, ctypes.byref(no)),
        "execute_shard": lambda: lib.lrb200_graph_execute_shard(g, None, dx, halo, per, per, dy, ctypes.byref(no), None),
    }
    try:
        _lib.check(lib.lrb200_memset(dx, 0, (halo + per) * 8), "memset")
        _lib.check(lib.lrb200_graph_set_superchunk(g, S), "set_superchunk")
        for name, run in runs.items():                   # with nothing fed, then with a partial slot
            assert run() != 0, name
            assert DIRECTLY in _lib.last_error(), (name, _lib.last_error())
            graph_calls(lib, g, rnd_c(np.random.default_rng(42), VEC), [VEC])
        graph_calls(lib, g, np.zeros(0, np.complex64), [], flush=True)
        _lib.check(lib.lrb200_graph_set_superchunk(g, 0), "set_superchunk(0)")
        for name, run in runs.items():
            _lib.check(run(), name)
            _lib.check(lib.lrb200_sync(), "sync")
            assert no.value > 0, name
    finally:
        lib.lrb200_free(dx)
        lib.lrb200_free(dy)


@pytest.mark.parametrize("fuse", [1, 0])
def test_graph_host_call_is_cut_every_2_23_samples(lib, chain, fuse):
    n = 2 * GRAPH_CHUNK + 12345
    x = rnd_c(np.random.default_rng(43), n)
    g = chain(fuse)
    one = graph_calls(lib, g, x, [n])
    _lib.check(lib.lrb200_graph_reset(g), "reset")
    cut = graph_calls(lib, g, x, [GRAPH_CHUNK, GRAPH_CHUNK, 12345])
    assert len(one) == -(-n // 25)
    same_bits(one, cut, "one call against calls of 2^23")


def block_calls(lib, make, xs, lengths, out_dtypes):
    """A fresh host-mode block from make() through lrb200_block_execute_multi in calls of `lengths`: every output port."""
    h = _lib.check_handle(make(), "block")
    outs, pos, no = [[] for _ in out_dtypes], 0, ctypes.c_size_t()
    try:
        for n in lengths:
            ys = [np.zeros(n, dt) for dt in out_dtypes]
            xa = (ctypes.c_void_p * len(xs))(*[x[pos:pos + n].ctypes.data for x in xs])
            ya = (ctypes.c_void_p * len(ys))(*[y.ctypes.data for y in ys])
            _lib.check(lib.lrb200_block_execute_multi(h, xa, len(xs), n, ya, len(ys), ctypes.byref(no)), "execute_multi")
            assert no.value == n
            for o, y in zip(outs, ys):
                o.append(y)
            pos += n
    finally:
        lib.lrb200_block_destroy(h)
    return [np.concatenate(o) for o in outs]


def pll_parallel(lib):
    h = lib.lrb200_pll_create(*PLL_ARGS, 0)
    if h:
        _lib.check(lib.lrb200_pll_set_mode(h, 1), "pll_set_mode")
    return h


def pilot(n, seed):
    t = np.arange(n) / PLL_ARGS[4]
    return (0.8 * np.exp(2j * np.pi * 19000.3 * t + 0.4j) + 0.05 * rnd_c(np.random.default_rng(seed), n)).astype(np.complex64)


@pytest.mark.parametrize("name", ["multiply_conjugate", "pll_parallel"])
def test_host_mode_block_call_is_cut_every_2_24_samples(lib, name):
    n = 2 * BLOCK_CHUNK + 777
    if name == "multiply_conjugate":
        rng = np.random.default_rng(44)
        make, xs, dts = lambda: lib.lrb200_binary_create(b"multiplyconjugate", 1, 0), [rnd_c(rng, n), rnd_c(rng, n)], [np.complex64]
    else:
        make, xs, dts = lambda: pll_parallel(lib), [pilot(n, 45)], [np.complex64, np.float32]
    one = block_calls(lib, make, xs, [n], dts)
    cut = block_calls(lib, make, xs, [BLOCK_CHUNK, BLOCK_CHUNK, 777], dts)
    for k, (a, b) in enumerate(zip(one, cut)):
        same_bits(a, b, "output %d: one call against calls of 2^24" % k)


def test_stereo_dag_host_call_is_not_cut(lib):
    """A DAG's host call of 3 * 2^23 samples is one upload and one run: lrb200_dag_execute_device of the same call."""
    n = 3 * GRAPH_CHUNK
    x = stereo_input(n, 46)
    make = lambda y: stereo_top(y, parallel_pll=True)       # noqa: E731
    top_h, dag_h = planned_dag(make, x)
    top_d, dag_d = planned_dag(make, x)
    sizes = [p.data_type.dtype.itemsize for p in dag_d.ext_out]
    dx = lib.lrb200_malloc(n * 8)
    dys = [lib.lrb200_malloc(lib.lrb200_dag_max_output(dag_d.dag, k, n) * s) for k, s in enumerate(sizes)]
    try:
        want = host_execute(lib, dag_h, x)
        _lib.check(lib.lrb200_memcpy_h2d(dx, x.ctypes.data, n * 8), "h2d")
        n_out = (ctypes.c_size_t * len(dys))()
        _lib.check(lib.lrb200_dag_execute_device(dag_d.dag, dx, n, (ctypes.c_void_p * len(dys))(*dys), n_out), "execute_device")
        for k, w in enumerate(want):
            got = np.zeros(n_out[k], w.dtype)
            _lib.check(lib.lrb200_memcpy_d2h(got.ctypes.data, dys[k], n_out[k] * sizes[k]), "d2h")
            _lib.check(lib.lrb200_sync(), "sync")
            assert len(w) == -(-n // 5)
            same_bits(got, w, "port %d" % k)
    finally:
        lib.lrb200_free(dx)
        for d in dys:
            lib.lrb200_free(d)
        release(top_h)
        release(top_d)
