"""IIRFilterBlock with at most 10 taps on each side on the GPU (iir.cu: the single-pole scan and the general-order
kernel), every output held to the per-output bound of tests/iir_small_ref.py against the float64 recurrence."""
import ctypes

import numpy as np
import pytest

from luaradio_b200 import _lib
from tests import iir_order_ref as R
from tests import iir_small_ref as S

pytestmark = pytest.mark.gpu

SCAN = S.scan_filters()
GENERAL = S.general_filters()
# 0, 1, 2; T - 1, T, T + 1, 2T +- 1 for the tile T = 4096 and the LOCAL payload 3584
CALLS = (0, 1, 2, 4095, 4096, 4097, 8191, 8193, 3583, 3584, 3585, 7167, 7169, 37, 100000)


def _create(lib, b, a, cplx, flags=0):
    fn = lib.lrb200_iir_create_crcf if cplx else lib.lrb200_iir_create_rrrf
    return fn(b.ctypes.data, len(b), a.ctypes.data, len(a), flags)


def _execute(lib, h, x, cplx):
    y = np.zeros(len(x), np.complex64 if cplx else np.float32)
    no = ctypes.c_size_t()
    _lib.check(lib.lrb200_block_execute(h, x.ctypes.data, len(x), y.ctypes.data, ctypes.byref(no)), "execute")
    assert no.value == len(x)
    return y


def _input(rng, n, cplx):
    v = rng.uniform(-1, 1, n)
    if cplx:
        v = v + 1j * rng.uniform(-1, 1, n)
    return v.astype(np.complex64 if cplx else np.float32)


def _stream_through(name, b, a, cplx, calls, check, kind, after_reset=(5000, 1, 8193)):
    lib = _lib.require_device()
    h = _lib.check_handle(_create(lib, b, a, cplx), "iir")
    try:
        assert lib.lrb200_block_name(h).decode() == "iir_%s%s" % ("crcf" if cplx else "rrrf", kind), name
        rng = np.random.default_rng(sum(map(ord, name)))
        xs = [_input(rng, n, cplx) for n in calls]
        check(xs, [_execute(lib, h, x, cplx) for x in xs])
        # a reset in the middle of the stream: the rest is a fresh stream
        _lib.check(lib.lrb200_block_reset(h), "reset")
        xs2 = [_input(rng, n, cplx) for n in after_reset]
        check(xs2, [_execute(lib, h, x, cplx) for x in xs2])
    finally:
        lib.lrb200_block_destroy(h)


def _scan_check(b, a, cplx, D=1):
    def check(xs, ys):
        _, ref, bnd, _ = S.scan_bound(b, a, xs, cplx, D)
        e = S.excess(np.concatenate(ys), ref, bnd)
        print("error / bound %.3g" % e)
        assert e <= 1.0, "error %.3g of the bound" % e
    return check


def _general_check(b, a, cplx):
    def check(xs, ys):
        ref, bnd, _ = S.general_bound(b, a, xs, cplx)
        e = S.excess(np.concatenate(ys), ref, bnd)
        print("error / bound %.3g" % e)
        assert e <= 1.0, "error %.3g of the bound" % e
    return check


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", list(SCAN))
def test_scan_stream(name, cplx):
    b, a = SCAN[name]
    _stream_through(name, b, a, cplx, CALLS, _scan_check(b, a, cplx), "")


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", list(GENERAL))
def test_general_stream(name, cplx):
    b, a = GENERAL[name]
    calls, after_reset = CALLS, (5000, 1, 8193)
    if name == "resonator_w64k":
        calls = CALLS + (300000,)          # chunks of 4W: one call of two chunks, the second warmed up 63961 samples
    if name == "resonator_nodecay":
        # one thread runs each call; the bound grows with the stream, so the stream stays short enough that it is
        # below 1e-2 of the output (tests/test_iir_small_ref.py::test_general_bound_is_tight)
        calls, after_reset = (0, 1, 2, 37, 600, 1200), (1000, 1, 700)
    _stream_through(name, b, a, cplx, calls, _general_check(b, a, cplx), "(general)", after_reset)


@pytest.mark.parametrize("name", list(S.inexact_filters()))
def test_inexact_normalisation_runs_in_double(name):
    """a0 = 3 or 0.7: where fl32(b / a0), fl32(a / a0) would be a different filter the block is IirOrderBlock, held to
    its own bound (tests/iir_order_ref.py); where every quotient happens to be exact it keeps its small kernel"""
    b, a = S.inexact_filters()[name]
    a0 = np.float64(a[0])
    exact = all(S._f32(v / a0) == v / a0 for v in np.concatenate([b, a]).astype(np.float64))
    lib = _lib.require_device()
    h = _lib.check_handle(_create(lib, b, a, False), "iir")
    try:
        rng = np.random.default_rng(7)
        xs = [_input(rng, n, False) for n in (4097, 1, 30000)]
        ys = np.concatenate([_execute(lib, h, x, False) for x in xs])
        if exact:
            assert lib.lrb200_block_name(h).decode() == ("iir_rrrf" if len(a) <= 2 else "iir_rrrf(general)")
            bnd = S.scan_bound(b, a, xs, False)[1:3] if len(a) <= 2 else S.general_bound(b, a, xs, False)[:2]
            assert S.excess(ys, *bnd) <= 1.0
        else:
            assert lib.lrb200_block_name(h).decode() == "iir_rrrf(scan,%d)" % (len(a) - 1)
            _, ref, bnd = R.bound(b, a, xs, False)
            assert R.excess(ys, ref, bnd) <= 1.0
    finally:
        lib.lrb200_block_destroy(h)


def _gated(x, burst):
    return (x * (((np.arange(len(x)) // burst) % 2) == 0)).astype(x.dtype)


@pytest.mark.parametrize("name", list(SCAN))
def test_scan_gated(name):
    """noise switched on and off every 1000 samples: where a LOCAL restart or a look-back cut-off falls into the
    silence, what it leaves out is the whole output, so a warm-up or cut-off that is too short shows"""
    b, a = SCAN[name]
    lib = _lib.require_device()
    h = _lib.check_handle(_create(lib, b, a, False), "iir")
    try:
        x = _gated(_input(np.random.default_rng(11), 60000, False), 1000)
        xs = [x[:4097], x[4097:4097 + 3585], x[4097 + 3585:]]
        _scan_check(b, a, False)(xs, [_execute(lib, h, v, False) for v in xs])
    finally:
        lib.lrb200_block_destroy(h)


@pytest.mark.parametrize("name", [k for k, (b, a) in GENERAL.items() if 0 <= S.GeneralModel(b, a, False).W < 4096])
def test_general_gated(name):
    """one call of 12 chunks whose input falls silent 3W/4 before every other chunk's start: a warm-up shorter than
    that misses the decaying tail of the recurrence"""
    b, a = GENERAL[name]
    m = S.GeneralModel(b, a, False)
    chunk = m.plan(1 << 30)[0]
    x = _input(np.random.default_rng(12), 12 * chunk, False)
    for s0 in range(chunk, len(x), 2 * chunk):
        x[s0 - 3 * m.W // 4:s0 + chunk // 2] = 0
    lib = _lib.require_device()
    h = _lib.check_handle(_create(lib, b, a, False), "iir")
    try:
        _general_check(b, a, False)([x], [_execute(lib, h, x, False)])
    finally:
        lib.lrb200_block_destroy(h)


def _graph(lib, b, a, D, cplx):
    import luaradio_b200 as radio
    from luaradio_b200.types import ComplexFloat32, Float32
    from tests.test_gpu_stream import mk
    t = ComplexFloat32 if cplx else Float32
    blocks = [mk(radio.IIRFilterBlock, [Float32.vector_from_array(b), Float32.vector_from_array(a)], t),
              mk(radio.DownsamplerBlock, (D,), t)]
    g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
    for blk in blocks:
        _lib.check(lib.lrb200_graph_append(g, blk.make_device_handle()), "append")
    _lib.check(lib.lrb200_graph_commit(g, 1), "commit")
    return g


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", ["deemph", "pslow_nb2", "p0.948_nb5"])
@pytest.mark.parametrize("D", [2, 3, 7])
def test_fused_decimation(D, name, cplx):
    """IIRFilterBlock -> DownsamplerBlock(D) as one scan with a strided store, a LOCAL pole and two look-back poles,
    ragged source chunks"""
    lib = _lib.require_device()
    b, a = SCAN[name]
    g = _graph(lib, b, a, D, cplx)
    try:
        assert lib.lrb200_graph_describe(g).decode() == "iir_%s[fused x2]" % ("crcf" if cplx else "rrrf")
        rng = np.random.default_rng(D)
        xs = [_input(rng, n, cplx) for n in CALLS + (5, 4099)]
        ys = []
        for x in xs:
            y = np.zeros(lib.lrb200_graph_max_output(g, len(x)), x.dtype)
            no = ctypes.c_size_t()
            _lib.check(lib.lrb200_graph_execute(g, x.ctypes.data, len(x), y.ctypes.data, ctypes.byref(no)), "execute")
            ys.append(y[:no.value])
        _scan_check(b, a, cplx, D)(xs, ys)
    finally:
        lib.lrb200_graph_destroy(g)


def test_long_call():
    """one DEVICE-mode call of 2^27 + 4099 real samples through a committed IIR -> Downsampler(3) graph: the fused
    block splits it into launches of 2^27 and 4099 samples, the second starting at decimation phase 1 from the first's
    carried output and input history.  Held to scan_closed_excess (no model run at this size)."""
    import torch
    lib = _lib.require_device()
    b, a = SCAN["p-0.948_nb2"]
    n = (1 << 27) + 4099
    x = _input(np.random.default_rng(5), n, False)
    g = _graph(lib, b, a, 3, False)
    try:
        assert lib.lrb200_graph_describe(g).decode() == "iir_rrrf[fused x2]"
        dx = torch.from_numpy(x).cuda()
        dy = torch.empty(lib.lrb200_graph_max_output(g, n), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        no = ctypes.c_size_t()
        _lib.check(lib.lrb200_graph_execute_device(g, dx.data_ptr(), n, dy.data_ptr(), ctypes.byref(no)), "execute")
        _lib.check(lib.lrb200_sync(), "sync")
        assert no.value == -(-n // 3)
        got = dy[:no.value].cpu().numpy()
        del dx, dy
        e = S.scan_closed_excess(b, a, x, got, 3)
        print("error / bound %.3g" % e)
        assert e <= 1.0, "error %.3g of the bound" % e
    finally:
        lib.lrb200_graph_destroy(g)
