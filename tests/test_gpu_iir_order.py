"""IIRFilterBlock with 11..64 taps on either side on the GPU (iir_order.cu), every output held to the per-output bound of
tests/iir_order_ref.py against the float64 recurrence."""
import ctypes

import numpy as np
import pytest

from luaradio_b200 import _lib
from tests import iir_order_ref as R
from tests import test_gpu_bounds as GB

pytestmark = pytest.mark.gpu

FILTERS = R.filters()


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


def _check(b, a, xs, ys, cplx):
    _, ref, bnd = R.bound(b, a, xs, cplx)
    e = R.excess(np.concatenate(ys), ref, bnd)
    assert e <= 1.0, "error %.3g of the bound" % e


CALLS = (0, 1, 2, 8192, 8192, 2047, 2048, 2049, 37, 3 * 2048 + 5, 8192, 100000)


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", list(FILTERS))
def test_stream(name, cplx):
    lib = _lib.require_device()
    b, a = FILTERS[name]
    h = _lib.check_handle(_create(lib, b, a, cplx), "iir")
    try:
        assert lib.lrb200_block_name(h).decode() == "iir_%s(scan,%d)" % ("crcf" if cplx else "rrrf", len(a) - 1)
        rng = np.random.default_rng(len(b) * 100 + len(a))
        xs = [_input(rng, n, cplx) for n in CALLS]
        ys = [_execute(lib, h, x, cplx) for x in xs]
        _check(b, a, xs, ys, cplx)
        # a reset in the middle of the stream: the rest is a fresh stream
        _lib.check(lib.lrb200_block_reset(h), "reset")
        xs2 = [_input(rng, n, cplx) for n in (5000, 1, 8192)]
        _check(b, a, xs2, [_execute(lib, h, x, cplx) for x in xs2], cplx)
    finally:
        lib.lrb200_block_destroy(h)


@pytest.mark.parametrize("name", ["resonator", "comb33"])
def test_long_call(name):
    """one 2^26-sample call across 32768 tiles (DEVICE mode)"""
    import torch
    lib = _lib.require_device()
    b, a = FILTERS[name]
    n = 1 << 26
    x = _input(np.random.default_rng(5), n, False)
    h = _lib.check_handle(_create(lib, b, a, False, _lib.LRB200_DEVICE), "iir")
    try:
        dx = torch.from_numpy(x).cuda()
        dy = torch.empty_like(dx)
        torch.cuda.synchronize()
        no = ctypes.c_size_t()
        _lib.check(lib.lrb200_block_execute(h, dx.data_ptr(), n, dy.data_ptr(), ctypes.byref(no)), "execute")
        _lib.check(lib.lrb200_sync(), "sync")
        _check(b, a, [x], [dy.cpu().numpy()], False)
    finally:
        lib.lrb200_block_destroy(h)


@pytest.mark.parametrize("cplx", [False, True])
def test_offset_input_bitwise(cplx):
    """the same multi-tile stream with the input one element further into the buffer gives bit-identical outputs (the
    look-back walk is fixed, so no sum depends on timing)"""
    lib = _lib.require_device()
    b, a = FILTERS["cheby18_bandpass"]
    rng = np.random.default_rng(3)
    xs = [_input(rng, n, cplx) for n in (8192, 1, 20000, 2048, 100003)]
    outs = []
    for off in (0, 1):
        h = _lib.check_handle(_create(lib, b, a, cplx), "iir")
        try:
            ys = []
            for x in xs:
                buf = np.zeros(len(x) + 1, x.dtype)
                buf[off:off + len(x)] = x
                ys.append(_execute(lib, h, buf[off:off + len(x)], cplx))
            outs.append(np.concatenate(ys))
        finally:
            lib.lrb200_block_destroy(h)
    assert np.array_equal(outs[0].view(np.uint8), outs[1].view(np.uint8))


def test_refuses_65_taps():
    lib = _lib.require_device()
    for nb, na in ((65, 3), (3, 65)):
        b = np.full(nb, 0.1, np.float32)
        a = np.zeros(na, np.float32)
        a[0] = 1.0
        assert not _create(lib, b, a, False)
        assert lib.lrb200_last_error().decode() == "iir: at most 64 feed-forward and 64 feedback taps"
    assert not _create(lib, np.ones(12, np.float32), np.zeros(12, np.float32), False)


def test_short_filters_keep_their_kernels():
    lib = _lib.require_device()
    for (b, a), name in ((([0.2, 0.3], [1.0, -0.5]), "iir_rrrf"), (([0.2] * 10, [1.0, -0.5, 0.2] + [0.0] * 7), "iir_rrrf(general)")):
        h = _lib.check_handle(_create(lib, np.float32(b), np.float32(a), False), "iir")
        assert lib.lrb200_block_name(h).decode() == name
        lib.lrb200_block_destroy(h)


def _graph_blocks(b, a):
    import luaradio_b200 as radio
    from luaradio_b200.types import Float32
    from tests.test_gpu_graph_rewrites import mk, _down
    return [mk(radio.IIRFilterBlock, (b, a), Float32), _down(4, Float32)]


@pytest.mark.parametrize("fuse", [1, 0])
def test_graph_description(fuse):
    from tests.test_gpu_graph_rewrites import observe, CASES
    b, a = FILTERS["butter5_bandpass"]
    CASES["iir-order+down"] = (lambda: _graph_blocks(b, a), True)
    try:
        assert observe("iir-order+down", fuse) == ("iir_rrrf(scan,10) | downsample", 2, 2)
    finally:
        del CASES["iir-order+down"]


def test_graph_halo():
    lib = _lib.require_device()
    b, a = FILTERS["butter5_bandstop"]
    h = _lib.check_handle(_create(lib, b, a, False, _lib.LRB200_DEVICE), "iir")
    g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
    try:
        _lib.check(lib.lrb200_graph_append(g, h), "append")
        _lib.check(lib.lrb200_graph_commit(g, 1), "commit")
        halo = lib.lrb200_graph_halo(g)
        assert halo > 0
        # a shard started `halo` samples early from a zero state matches the streamed GPU output: what the halo
        # leaves out has decayed below 1e-10 of the impulse response's peak
        n, start = 200000, 120000
        x = _input(np.random.default_rng(9), n, False)
        s = _lib.check_handle(_create(lib, b, a, False), "iir")
        t = _lib.check_handle(_create(lib, b, a, False), "iir")
        try:
            stream = _execute(lib, t, x, False)
            part = _execute(lib, s, x[start - halo:], False)[halo:]
        finally:
            lib.lrb200_block_destroy(s)
            lib.lrb200_block_destroy(t)
        tol = 1e-6 * float(np.max(np.abs(stream)))
        assert np.max(np.abs(part - stream[start:])) <= tol
    finally:
        lib.lrb200_graph_destroy(g)
    comb_b, comb_a = FILTERS["comb33"]
    h2 = _lib.check_handle(_create(lib, comb_b, comb_a, False, _lib.LRB200_DEVICE), "iir")
    g2 = _lib.check_handle(lib.lrb200_graph_create(), "graph")
    try:
        _lib.check(lib.lrb200_graph_append(g2, h2), "append")
        _lib.check(lib.lrb200_graph_commit(g2, 1), "commit")
        assert lib.lrb200_graph_halo(g2) < 0
    finally:
        lib.lrb200_graph_destroy(g2)


def _bounds_case(name, cplx):
    b, a = FILTERS[name]
    bounds = {}

    def ref(xs):
        _, r, bnd = R.bound(b, a, [xs[0]], cplx)
        bounds[len(r)] = bnd
        return [r]

    def cmp(got, r, what):
        assert R.excess(got, np.asarray(r, np.complex128), bounds[len(r)]) <= 1.0, what
    port = GB.CPX if cplx else GB.FLT
    return GB.Case("lrb200_iir_create_" + ("crcf" if cplx else "rrrf"),
                   lambda lib: _create(lib, b, a, cplx, _lib.LRB200_DEVICE), [port], [port],
                   GB.base_lengths(R.T, 8192), lambda rng, n: [(GB.rnd_c if cplx else GB.rnd_f)(rng, n)],
                   ref, cmp, exact=True)


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("name", ["cheby18_bandstop", "allpole40", "resonator"])
def test_device_bounds(name, cplx):
    GB.check_case(_bounds_case(name, cplx))
