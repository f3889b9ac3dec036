"""PLLBlock on the GPU in both forms (aux_blocks.cu), held per output to the phase bound of tests/pll_ref.py and, in the
chunk-parallel form, to ERR_TOL / out_tol of a sequential run of the same input once the loop is locked.

Call lengths around the switch-over (2 L - 1, 2 L, 2 L + 1), one and two CTAs of chunks (128 L, 128 L + 1), a ragged
257 L + 5, sequential and parallel calls mixed with the chunk buffer growing mid-stream, a reset mid-stream, one
DEVICE-mode call of 2^26 + 3 samples with the stereo loop (1328 chunks), and the parallel form on noise and zeros."""
import ctypes

import numpy as np
import pytest

from luaradio_b200 import _lib
from tests import pll_ref as R

pytestmark = pytest.mark.gpu


def _create(lib, lp, mode, flags=0):
    bw, fmin, fmax, m, rate = lp.args
    h = _lib.check_handle(lib.lrb200_pll_create(bw, fmin, fmax, m, rate, flags), "pll")
    _lib.check(lib.lrb200_pll_set_mode(h, mode), "pll_set_mode")
    return h


def _execute(lib, h, x):
    out, err = np.zeros(len(x), np.complex64), np.zeros(len(x), np.float32)
    xa = (ctypes.c_void_p * 1)(x.ctypes.data)
    ya = (ctypes.c_void_p * 2)(out.ctypes.data, err.ctypes.data)
    no = ctypes.c_size_t()
    _lib.check(lib.lrb200_block_execute_multi(h, xa, 1, len(x), ya, 2, ctypes.byref(no)), "execute")
    assert no.value == len(x)
    return out, err


def _stream(lib, lp, mode, x, lengths):
    h = _create(lib, lp, mode)
    try:
        parts, pos = [], 0
        for n in lengths:
            parts.append(_execute(lib, h, x[pos:pos + n]))
            pos += n
    finally:
        lib.lrb200_block_destroy(h)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def _bound_ratio(lp, out, err):
    """error / bound of out against the multiplied phase rebuilt from err (the GPU fuses freq + beta e)."""
    ratio = R.out_ratio(out, R.rebuild_phase(err, lp, fma=True), R.phase_bound(lp, len(out)))
    print("error / bound %.3g" % ratio)
    return ratio


def _check_parallel(lp, lengths, seq, par, skip):
    """err and out of the parallel run against the sequential one from sample `skip` on, at ERR_TOL and at out_tol
    of the stream's lead-ins."""
    tol = R.out_tol(R.lead_ins(lengths, lp))
    de = float(np.max(np.abs(par[1][skip:].astype(np.float64) - seq[1][skip:])))
    do = float(np.max(np.abs(par[0][skip:].astype(np.complex128) - seq[0][skip:])))
    print("parallel vs sequential: err %.3g (%.3g of ERR_TOL), out %.3g (%.3g of out_tol, %d lead-ins)" % (
        de, de / R.ERR_TOL, do, do / tol, R.lead_ins(lengths, lp)))
    assert de <= R.ERR_TOL and do <= tol, (de, do)


@pytest.mark.parametrize("name", ["stereo", "rds"])
def test_call_lengths(name):
    lib = _lib.require_device()
    lp = R.Loop(*R.LOOPS[name])
    L = lp.L
    first = lp.W + 8000                                    # sequential: the loop acquires in the exact form
    lengths = [first, 2 * L - 1, 2 * L, 2 * L + 1, 5, 128 * L, 3 * L, 128 * L + 1, 257 * L + 5, 2 * L + 7]
    x = R.pilot(lp, sum(lengths), "noisy", seed=11)
    seq = _stream(lib, lp, 0, x, lengths)
    assert _bound_ratio(lp, *seq) <= 1.0
    par = _stream(lib, lp, 1, x, lengths)
    assert np.array_equal(par[0][:first], seq[0][:first]) and np.array_equal(par[1][:first], seq[1][:first])
    _check_parallel(lp, lengths, seq, par, first)
    again = _stream(lib, lp, 1, x, lengths)
    assert np.array_equal(again[0], par[0]) and np.array_equal(again[1], par[1])          # bit-identical rerun


@pytest.mark.parametrize("kind", ["clean", "offset", "drift"])
def test_pilots(kind):
    lib = _lib.require_device()
    lp = R.Loop(*R.LOOPS["rds"])
    lengths = [lp.W + 8000, 40 * lp.L + 3, 2 * lp.L]
    x = R.pilot(lp, sum(lengths), kind, seed=12)
    seq = _stream(lib, lp, 0, x, lengths)
    assert _bound_ratio(lp, *seq) <= 1.0
    _check_parallel(lp, lengths, seq, _stream(lib, lp, 1, x, lengths), lengths[0])


@pytest.mark.parametrize("mode", [0, 1])
def test_reset_mid_stream(mode):
    """After a reset the block is a fresh one: bit-identical to a new handle on the rest of the stream."""
    lib = _lib.require_device()
    lp = R.Loop(*R.LOOPS["rds"])
    before, after = [lp.W + 100, 3 * lp.L + 1], [lp.W + 100, 2 * lp.L, 5 * lp.L + 9]
    x = R.pilot(lp, sum(before) + sum(after), "noisy", seed=13)
    h = _create(lib, lp, mode)
    try:
        pos = 0
        for n in before:
            _execute(lib, h, x[pos:pos + n])
            pos += n
        _lib.check(lib.lrb200_block_reset(h), "reset")
        got = []
        for n in after:
            got.append(_execute(lib, h, x[pos:pos + n]))
            pos += n
    finally:
        lib.lrb200_block_destroy(h)
    ref = _stream(lib, lp, mode, x[sum(before):], after)
    assert np.array_equal(np.concatenate([g[0] for g in got]), ref[0])
    assert np.array_equal(np.concatenate([g[1] for g in got]), ref[1])
    if mode == 0:
        assert _bound_ratio(lp, *ref) <= 1.0


def _device_call(lib, lp, mode, x):
    n = len(x)
    h = _create(lib, lp, mode, _lib.LRB200_DEVICE)
    bufs = [_lib.check_handle(lib.lrb200_malloc(n * s), "buffer") for s in (8, 8, 4)]
    try:
        _lib.check(lib.lrb200_memcpy_h2d(bufs[0], x.ctypes.data, n * 8), "h2d")
        xa = (ctypes.c_void_p * 1)(bufs[0])
        ya = (ctypes.c_void_p * 2)(bufs[1], bufs[2])
        no = ctypes.c_size_t()
        _lib.check(lib.lrb200_block_execute_multi(h, xa, 1, n, ya, 2, ctypes.byref(no)), "execute")
        assert no.value == n
        out, err = np.empty(n, np.complex64), np.empty(n, np.float32)
        _lib.check(lib.lrb200_memcpy_d2h(out.ctypes.data, bufs[1], n * 8), "d2h")
        _lib.check(lib.lrb200_memcpy_d2h(err.ctypes.data, bufs[2], n * 4), "d2h")
        _lib.check(lib.lrb200_sync(), "sync")
    finally:
        for b in bufs:
            lib.lrb200_free(b)
        lib.lrb200_block_destroy(h)
    return out, err


def test_device_call_of_2_26_samples():
    """One call of 2^26 + 3 samples, stereo loop (1328 chunks).  The sequential form is held to the phase bound
    (1.2e-7 at the end); the chunk-parallel form, which acquires in its exact chunk 0, to the sequential one (a rebuild
    from the parallel form's own errors would integrate their lead-in differences open-loop, see tests/pll_ref.py).  A
    running sum of the multiplied phase over the call (7e7 rad at the end), as the parallel form once kept, leaves
    2.8e-4 here on an H100 (out_tol is 5.1e-6)."""
    lib = _lib.require_device()
    lp = R.Loop(*R.LOOPS["stereo"])
    n = (1 << 26) + 3
    x = R.pilot(lp, n, "clean", seed=14)
    seq = _device_call(lib, lp, 0, x)
    assert _bound_ratio(lp, *seq) <= 1.0
    par = _device_call(lib, lp, 1, x)
    assert (n + lp.L - 1) // lp.L == 1328
    d = np.abs(par[0][-lp.L:].astype(np.complex128) - seq[0][-lp.L:])
    print("last chunk: parallel vs sequential out %.3g" % float(np.max(d)))
    _check_parallel(lp, [n], seq, par, 0)


@pytest.mark.parametrize("kind", ["noise", "zeros"])
def test_parallel_form_on_noise_and_zeros(kind):
    """No lock to keep: the parallel form is not asserted equal to the sequential one, only well formed."""
    lib = _lib.require_device()
    lp = R.Loop(*R.LOOPS["stereo"])
    lengths = [3 * lp.L + 1, 130 * lp.L]
    x = R.pilot(lp, sum(lengths), kind, seed=15)
    out, err = _stream(lib, lp, 1, x, lengths)
    assert np.all(np.isfinite(out)) and np.all(np.isfinite(err))
    assert float(np.max(np.abs(err))) <= np.float32(np.pi)
    assert float(np.max(np.abs(np.abs(out.astype(np.complex128)) - 1.0))) <= 2.0 ** -23
