"""PLLBlock on the GPU in both forms (pll.cu).  The sequential form is held per output to the phase bound of
tests/pll_ref.py.  The verified chunk-parallel form (lrb200_pll_set_mode(q, 1)) is held to the sequential one: at
ERR_TOL / out_tol once the loop is locked, and with the assertions of tests/test_pll_ref.py on locked pilots and on
zeros, noise and gaps (within ERR_TOL / out_tol from the first sample, err bit for bit before the first accepted chunk,
the re-run counts of lrb200_pll_chunk_counts equal to the model's).

Call lengths around the switch-over (2 L - 1, 2 L, 2 L + 1), one and two CTAs of chunks (128 L, 128 L + 1), a ragged
257 L + 5, sequential and parallel calls mixed with the chunk buffer growing mid-stream, ragged and mixed calls over a
zero gap and a noise burst, a reset mid-stream and the counts after it, DEVICE-mode calls of 2^26 + 3 samples with the
stereo loop (1328 chunks), with and without a zero stretch, the parallel form on noise and zeros, a guard-banded case
with a zero gap, and the WBFM-stereo and AM-synchronous DAGs with a parallel PLL on I/Q with 0.5 s of zeros."""
import ctypes

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from tests import pll_ref as R
from tests.test_gpu_bounds import CPX, FLT, PLL_ARGS, PLL_PARALLEL_LENGTHS, Case, _pll_parallel, check_case, cmp_abs
from tests.test_gpu_dag_boundary import RATE, am_input, am_top, run_top, stereo_input, stereo_top

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


def _counts(lib, h):
    c, r = ctypes.c_uint64(), ctypes.c_uint64()
    _lib.check(lib.lrb200_pll_chunk_counts(h, ctypes.byref(c), ctypes.byref(r)), "pll_chunk_counts")
    return c.value, r.value


def _stream(lib, lp, mode, x, lengths):
    """(out, err, (chunks, reruns)) of one handle over the calls."""
    h = _create(lib, lp, mode)
    try:
        parts, pos = [], 0
        for n in lengths:
            parts.append(_execute(lib, h, x[pos:pos + n]))
            pos += n
        cnt = _counts(lib, h)
    finally:
        lib.lrb200_block_destroy(h)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), cnt


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
    assert _bound_ratio(lp, seq[0], seq[1]) <= 1.0
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
    assert _bound_ratio(lp, seq[0], seq[1]) <= 1.0
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
        assert _bound_ratio(lp, ref[0], ref[1]) <= 1.0


def _device_call(lib, lp, mode, x):
    """(out, err, (chunks, reruns)) of one DEVICE-mode call on a fresh handle."""
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
        cnt = _counts(lib, h)
    finally:
        for b in bufs:
            lib.lrb200_free(b)
        lib.lrb200_block_destroy(h)
    return out, err, cnt


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
    assert _bound_ratio(lp, seq[0], seq[1]) <= 1.0
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
    out, err, _ = _stream(lib, lp, 1, x, lengths)
    assert np.all(np.isfinite(out)) and np.all(np.isfinite(err))
    assert float(np.max(np.abs(err))) <= np.float32(np.pi)
    assert float(np.max(np.abs(np.abs(out.astype(np.complex128)) - 1.0))) <= 2.0 ** -23


def check_gpu(lp, x, lengths, locked):
    lib = _lib.require_device()
    o0, e0, _ = _stream(lib, lp, 0, x, lengths)
    o1, e1, (chunks, reruns) = _stream(lib, lp, 1, x, lengths)
    model = R.run_verified(lp, x, lengths)
    m = model[2]
    print("GPU chunks %d reruns %d, model %d %d" % (chunks, reruns, m.chunks, m.reruns))
    assert (chunks, reruns) == (m.chunks, m.reruns)
    # the model's decisions place the first accepted chunk; the comparison is the GPU's own mode 0
    res, nums = R.check(lp, x, lengths, (o0, e0), (o1, e1, m, model[3]), locked)
    assert all(res.values()), (res, nums)
    return chunks, reruns


@pytest.mark.parametrize("kind", R.LOCKED + R.UNLOCKED)
@pytest.mark.parametrize("name", list(R.LOOPS))
def test_against_sequential(name, kind):
    lp = R.loop(name)
    x, lengths = R.make_input(lp, kind)
    chunks, reruns = check_gpu(lp, x, lengths, kind in R.LOCKED)
    if kind in R.LOCKED:
        assert reruns == 0
    if kind == "zeros":
        assert reruns == chunks > 0


def test_ragged_and_mixed_calls():
    """Sequential-length and parallel calls, ragged last chunks, over a pilot with a zero gap and a noise burst."""
    lp = R.loop("rds")
    L = lp.L
    lengths = [L + 5, 2 * L - 1, 2 * L, 7, 2 * L + 1, 5 * L + 3, L, 9 * L + 11, 3 * L - 2]
    x = R.pilot(lp, sum(lengths), "noisy", seed=31)
    a = sum(lengths[:5]) + L // 3
    x[a:a + 3 * L] = 0
    b = sum(lengths[:7]) + 2 * L
    x[b:b + 2 * L] = R.pilot(lp, 2 * L, "noise", seed=32)
    _, reruns = check_gpu(lp, x, lengths, False)
    assert reruns >= 3


def test_reset_clears_the_counts():
    lib = _lib.require_device()
    lp = R.loop("rds")
    x = R.pilot(lp, 6 * lp.L, "zeros")
    h = _create(lib, lp, 1)
    try:
        _execute(lib, h, x)
        assert _counts(lib, h) == (5, 5)
        _lib.check(lib.lrb200_block_reset(h), "reset")
        assert _counts(lib, h) == (0, 0)
        _execute(lib, h, x[:3 * lp.L])
        assert _counts(lib, h) == (2, 2)
    finally:
        lib.lrb200_block_destroy(h)


def test_device_call_of_2_26_samples_with_a_zero_stretch():
    """One DEVICE call of 2^26 + 3 samples, stereo loop (1328 chunks), with 3.5 L of zeros after chunk 600: the chunks
    in and just after the stretch are run again and the rest accepted; the call is within ERR_TOL and out_tol of the
    sequential one from the first sample."""
    lib = _lib.require_device()
    lp = R.loop("stereo")
    n = (1 << 26) + 3
    x = R.pilot(lp, n, "clean", seed=33)
    z = 600 * lp.L + 1234
    x[z:z + 7 * lp.L // 2] = 0
    seq = _device_call(lib, lp, 0, x)
    out, err, (chunks, reruns) = _device_call(lib, lp, 1, x)
    print("chunks %d reruns %d" % (chunks, reruns))
    assert chunks == 1327 and 3 <= reruns <= 6
    de = float(np.max(np.abs(err.astype(np.float64) - seq[1])))
    do = float(np.max(np.abs(out.astype(np.complex128) - seq[0])))
    tol = R.out_tol(chunks - reruns)
    print("err %.3g of ERR_TOL, out %.3g of out_tol" % (de / R.ERR_TOL, do / tol))
    assert de <= R.ERR_TOL and do <= tol


def _gap_input(rng, n):
    t = np.arange(n) / PLL_ARGS[4]
    x = (0.8 * np.exp(2j * np.pi * 19000.3 * t + 0.4j) + 0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n)) / np.sqrt(2))
    x[n // 3:n // 3 + 5 * R.Loop(*PLL_ARGS).L // 2] = 0
    return [x.astype(np.complex64)]


def test_guard_banded_case_with_a_zero_gap():
    """The pll_parallel case of tests/test_gpu_bounds.py (calls of 1, 2 L - 1, 2 L, 2 L + 1 and 3 L + 5 in poisoned,
    aligned and unaligned buffers) on a pilot with 2.5 L of zeros, held to its tolerance from the first sample; the old
    form (every lead-in accepted) misses that tolerance on this input by orders of magnitude."""
    from oracle import lr_oracle as O
    lp = R.Loop(*PLL_ARGS)
    tol = 2e-5 + max(R.ERR_TOL, R.out_tol(R.lead_ins(PLL_PARALLEL_LENGTHS * 8, lp)))
    check_case(Case("lrb200_pll_create", _pll_parallel, [CPX], [CPX, FLT], PLL_PARALLEL_LENGTHS, _gap_input,
                    lambda xs: list(O.PLL(*PLL_ARGS).process(xs[0])), cmp_abs(tol), exact=True))
    x = _gap_input(np.random.default_rng(5), sum(PLL_PARALLEL_LENGTHS))[0]
    ref = R.Model(lp, 0).process(x)
    old = R.run_verified(lp, x, PLL_PARALLEL_LENGTHS, "accept_all")
    do = float(np.max(np.abs(old[0].astype(np.complex128) - ref[0])))
    print("accept-all model: out %.3g, tolerance %.3g" % (do, tol))
    assert do > 100 * tol


def _dag_pair(make_par, make_ser, x, S, lead_ins):
    _, serial = run_top(make_ser, x, S)
    top, par = run_top(make_par, x, S)
    assert "pll" in top.describe_gpu_graph()
    tol = 10 * R.out_tol(lead_ins)
    for k, (g, r) in enumerate(zip(par, serial)):
        assert len(g) == len(r) > 0
        d = float(np.max(np.abs(g.astype(np.float64) - r)))
        print("port %d: parallel vs serial PLL %.3g (%.3g of 10 out_tol)" % (k, d, d / tol))
        assert d <= tol, (k, d, tol)


def test_stereo_dag_with_a_zero_stretch():
    """WBFM stereo in super-chunks of 2^20 with PLLBlock.parallel = True against the serial PLL, on 2^22 samples of
    I/Q with 0.5 s of zeros from sample 1.5e6: equal from the first sample within 10 out_tol, the after-lock tolerance
    of test_gpu_dag_boundary.py."""
    x = stereo_input(1 << 22, 41)
    a = 1500000
    x[a:a + int(0.5 * RATE)] = 0
    _dag_pair(lambda y: stereo_top(y, parallel_pll=True), stereo_top, x, 1 << 20, -(-((1 << 22) // 5) // 50536))


def test_am_synchronous_dag_starting_with_zeros():
    """AM synchronous at 48 kS/s, super-chunks of 2^20, parallel PLL against the serial one on 2^22 samples whose
    first 0.5 s is zeros, and with another 0.5 s of zeros later on."""
    x = am_input(1 << 22, 42)
    x[:24000] = 0
    x[2000000:2024000] = 0

    def make(parallel):
        def mk(y):
            top, sinks = am_top(y)
            for blk in _pll_blocks(top):
                blk.parallel = parallel
            return top, sinks
        return mk
    _dag_pair(make(True), make(False), x, 1 << 20, -(-(1 << 22) // 16384))


def _pll_blocks(top):
    found, todo = [], [top]
    while todo:
        b = todo.pop()
        if isinstance(b, radio.PLLBlock):
            found.append(b)
        todo += list(getattr(b, "_blocks", []))
    assert found
    return found
