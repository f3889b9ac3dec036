"""The geometry model, bounds and mutants of tests/fft_fir_ref.py, checked without a GPU:

  * the geometry model agrees with hand-worked examples of fir_fft.cu's block split and launch counts;
  * the bound cannot fail a correct kernel: a float32 emulation of the kernels' arithmetic (the generated 32-point
    radix-2 networks with their FMA butterflies, the 32 x 32 four-step with float32 twiddles, H / N in float32, the
    delay line's FMA accumulation and read-modify-write launches, the translator's E and P_b) stays below a quarter
    of it in every mode, and so does the C oracle's own float32 four-step overlap-save at M = 128;
  * the inputs separate right from wrong: every mutant exceeds 4x the bound at some output of every case of
    tests/test_gpu_fft_fir.py, on that case's own input."""
import math

import numpy as np
import pytest

from oracle import cbuild
from tests import fft_fir_ref as F
from tests import test_gpu_fft_fir as T

F32 = np.float32


# ---- the geometry model ---------------------------------------------------------------------------------------------
def test_geometry_hand_worked():
    # M = 513 under AUTO: L = 512; below 8L the catch-all (history + 1), from 8L on the overlap-save kernel with
    # blocks [0, 8): block 0 reads the history (edge), 1..7 are interior
    m = F.FirModel("crcf", 513)
    assert m.L == 512
    assert m.plan(8 * 512 - 1, 0) == ("direct", 2, [])
    assert m.plan(8 * 512, 0) == ("fft", 3, [(1, 8, 8)])
    # packed real, M = 33: L = 992, one transform covers 1984 outputs; 3 transforms, the last one partial (odd count of
    # L-blocks: 5947 = 5 L + 987): edge work is transforms 0 and 2, transform 1 is interior
    m = F.FirModel("rrrf", 33, algo="fft")
    assert (m.L, m.per) == (992, 1984)
    assert m.plan(5947, 0) == ("fft", 3, [(1, 2, 3)])
    # one short call: nothing interior
    assert m.plan(100, 0) == ("fft", 2, [(1, 1, 1)])
    # delay line with nb < pc + p0: all edge work
    m = F.FirModel("cccf", 2048, algo="fft")
    assert m.nparts == 4
    assert m.plan(1000, 0) == ("fdl", 2, [(2, 2, 2)])
    # 9 partitions in groups of 4, 4, 1: n = 3000 is 6 blocks; the first group has one interior block, the later ones
    # none
    m = F.FirModel("crcf", 4097, algo="fft")
    assert m.plan(3000, 0) == ("fdl", 5, [(4, 5, 6), (6, 6, 6), (6, 6, 6)])
    # a single tap: no history update
    assert F.FirModel("crcf", 1, algo="fft").plan(5000, 0) == ("fft", 2, [(1, 4, 5)])
    # the catch-all launches nothing when the call keeps no output
    assert F.FirModel("crcf", 9000, D=1).plan(10, 0) == ("direct", 2, [])
    assert F.FirModel("crcf", 2000, D=5).plan(3, 1) == ("direct", 1, [])
    # the generic polyphase kernel takes the direct decimators it covers
    assert F.FirModel("crcf", 514, D=2).plan(100000, 0)[0] == "poly_generic"


# ---- float32 emulation of the kernels -------------------------------------------------------------------------------
def _fma(a, b, c):
    return (a.astype(np.float64) * np.float64(b) + c.astype(np.float64)).astype(F32) if np.ndim(b) == 0 else \
        (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def _bitrev5(i):
    return int("{:05b}".format(i)[::-1], 2)


def _stages():
    """tools/gen_fft32.py's network: (logical i0, i1, twiddle index m) per stage"""
    out, span = [], 1
    while span < 32:
        out.append([(g + j, g + j + span, j * (16 // span)) for g in range(0, 32, 2 * span) for j in range(span)])
        span *= 2
    return out


STAGES = _stages()


def _net(re, im, inv, br_in):
    """fft32_nat2br (br_in False: register = bitrev(logical)) / fft32_br2nat (register = logical), last axis."""
    re, im = re.copy(), im.copy()
    reg = (lambda i: _bitrev5(i)) if not br_in else (lambda i: i)
    for stage in STAGES:
        for i0, i1, m in stage:
            r0, r1 = reg(i0), reg(i1)
            ar, ai, br, bi = re[..., r0], im[..., r0], re[..., r1], im[..., r1]
            if m == 0:
                na, nb = (ar + br, ai + bi), (ar - br, ai - bi)
            elif m == 8:
                wx, wy = (-bi, br) if inv else (bi, -br)
                na, nb = (ar + wx, ai + wy), (ar - wx, ai - wy)
            else:
                wr = F32("%.9e" % math.cos(2 * math.pi * m / 32))
                wi = F32("%.9e" % -math.sin(2 * math.pi * m / 32))
                if inv:
                    wi = -wi
                tx, ty = _fma(br, wr, ar), _fma(bi, wr, ai)
                yx, yy = _fma(-bi, wi, tx), _fma(br, wi, ty)
                na, nb = (yx, yy), (_fma(ar, F32(2), -yx), _fma(ai, F32(2), -yy))
            re[..., r0], im[..., r0] = na
            re[..., r1], im[..., r1] = nb
    return re, im


def _cmul(ar, ai, wr, wi, conj=False):
    """fir_fft.cu cmul_conj_if"""
    wi = -wi if conj else wi
    tx, ty = (-ai) * wi, ar * wi
    return _fma(ar, wr, tx), _fma(ai, wr, ty)


def _tables():
    a = np.arange(32)
    e = (a[:, None] * a[None, :]) % 1024
    tw = np.exp(-2j * np.pi * e / 1024)
    return tw.real.astype(F32), tw.imag.astype(F32)          # [a][c]


TWR, TWI = _tables()


def _forward(re, im):
    """blocks (nb, 1024) float32 re / im -> X[k1 + 32 k2] as (nb, lane k1, register bitrev(k2))"""
    nb = re.shape[0]
    vr = re.reshape(nb, 32, 32).transpose(0, 2, 1)            # [b][lane n2][register n1]
    vi = im.reshape(nb, 32, 32).transpose(0, 2, 1)
    vr, vi = _net(vr, vi, False, False)
    perm = [_bitrev5(k) for k in range(32)]
    tr, ti = vr[..., perm], vi[..., perm]                       # [b][n2][k1]
    wr, wi = TWR.T[None], TWI.T[None]                           # s_tw[k1 * 32 + lane]: [lane n2][k1]
    xr, xi = _cmul(tr, ti, wr, wi)
    xr[..., 0], xi[..., 0] = tr[..., 0], ti[..., 0]
    vr, vi = xr.transpose(0, 2, 1).copy(), xi.transpose(0, 2, 1).copy()    # [b][lane k1][register n2]
    return _net(vr, vi, False, False)


def _inverse(vr, vi):
    """Y as (nb, lane k1, register bitrev(k2)) -> y (nb, 1024) natural"""
    nb = vr.shape[0]
    vr, vi = _net(vr, vi, True, True)                           # [b][k1][n2]
    wr, wi = TWR.T[None], TWI.T[None]                           # s_tw[n2 * 32 + lane]: [lane k1][n2]
    tr, ti = _cmul(vr, vi, wr, wi, conj=True)
    tr[..., 0], ti[..., 0] = vr[..., 0], vi[..., 0]
    vr, vi = tr.transpose(0, 2, 1).copy(), ti.transpose(0, 2, 1).copy()    # [b][lane n2][register k1]
    vr, vi = _net(vr, vi, True, False)                          # y[n2 + 32 n1] at register bitrev(n1)
    perm = [_bitrev5(k) for k in range(32)]
    yr, yi = vr[..., perm].transpose(0, 2, 1), vi[..., perm].transpose(0, 2, 1)   # [b][n1][n2]
    return yr.reshape(nb, 1024), yi.reshape(nb, 1024)


def _spectrum(h):
    """float32 H / N in the kernel's [k2][k1] -> (lane k1, register bitrev(k2)) placement"""
    Hn = np.fft.fft(np.asarray(h).astype(np.complex128), F.FF_N) / F.FF_N
    perm = np.array([_bitrev5(k) for k in range(32)])
    Hk = Hn.reshape(32, 32)                                     # [k2][k1]
    Hp = np.empty((32, 32), np.complex128)
    Hp[:, perm] = Hk.T                                          # [k1][bitrev(k2)] = H[k1 + 32 k2]
    return Hp.real.astype(F32), Hp.imag.astype(F32)


def _gather(x, idx, lo, hi):
    """x[idx] where lo <= idx < hi, else 0"""
    ok = (idx >= lo) & (idx < hi)
    return np.where(ok, x[np.clip(idx, 0, len(x) - 1)], 0)


def _phasor(fix):
    """common.cuh phasor_from_fix: the top 32 bits as a signed fraction of a half turn, sincospif"""
    t = fix >> 32
    t = t - (1 << 32) if t >= 1 << 31 else t
    ht = F32(t) * F32(4.656612873077393e-10)
    return F32(math.cos(math.pi * float(ht))), F32(math.sin(math.pi * float(ht)))


def _emulate_call(case, x, n0, s, n, first):
    """One call's full-rate outputs [s, s + n) as the overlap-save kernel computes them in float32 (complex64)."""
    m, M = case.model, case.M
    out = np.zeros(n, np.complex64)
    if m.nparts > 1:
        P = m.nparts
        nb = -(-n // F.HOP)
        he = np.asarray(case.h).astype(np.complex128)
        t = np.arange(F.FF_N)
        acc = None
        for p0 in range(0, P, F.MAXPC):
            pc = min(F.MAXPC, P - p0)
            bs = np.arange(-(pc - 1), nb)
            i = (bs[:, None] - 1) * F.HOP - p0 * F.HOP + t[None]            # call-relative inputs
            v = _gather(x, s + i, 0, len(x)) * ((i >= -(M - 1)) & (i < n))
            Xr, Xi = _forward(v.real.astype(F32), v.imag.astype(F32))
            Hs = [_spectrum(he[(p0 + pp) * F.HOP:(p0 + pp + 1) * F.HOP]) for pp in range(pc)]
            k = pc - 1                                                       # X of block b at k + b
            yr, yi = _cmul(Xr[k:], Xi[k:], Hs[0][0][None], Hs[0][1][None])
            for pp in range(1, pc):
                ar, ai = Xr[k - pp:k - pp + nb], Xi[k - pp:k - pp + nb]
                yr, yi = _fma(ar, Hs[pp][0][None], yr), _fma(ai, Hs[pp][0][None], yi)
                yr, yi = _fma(-ai, Hs[pp][1][None], yr), _fma(ar, Hs[pp][1][None], yi)
            tr, ti = _inverse(yr, yi)
            yb = (tr[:, 512:] + 1j * ti[:, 512:]).astype(np.complex64).reshape(-1)[:n]
            acc = yb if acc is None else (acc.real + yb.real) + 1j * (acc.imag + yb.imag).astype(np.complex64)
        return acc
    L, per = m.L, m.per
    nblocks = -(-n // per)
    b = np.arange(nblocks)
    t = np.arange(F.FF_N)
    Hr, Hi = _spectrum(F.effective_taps(case.kind, case.h))
    if case.kind == "rrrf":
        i0 = (2 * b[:, None]) * L - (M - 1) + t[None]
        xr = _gather(x, s + i0, 0, s + n).astype(F32)
        xi = _gather(x, s + i0 + L, 0, s + n).astype(F32)
    else:
        i0 = b[:, None] * L - (M - 1) + t[None]
        v = _gather(x, s + i0, 0, s + n)
        xr, xi = v.real.astype(F32), np.asarray(v.imag).astype(F32)
        if case.turns is not None:
            fix = int(math.floor((case.turns % 1.0) * 2 ** 64)) % (1 << 64)
            E = np.array([np.exp(2j * np.pi * float((fix * j % (1 << 64)) / 2 ** 64)) for j in range(F.FF_N)])
            xr, xi = _cmul(xr, xi, E.real.astype(F32)[None], E.imag.astype(F32)[None])
    Xr, Xi = _forward(xr, xi)
    Yr, Yi = _cmul(Xr, Xi, Hr[None], Hi[None])
    yr, yi = _inverse(Yr, Yi)
    nn = t[M - 1:]
    if case.kind == "rrrf":
        o0 = (2 * b[:, None]) * L - (M - 1) + nn[None]
        for o, vals in ((o0, yr[:, M - 1:]), (o0 + L, yi[:, M - 1:])):
            ok = o < n
            out[o[ok]] = vals[ok]
        return out
    o = b[:, None] * L - (M - 1) + nn[None]
    vr, vi = yr[:, M - 1:], yi[:, M - 1:]
    if case.turns is not None:
        fix = int(math.floor((case.turns % 1.0) * 2 ** 64)) % (1 << 64)
        for bb in range(nblocks):
            pr, pi = _phasor(fix * ((n0 + s + bb * L - (M - 1)) % (1 << 64)) % (1 << 64))
            vr[bb], vi[bb] = _cmul(vr[bb], vi[bb], pr, pi)
    ok = o < n
    out[o[ok]] = vr[ok] + 1j * vi[ok]
    return out


def emulate(case, x, n0, calls):
    """The stream's kept outputs as the overlap-save kernels compute them (every call must run overlap-save)."""
    full = np.zeros(len(x), np.complex64)
    s = 0
    for (path, _, _), n in zip(case.plans(n0, calls), calls):
        assert path in ("fft", "fdl")
        full[s:s + n] = _emulate_call(case, x, n0, s, n, 0)
        s += n
    y = full[case.kept(n0, len(x))]
    return y.real if case.kind == "rrrf" else y


EMULATED = ["os_crcf_m128", "os_cccf_m33", "os_crcf_m513_impulse256", "os_crcf_m129_alternating", "dec_rrrf_m33_d2",
            "dec_cccf_m513_d33", "real_m257_d1", "real_m2_d5", "hilbert_m65_fft", "hilbert_m513_fft",
            "rot_cccf_m129_d5", "rot_crcf_m33_d1", "rot_crcf_m513_d33", "fdl_crcf_m514", "fdl_cccf_m2048",
            "fdl_crcf_m2049", "fdl_cccf_m8192"]
EMU_CALLS = 12          # the stream's first calls: the short ones, per +- 1 and the k per +- 1 with interior blocks


@pytest.mark.parametrize("name", EMULATED)
def test_float32_emulation_stays_within_a_quarter_of_the_bound(name):
    case = T.CASES[name]()
    n0, calls = case.streams[0]
    calls = calls[:EMU_CALLS]
    x = case.gen(sum(calls))
    ref, bound, _, _ = case.expect(x, n0, calls)
    got = emulate(case, x, n0, calls)
    ex = F.excess(got, ref, bound)
    print("\n%s: float32 emulation at %.3g of the bound" % (name, ex))
    assert ex < 0.25, "%s: %.3g of the bound" % (name, ex)


@pytest.mark.parametrize("real", [False, True])
def test_c_oracle_overlap_save_stays_within_a_quarter_of_the_bound(real):
    """lr_oracle.c's four-step float32 overlap-save (N = 1024 at M = 128, the kernel's geometry from a zero history;
    real input packs two blocks per transform as the kernel does), one call, against the kernel's bound."""
    lib = cbuild.load()
    name = "real_m128_d1" if real else "os_crcf_m128"
    case = T.CASES[name]()
    n = 200000
    x = case.gen(n)
    h = np.ascontiguousarray(case.h)
    f = lib.lro_firfft_new(h.ctypes.data, 128, 0, int(real))
    y = np.zeros(n + 4096, np.float32 if real else np.complex64)
    try:
        proc = lib.lro_firfft_process_r if real else lib.lro_firfft_process_c
        flush = lib.lro_firfft_flush_r if real else lib.lro_firfft_flush_c
        no = proc(f, x.ctypes.data, n, y.ctypes.data)
        no += flush(f, y[no:].ctypes.data)
    finally:
        lib.lro_firfft_free(f)
    assert no == n
    ref, bound, _, _ = case.expect(x, 0, [n])
    ex = F.excess(y[:n], ref, bound)
    print("\n%s: C oracle at %.3g of the bound" % (name, ex))
    assert ex < 0.25


# ---- the inputs separate right from wrong -----------------------------------------------------------------------------
def _prefix(calls):
    """The calls before the long one: every mutant is causal, so its margin there is a lower bound of its margin over
    the whole stream."""
    k = max(range(len(calls)), key=lambda i: calls[i])
    return calls[:k] if calls[k] >= 1 << 20 else calls


def margins(case):
    """(smallest over mutants of the largest |mutant - reference| / bound, which mutant, how many mutants)"""
    worst, count = (np.inf, None), 0
    for n0, calls in case.streams:
        calls = _prefix(calls)
        x = case.gen(sum(calls))
        ref, bound, _, _ = case.expect(x, n0, calls)
        for name, mut in case.mutants(x, n0, calls).items():
            count += 1
            m = F.excess(mut, ref, bound)
            if m < worst[0]:
                worst = (m, "%s (n0=%d)" % (name, n0))
    return worst[0], worst[1], count


FAMILIES = ("os_", "dec_crcf", "dec_cccf", "dec_rrrf", "rot_", "real_", "hilbert_", "fdl_", "catchall_", "direct_",
            "auto_")


@pytest.mark.parametrize("family", FAMILIES)
def test_every_mutant_exceeds_four_times_the_bound(family):
    report = []
    for name, make in T.CASES.items():
        if not name.startswith(family):
            continue
        margin, which, count = margins(make())
        assert count, name
        report.append((margin, name, which))
        assert margin >= 4, "%s: mutant '%s' stays within %.3gx of the bound" % (name, which, margin)
    assert report
    margin, name, which = min(report)
    print("\n%s: %d cases, smallest mutant margin %.3gx (%s, %s)" % (family, len(report), margin, name, which))


def test_bounds_are_per_block():
    """On a bursty stream the bound of a quiet block is set by that block: orders of magnitude below a loud one's."""
    case = T.CASES["fdl_crcf_m8192_impulse8191"]()
    n0, calls = case.streams[0]
    calls = _prefix(calls)
    x = case.gen(sum(calls))
    _, bound, _, _ = case.expect(x, n0, calls)
    assert np.max(bound) / np.min(bound[8192:]) > 100
