"""Numpy models of the two IIR kernels for filters with at most 10 taps on each side (iir.cu), and the per-output error
bound the GPU outputs are held to.

ScanModel runs iir1_scan_kernel (IirBlock: na <= 2, nb <= 9) call by call in float32: the block's coefficients
b^ = fl32(b / a0), c^ = fl32(-a1 / a0); the power table cp[k] = fl32(c^(8 2^k)) built in double as launch_iir1 does;
4096-sample tiles of 512 threads x V = 8 samples; per thread the FIR sum (a chain of nb FMAs) and V sequential steps;
a Kogge-Stone warp scan with cp[0..4]; Horner over the 16 warps with cp[5]; the tile aggregate; then either the LOCAL
restart (|c^|^512 < 1e-12: every tile after the first restarts 512 samples early from a zero state) or the decoupled
look-back.  The look-back's order depends on timing in the kernel; the model takes one fixed walk (`walk` = the distance
at which a predecessor's inclusive prefix is found, None = aggregates only, down to tile 0 or the first dead
predecessor, |cT^d| < 1e-12).  Every FMA is a float64 product-sum rounded once to float32 (the product of two float32
values is exact in float64).  Calls longer than 2^27 samples are split as IirBlock::run splits them, and a fused
decimator keeps the samples whose global index is a multiple of D.

GeneralModel runs iir_general_kernel (IirGeneralBlock: 2 < na <= 10 or nb = 10): the float64 impulse response of 1/A^
gives the warm-up W (the last index where |h| >= 1e-10 of its peak in 65536 samples, plus na + nb; -1 when it does not
decay); chunks of max(4W, 512) samples, each run by one thread from W samples early with true past inputs and zero past
outputs (chunk 0 from the carried state); the direct form I as a chain of nb + na - 1 FMAs per output, in the kernel's
tap order; carried state as IirGeneralBlock::run leaves it.

Bound, per output n, against the float64 recurrence y_ref (scipy lfilter on the user's taps, as the oracle):

    |y_gpu[n] - y_ref[n]| <= u32 |y_ref[n]| + C E_alg[n] + 2 |trunc[n]| + |coef[n]| + C u64 E_ref[n],     C = 2

  - E_alg, a first-order running error analysis of the model's own operations (u32 = 2^-24; complex values measured
    by |re| + |im|).  Each operation injects u32 times the magnitude of the value it produces; an operation that
    applies a power-table entry or a product of entries (cp, f_lane, f_thread, cpow, the look-back weights) also
    injects that entry's own error (computed exactly against the extended-precision power) times the magnitude it
    multiplies.  Scan: an error in a value that stands for the recurrence at sample t reaches later outputs through
    |c^|^k, so E_alg = lfilter([1], [1, -|c^|], injections) + the errors of the per-thread values (excl, carry_t, the
    output FMA), which reach their own outputs only.  Each look-back round is bounded by the magnitude sum of every
    term any walk could use (the aggregate and the prefix of each predecessor down to tile 0 or the first dead one),
    so the bound holds whatever order the kernel's sum takes.  General: each output's FMA chain injects
    gamma(nb + na - 1) (sum |b^||x| + sum |a^||y|), with |y| the largest value any chunk's thread computes for that
    sample (warm-ups included), propagated through |h| of 1/A^.
  - trunc, computed exactly in float64: the model run in float64 (walk = None, the longest walk) minus the float64
    recurrence with the block's coefficients; this is what the LOCAL restart, the dead-predecessor cut-off and the
    general kernel's zero-output restart leave out.
  - coef = |lfilter64(b^, a^) - lfilter64(b / a0, a / a0)|, the block's one rounding of the normalised taps.  It is
    exactly 0 when a0 = +-2^k.
  - u32 |y_ref| for the one rounding of each output to float32; E_ref (iir_order_ref.ref_error) bounds the float64
    reference's own rounding.
C = 2 absorbs gamma_m = m u / (1 - m u), the double rounding of the emulated FMAs and second-order products.  Nothing
is fitted to observed errors; `test_iir_small_ref.py::test_bound_is_tight` shows how far above u32 |y_ref| it sits.
"""
import functools

import numpy as np
import scipy.signal

from tests import iir_order_ref as R

U32, U64 = R.U32, R.U64
C_BOUND = 2.0
T, V, NT, WARM = 4096, 8, 512, 512        # iir.cu: IIR_TILE, IIR_V, IIR_THREADS, IIR_WARM
LAUNCH = 1 << 27                          # iir_max_per_launch: 2^15 tiles
FLOOR = 2.0 ** -140                       # per sample: the absolute error of float32 results that are subnormal
GEN_LIMIT = 1 << 16                       # IirGeneralBlock: impulse-response span searched for W

SCAN_MUTANTS = ("power", "lookback", "dead", "warm", "xhist", "ystate", "phase", "a0")
GENERAL_MUTANTS = ("halfw", "first", "yrev", "xhist", "decay")


def _f32(v):
    return np.asarray(v, np.float64).astype(np.float32).astype(np.float64)


def _ident(v):
    return np.asarray(v, np.float64)


def _comps(x, cplx):
    x = np.asarray(x)
    if cplx:
        return np.stack([x.real, x.imag], -1).astype(np.float64)
    return np.asarray(x.real, np.float64)[:, None]


def _join(y, cplx):
    return y[..., 0] + 1j * y[..., 1] if cplx else y[..., 0].copy()


def _mag(v):
    """|re| + |im| over the trailing component axis"""
    return np.sum(np.abs(v), -1)


def _err(vals, c, ms):
    """|vals - c^ms| in extended precision: the exact error of a float32 table of powers of c"""
    exact = np.longdouble(c) ** np.asarray(ms, np.longdouble)
    return np.abs(np.asarray(vals, np.longdouble) - exact).astype(np.float64)


def _pow(c, ms):
    return (np.longdouble(c) ** np.asarray(ms, np.longdouble)).astype(np.float64)


def _tree(v, r):
    """the kernel's xor-butterfly sum of 32 lanes: lane l takes l + l ^ off, off = 16 .. 1"""
    for off in (16, 8, 4, 2, 1):
        v = r(v[:off] + v[off:2 * off])
    return v[0]


def scan_coefs(b, a, mutant=None):
    """IirBlock's coefficients: b^ = fl32(b / a0), c^ = fl32(-a1 / a0), divided in double (capi.cu)"""
    b64, a64 = np.asarray(b, np.float64), np.asarray(a, np.float64)
    a0 = 1.0 if mutant == "a0" else a64[0]
    return _f32(b64 / a0), float(_f32(-a64[1] / a0)) if len(a64) > 1 else 0.0


def is_local(c):
    return abs(float(c)) ** WARM < 1e-12


class ScanModel:
    """mutant: None, 'power' (cp one power of c off), 'lookback' (a predecessor's aggregate taken for its inclusive
    prefix), 'dead' (dead-predecessor cut-off 1e-6 instead of 1e-12), 'warm' (LOCAL warm-up of 256 samples), 'xhist'
    (input history dropped across calls), 'ystate' (carried output dropped across calls), 'phase' (decimation phase
    off by one after the first call), 'a0' (a0 not divided out).  exact: every operation and table in float64 (the
    truncation model)."""

    def __init__(self, b, a, cplx, D=1, mutant=None, walk=1, exact=False):
        self.b, self.c = scan_coefs(b, a, mutant)
        self.nb, self.cplx, self.K, self.D = len(self.b), cplx, 2 if cplx else 1, D
        self.mutant, self.walk, self.exact = mutant, walk, exact
        self.r = _ident if exact else _f32
        c = self.c
        self.local = is_local(c)
        self.warm = WARM // 2 if mutant == "warm" else WARM
        self.thr = float(np.float32(1e-6 if mutant == "dead" else 1e-12))
        # cp[k] = c^(V 2^k), k = 0 .. 9, built in double from c^V and rounded once (launch_iir1)
        p = 1.0
        for _ in range(V + (1 if mutant == "power" else 0)):
            p *= c
        cp = []
        for _ in range(10):
            cp.append(p)
            p = p * p
        ms = V * 2.0 ** np.arange(10)
        if exact:
            self.cp, self.cp_e = _pow(c, ms), np.zeros(10)
        else:
            self.cp = _f32(cp)
            self.cp_e = _err(self.cp, c, ms)
        r, cpv = self.r, self.cp
        lane = np.arange(32)
        fl = np.ones(32)
        for k in range(5):
            fl = np.where(lane & (1 << k), r(fl * cpv[k]), fl)
        ft = np.tile(fl, 16)
        warp = np.repeat(np.arange(16), 32)
        for k in range(4):
            ft = np.where(warp & (1 << k), r(ft * cpv[5 + k]), ft)
        cpow = [c]
        for _ in range(V - 1):
            cpow.append(float(r(cpow[-1] * c)))
        self.fa = float(r(fl[31] * cpv[0]))                       # c^256: a warp's span, for the tile aggregate
        if exact:
            fl, ft, cpow, self.fa = _pow(c, V * lane), _pow(c, V * np.arange(NT)), _pow(c, np.arange(1, V + 1)), float(_pow(c, 256))
        self.fl, self.ft, self.cpow = fl, ft, np.asarray(cpow, np.float64)
        self.fl_e, self.ft_e = _err(fl, c, V * lane), _err(ft, c, V * np.arange(NT))
        self.cpow_e, self.fa_e = _err(self.cpow, c, np.arange(1, V + 1)), float(_err([self.fa], c, [256])[0])
        # look-back weights: wl = cT^lane by squaring, mult = (cT^32)^round, as the kernel computes them in float32
        cT = cpv[9]
        wl, pw = np.ones(32), cT
        for k in range(5):
            wl = np.where(lane & (1 << k), r(wl * pw), wl)
            pw = float(r(pw * pw))
        self.wl, self.pw32 = wl, pw
        self.wl_e = _err(wl, c, float(T) * lane)
        self.xh = np.zeros((self.nb - 1, self.K))
        self.ys = np.zeros(self.K)
        self.pending = 0.0                # error of the carried output, injected at the next call's first sample
        self.consumed = 0

    def _mults(self, rounds):
        m = [1.0]
        for _ in range(rounds - 1):
            m.append(float(self.r(m[-1] * self.pw32)))
        return np.asarray(m)

    def process(self, x):
        """Outputs of one IirBlock::run call (decimated when D > 1).  Also sets self.full (every sample's value),
        self.inj (errors that propagate through |c^|^k, at the sample they stand for) and self.direct (errors of a
        sample's own output)."""
        xc = _comps(x, self.cplx)
        n = len(xc)
        full, inj, direct = np.zeros((n, self.K)), np.zeros(n), np.zeros(n)
        outs = []
        for s in range(0, n, LAUNCH):
            e = min(n, s + LAUNCH)
            full[s:e], inj[s:e], direct[s:e] = self._launch(xc[s:e])
            first = (-self.consumed) % self.D
            if self.mutant == "phase" and self.consumed:
                first = (first + 1) % self.D
            outs.append(full[s + first:e:self.D])
            self.consumed += e - s
        self.full, self.inj, self.direct = full, inj, direct
        y = np.concatenate(outs) if outs else np.zeros((0, self.K))
        return _join(y, self.cplx)

    def _launch(self, x):
        n, K, nh, r, c = len(x), self.K, self.nb - 1, self.r, self.c
        if self.local:
            P = T - self.warm
            tiles = 1 if n <= T else 1 + -(-(n - T) // P)
            t_ = np.arange(tiles)
            span0 = np.where(t_ == 0, 0, T + (t_ - 1) * P - self.warm)
            lo = np.where(t_ == 0, 0, self.warm)
        else:
            tiles = -(-n // T)
            span0, lo = np.arange(tiles) * T, np.zeros(tiles, int)
        ext = np.concatenate([self.xh, x, np.zeros((T + V, K))])
        idx = span0[:, None] + np.arange(T)[None, :]                    # (tiles, T) global sample index
        u, firm = None, 0.0
        for j in range(self.nb):
            xj = ext[idx + nh - j]
            u = r(self.b[j] * xj) if j == 0 else r(self.b[j] * xj + u)
            firm = firm + abs(self.b[j]) * _mag(xj)
        yl = u.reshape(tiles, NT, V, K).copy()
        for i in range(1, V):
            yl[:, :, i] = r(c * yl[:, :, i - 1] + yl[:, :, i])
        inj_t = (self.nb * U32 * firm).reshape(tiles, NT, V)
        inj_t[:, :, 1:] += U32 * _mag(yl[:, :, 1:])
        # warp scan of the thread end values
        B = yl[:, :, V - 1].reshape(tiles, 16, 32, K).copy()
        ks = np.zeros((tiles, 16, 32))
        for k in range(5):
            s = 1 << k
            o = np.zeros_like(B)
            o[:, :, s:] = B[:, :, :-s]
            nv = r(self.cp[k] * o + B)
            ks[:, :, s:] += U32 * _mag(nv[:, :, s:]) + self.cp_e[k] * _mag(o[:, :, s:])
            B[:, :, s:] = nv[:, :, s:]
        inj_t[:, :, V - 1] += ks.reshape(tiles, NT)
        prevB = np.zeros_like(B)
        prevB[:, :, 1:] = B[:, :, :-1]
        # Horner over the warps: carryW[w] = value at the end of warp w - 1, zero state from the tile start
        carryW = np.zeros((tiles, 16, K))
        cw = np.zeros((tiles, K))
        flat = inj_t.reshape(tiles, T)
        for w in range(1, 16):
            nv = r(self.cp[5] * cw + B[:, w - 1, 31])
            flat[:, w * 256 - 1] += U32 * _mag(nv) + self.cp_e[5] * _mag(cw)
            cw = carryW[:, w] = nv
        excl = r(self.fl[None, None, :, None] * carryW[:, :, None, :] + prevB)
        agg = r(self.fa * carryW[:, 15] + B[:, 15, 31])
        flat[:, T - 1] += U32 * _mag(agg) + self.fa_e * _mag(carryW[:, 15])
        carry = np.zeros((tiles, K))
        carry[0] = self.ys
        if not self.local:
            self._lookback(tiles, agg, carry, flat)
        flat[0, 0] += self.pending
        # per-thread values: they reach their own outputs only
        excl = excl.reshape(tiles, NT, K)
        ct = r(self.ft[None, :, None] * carry[:, None, :] + excl)
        vals = r(self.cpow[None, None, :, None] * ct[:, :, None, :] + yl)
        e_ct = (np.tile(self.fl_e, 16)[None, :] * _mag(carryW).repeat(32, 1) + U32 * _mag(excl)
                + self.ft_e[None, :] * _mag(carry)[:, None] + U32 * _mag(ct))
        dir_t = np.abs(self.cpow)[None, None, :] * e_ct[:, :, None] + self.cpow_e[None, None, :] * _mag(ct)[:, :, None]
        # scatter: each tile stores [lo, hi) of its span; every span's injections count (a LOCAL warm-up included)
        hi = np.minimum(T, n - span0)
        rel = np.arange(T)[None, :]
        store = (rel >= lo[:, None]) & (rel < hi[:, None])
        y = np.zeros((n, K))
        y[idx[store]] = vals.reshape(tiles, T, K)[store]
        direct = np.zeros(n)
        direct[idx[store]] = dir_t.reshape(tiles, T)[store]
        inj = np.zeros(n)
        ok = idx < n
        np.add.at(inj, idx[ok], flat[ok])
        inj += FLOOR
        # carried state
        self.pending = direct[n - 1] + U32 * _mag(y[n - 1])
        self.ys = np.zeros(K) if self.mutant == "ystate" else y[n - 1].copy()
        if nh and self.mutant != "xhist":
            self.xh = np.concatenate([self.xh, x])[-nh:]
        return y, inj, direct

    def _lookback(self, tiles, agg, carry, flat):
        """carry[t] for t >= 1 by the model's walk; the bound term of every round covers any walk"""
        r, K = self.r, self.K
        rounds = tiles // 32 + 2
        mult = self._mults(rounds)
        mult_e = _err(mult, self.c, float(T) * 32 * np.arange(rounds))
        d = np.arange(1, 32 * rounds + 1)
        wl_d, wle_d = np.tile(self.wl, rounds), np.tile(self.wl_e, rounds)
        m_d, me_d = mult.repeat(32), mult_e.repeat(32)
        w_d = np.abs(_f32(wl_d * m_d))
        dead = np.flatnonzero(w_d < self.thr)
        dead_d = int(d[dead[0]]) if dead.size else 1 << 62      # the first dead distance
        pfx = np.zeros((tiles, K))
        pfx[0] = r(self.cp[9] * carry[0] + agg[0])
        flat[0, T - 1] += U32 * _mag(pfx[0]) + self.cp_e[9] * _mag(carry[0])
        magn = np.zeros(tiles)
        magn[0] = max(_mag(agg[0]), _mag(pfx[0]))
        for t in range(1, tiles):
            # bound: every candidate term down to tile 0 or the first dead predecessor
            L = min(t, dead_d - 1)
            M = magn[t - 1::-1][:L]
            nr = (L - 1) // 32 + 1
            ww = np.abs(wl_d[:L] * m_d[:L])
            flat[t, 0] += float(np.sum(((6 + nr) * U32 * ww + wle_d[:L] * np.abs(m_d[:L]) + np.abs(wl_d[:L]) * me_d[:L]) * M))
            # value: the model's walk
            acc = np.zeros(K)
            dd, stop = 1, False
            for rnd in range(rounds):
                lanes = np.zeros((32, K))
                for ln in range(32):
                    j = t - dd
                    if dd >= dead_d:
                        stop = True
                        break
                    pf = j == 0 or (self.walk is not None and dd >= self.walk)
                    v = (agg[j] if self.mutant == "lookback" else pfx[j]) if pf else agg[j]
                    lanes[ln] = r(self.wl[ln] * v)
                    dd += 1
                    if pf:
                        stop = True
                        break
                acc = r(mult[rnd] * _tree(lanes, r) + acc)
                if stop:
                    break
            carry[t] = acc
            pfx[t] = r(self.cp[9] * acc + agg[t])
            flat[t, T - 1] += U32 * _mag(pfx[t]) + self.cp_e[9] * _mag(acc)
            magn[t] = max(_mag(agg[t]), _mag(pfx[t]))


# ---- the general-order kernel -----------------------------------------------------------------------------------------
def general_coefs(b, a, mutant=None):
    """IirGeneralBlock's coefficients: fl32(b / a0), fl32(a / a0), divided in double"""
    b64, a64 = np.asarray(b, np.float64), np.asarray(a, np.float64)
    return _f32(b64 / a64[0]), _f32(a64 / a64[0])


def warm_length(ah, nb, crit=1e-10):
    """IirGeneralBlock's W: the last index where the float64 impulse response of 1/A^ is >= crit of its peak, within
    65536 samples, plus na + nb; -1 when that reaches the end of the span"""
    return _warm_length(tuple(float(v) for v in ah), nb, crit)


@functools.lru_cache(maxsize=None)
def _warm_length(a, nb, crit):
    na = len(a)
    h = [0.0] * GEN_LIMIT
    peak, last = 0.0, 0
    for i in range(GEN_LIMIT):
        v = 1.0 if i == 0 else 0.0
        for j in range(1, min(na - 1, i) + 1):
            v -= a[j] * h[i - j]
        h[i] = v
        if abs(v) > peak:
            peak = abs(v)
        if not np.isfinite(v):
            last = GEN_LIMIT
            break
        if abs(v) >= crit * peak:
            last = i
    return -1 if last + na + nb >= GEN_LIMIT - 1 else last + na + nb


class GeneralModel:
    """mutant: None, 'halfw' (W halved), 'first' (a chunk's first stored sample taken from the next chunk's warm-up),
    'yrev' (carried outputs read newest-first), 'xhist' (input history dropped across calls), 'decay' (W from a 1e-5
    criterion).  exact: float64 (scipy lfilter per chunk), the truncation model; it also records in self.ymag the
    largest |y| any chunk's thread computes for each sample."""

    def __init__(self, b, a, cplx, mutant=None, exact=False):
        self.b, self.a = general_coefs(b, a)
        self.nb, self.na, self.cplx, self.K = len(self.b), len(self.a), cplx, 2 if cplx else 1
        self.mutant, self.exact = mutant, exact
        self.r = _ident if exact else _f32
        w = warm_length(self.a, self.nb, 1e-5 if mutant == "decay" else 1e-10)
        self.W = w // 2 if mutant == "halfw" and w > 0 else w
        self.xh = np.zeros((self.nb - 1, self.K))
        self.yh = np.zeros((self.na - 1, self.K))          # oldest first

    def plan(self, n):
        """(chunk, warm) as launch_iir_general chooses them"""
        if 0 <= self.W < n:
            return max(4 * self.W, 512), self.W
        return n, n

    def process(self, x):
        xc = _comps(x, self.cplx)
        n, K, nh, ny, r = len(xc), self.K, self.nb - 1, self.na - 1, self.r
        if n == 0:
            self.ymag = np.zeros(0)
            return _join(np.zeros((0, K)), self.cplx)
        chunk, warm = self.plan(n)
        starts = np.arange(0, n, chunk)
        ext = np.concatenate([self.xh, xc])              # ext[i + nh] = x[i]
        y = np.zeros((n, K))
        ymag = np.zeros(n)
        yh = self.yh[::-1] if self.mutant == "yrev" else self.yh
        if self.exact:
            for g, s in enumerate(starts):
                e = min(n, s + chunk)
                beg = max(0, s - warm)
                ypast = yh[::-1] if s - warm <= 0 else np.zeros((ny, K))     # newest first
                xpast = ext[beg:beg + nh][::-1]
                seg = np.zeros((e - beg, K))
                for k in range(K):
                    zi = scipy.signal.lfiltic(self.b, self.a, ypast[:, k], xpast[:, k]) if max(nh, ny) else None
                    if zi is None:
                        seg[:, k] = scipy.signal.lfilter(self.b, self.a, xc[beg:e, k])
                    else:
                        seg[:, k] = scipy.signal.lfilter(self.b, self.a, xc[beg:e, k], zi=zi)[0]
                ymag[beg:e] = np.maximum(ymag[beg:e], _mag(seg))
                lo = s - beg - (1 if self.mutant == "first" and g else 0)
                y[beg + lo:e] = seg[lo:]
        else:
            # FIR part: the same for every thread (true past inputs)
            fir = None
            for j in range(self.nb):
                xj = ext[nh - j:nh - j + n]
                fir = r(self.b[j] * xj) if j == 0 else r(self.b[j] * xj + fir)
            G = len(starts)
            ends = np.minimum(n, starts + chunk)
            begs = np.maximum(0, starts - warm)
            ys = np.zeros((G, max(ny, 1), K))                    # ys[:, j] = y[i - 1 - j]
            from_state = starts - warm <= 0
            if ny:
                ys[from_state, :ny] = yh[::-1]
            span = int(np.max(ends - begs))
            fix = np.zeros((G, K))
            neg_a = -self.a
            for k in range(span):
                i = begs + k
                act = i < ends
                ii = np.minimum(i, n - 1)
                acc = fir[ii]
                for j in range(1, self.na):
                    acc = r(neg_a[j] * ys[:, j - 1] + acc)
                if ny:
                    ys[:, 1:] = ys[:, :-1]
                    ys[:, 0] = acc
                keep = act & (i >= starts)
                y[ii[keep]] = acc[keep]
                if self.mutant == "first":
                    sel = act & (i == starts - 1) & (np.arange(G) > 0)
                    fix[sel] = acc[sel]
            if self.mutant == "first":
                y[starts[1:] - 1] = fix[1:]
        if nh and self.mutant != "xhist":
            self.xh = ext[-nh:].copy()
        elif nh:
            self.xh = np.zeros((nh, K))
        if ny:
            self.yh = np.concatenate([self.yh, y])[-ny:].copy()
        self.ymag = ymag
        return _join(y, self.cplx)


# ---- the bound --------------------------------------------------------------------------------------------------------
def _lfilter(b, a, x, cplx):
    if len(x) == 0:
        return np.zeros(0, np.complex128 if cplx else np.float64)
    return scipy.signal.lfilter(np.asarray(b, np.float64), np.asarray(a, np.float64),
                                np.asarray(x).astype(np.complex128 if cplx else np.float64))


def reference(b, a, xs, cplx):
    """float64 outputs of the recurrence over the calls xs, with the user's taps (the oracle's IIRFilterFast)"""
    x = np.concatenate([np.asarray(v) for v in xs])
    return x, _lfilter(b, a, x, cplx)


def scan_bound(b, a, xs, cplx, D=1):
    """(float32 model outputs, float64 reference, per-output bound) for the stream of calls xs through IirBlock with a
    fused decimator D (see the module docstring)"""
    m = ScanModel(b, a, cplx, D)
    m64 = ScanModel(b, a, cplx, D, walk=None, exact=True)
    ys, inj, direct, full64 = [], [], [], []
    for x in xs:
        ys.append(m.process(x))
        inj.append(m.inj)
        direct.append(m.direct)
        m64.process(x)
        full64.append(_join(m64.full, cplx))
    x, ref = reference(b, a, xs, cplx)
    y = np.concatenate(ys)
    inj, direct, full64 = np.concatenate(inj), np.concatenate(direct), np.concatenate(full64)
    bh, ch = m.b, m.c
    yhat = _lfilter(bh, [1.0, -ch], x, cplx)
    b64, a64 = np.asarray(b, np.float64), np.asarray(a, np.float64)
    coef = np.abs(yhat - _lfilter(b64 / a64[0], a64 / a64[0], x, cplx))
    trunc = np.abs(full64 - yhat)
    e_alg = scipy.signal.lfilter([1.0], [1.0, -abs(ch)], inj) + direct
    e_ref = R.ref_error(bh, np.array([ch]), x, yhat, cplx, lambda w: scipy.signal.lfilter([1.0], [1.0, -abs(ch)], w))
    bnd = U32 * np.abs(ref) + C_BOUND * e_alg + 2 * trunc + coef + C_BOUND * U64 * e_ref
    terms = {"alg": C_BOUND * e_alg, "trunc": 2 * trunc, "coef": coef}
    return y, ref[::D], bnd[::D], {k: v[::D] for k, v in terms.items()}


def general_bound(b, a, xs, cplx):
    """(float32 model outputs, float64 reference, per-output bound, terms) for the stream of calls xs through
    IirGeneralBlock"""
    m64 = GeneralModel(b, a, cplx, exact=True)
    full64, ymag = [], []
    for v in xs:
        full64.append(m64.process(v))
        ymag.append(m64.ymag)
    x, ref = reference(b, a, xs, cplx)
    full64, ymag = np.concatenate(full64), np.concatenate(ymag)
    bh, ah = m64.b, m64.a
    yhat = _lfilter(bh, ah, x, cplx)
    b64, a64 = np.asarray(b, np.float64), np.asarray(a, np.float64)
    coef = np.abs(yhat - _lfilter(b64 / a64[0], a64 / a64[0], x, cplx))
    trunc = np.abs(full64 - yhat)
    N, nb, na = len(x), len(bh), len(ah)
    m = nb + na - 1
    gamma = m * U32 / (1 - m * U32)
    tm = np.convolve(R.mag(x.astype(np.complex128 if cplx else np.float64)), np.abs(bh))[:N]
    if na > 1:
        tm += np.convolve(np.concatenate([[0.0], np.maximum(ymag, np.abs(yhat))[:-1]]), np.abs(ah[1:]))[:N]
    h = R.impulse(-ah[1:], N)
    e_alg = R._causal_conv(h, gamma * tm + FLOOR)
    e_ref = R.ref_error(bh, -ah[1:], x, yhat, cplx, lambda w: R._causal_conv(h, w))
    bnd = U32 * np.abs(ref) + C_BOUND * e_alg + 2 * trunc + coef + C_BOUND * U64 * e_ref
    return ref, bnd, {"alg": C_BOUND * e_alg, "trunc": 2 * trunc, "coef": coef}


def scan_closed_excess(b, a, x, got, D=1, block=1 << 23):
    """max over the kept outputs of |got - y_ref| / bound for one long real call through IirBlock with a fused
    decimator D, with a bound that needs no model run, so that a 2^27-sample call fits in memory.  For |c^| < 1 every
    value the kernel forms at sample n -- a zero-state partial sum, a carried state, a per-thread value -- is at most
    m[n] = sum_k |c^|^k sum_j |b^_j| |x[n - k - j]| = lfilter(|b^|, [1, -|c^|], |x|)[n] in magnitude.  With Mw the
    largest m over the tiles a sample's tile, its look-back's live predecessors and the next tile can touch, every
    operation that ScanModel counts is charged to every sample (a thread's, warp's or tile's operations once per
    sample instead of once per thread, warp or tile; twice over a LOCAL warm-up):

        inj[n]    = nb u32 sum_j |b^_j||x[n-j]| + u32 m[n] + K Mw[n]      (K: every per-sample, per-thread, per-warp,
                                                                          per-tile and look-back operation with its
                                                                          table errors, from ScanModel's tables)
        bound[n]  = u32 |y_ref| + C (lfilter([1], [1, -|c^|], inj) + Kd Mw) + 2 |c^|^S Mw + C u64 (nb + 4) Mw / (1 - |c^|)

    with Kd the per-thread values' errors and S the samples a restart or the dead cut-off leaves behind (512, or T times
    the number of live predecessors).  It is order-independent and looser than scan_bound (tests/test_iir_small_ref.py
    checks both on the same stream); the normalisation must be exact (a0 = +-2^k)."""
    m = ScanModel(b, a, False, D)
    bh, c = m.b, abs(m.c)
    b64, a64 = np.asarray(b, np.float64), np.asarray(a, np.float64)
    assert c < 1.0 and np.array_equal(bh, b64 / a64[0]) and (len(a64) < 2 or -a64[1] / a64[0] == m.c)
    # live look-back predecessors and the weight, table and rounding constants of every operation
    rounds = 2 + (1 << 10)
    mult = m._mults(rounds)
    mult_e = _err(mult, m.c, float(T) * 32 * np.arange(rounds))
    wl_d, wle_d = np.tile(m.wl, rounds), np.tile(m.wl_e, rounds)
    m_d, me_d = mult.repeat(32), mult_e.repeat(32)
    dead = np.flatnonzero(np.abs(_f32(wl_d * m_d)) < m.thr)
    live = 0 if m.local else int(dead[0]) if dead.size else len(wl_d)
    assert m.local or dead.size, "a look-back that never cuts off: use scan_bound"
    nr = (live - 1) // 32 + 1 if live else 0
    Kw = float(np.sum((6 + nr) * U32 * np.abs(wl_d[:live] * m_d[:live]) + wle_d[:live] * np.abs(m_d[:live])
                      + np.abs(wl_d[:live]) * me_d[:live]))
    Kd = float(np.max(m.fl_e) + np.max(m.ft_e) + np.max(m.cpow_e)) + 2 * U32
    K = (5 * U32 + float(np.sum(m.cp_e[:5]))) + (U32 + m.cp_e[5]) + (U32 + m.fa_e) + (U32 + m.cp_e[9]) + Kw + Kd + U32
    K *= 2 if m.local else 1
    S = WARM if m.local else T * live
    x = np.asarray(x, np.float32)
    n = len(x)
    ax_b = np.abs(bh)
    # pass 1: the largest m per tile
    tiles = -(-n // T)
    tmax = np.zeros(tiles)
    zi_m = np.zeros(max(len(bh), 2) - 1)
    for s in range(0, n, block):
        ax = np.abs(x[s:s + block].astype(np.float64))
        mm, zi_m = scipy.signal.lfilter(ax_b, [1.0, -c], ax, zi=zi_m)
        pad = (-len(mm)) % T
        tmax[s // T:s // T + -(-len(mm) // T)] = np.max(np.concatenate([mm, np.zeros(pad)]).reshape(-1, T), 1)
    back = live + 2
    padded = np.concatenate([np.zeros(back), tmax, np.zeros(2)])
    wmax = np.lib.stride_tricks.sliding_window_view(padded, back + 3).max(1)[:tiles]     # tiles k - back .. k + 2
    # pass 2: reference, bound and excess over the kept outputs
    zi_r = np.zeros(max(len(b64), len(a64)) - 1)
    zi_m, zi_f, zi_e = np.zeros(max(len(bh), 2) - 1), np.zeros(max(len(bh) - 1, 1)), np.zeros(1)
    worst, pos = 0.0, 0
    got = np.asarray(got)
    kept = -(-n // D)
    if len(got) != kept:
        return np.inf
    for s in range(0, n, block):
        xb = x[s:s + block].astype(np.float64)
        ax = np.abs(xb)
        ref, zi_r = scipy.signal.lfilter(b64, a64, xb, zi=zi_r) if len(zi_r) else (scipy.signal.lfilter(b64, a64, xb), zi_r)
        mm, zi_m = scipy.signal.lfilter(ax_b, [1.0, -c], ax, zi=zi_m)
        F, zi_f = scipy.signal.lfilter(ax_b, [1.0], ax, zi=zi_f) if len(bh) > 1 else (ax_b[0] * ax, zi_f)
        Mw = wmax[(s + np.arange(len(xb))) // T]
        inj = len(bh) * U32 * F + U32 * mm + K * Mw + FLOOR
        E, zi_e = scipy.signal.lfilter([1.0], [1.0, -c], inj, zi=zi_e)
        bnd = U32 * np.abs(ref) + C_BOUND * (E + Kd * Mw) + 2 * c ** S * Mw + C_BOUND * U64 * (len(bh) + 4) * Mw / (1 - c)
        first = (-s) % D
        k = len(range(first, len(xb), D))
        g = got[pos:pos + k].astype(np.float64)
        err = np.abs(g - ref[first::D])
        err = np.where(np.isfinite(err), err, np.inf)
        worst = max(worst, float(np.max(err / bnd[first::D])) if k else 0.0)
        pos += k
    return worst


def excess(got, ref, bnd):
    """max over n of |got - ref| / bound; a length mismatch or a non-finite output counts as infinitely far off"""
    got = np.asarray(got)
    if got.shape != ref.shape:
        return np.inf
    return R.excess(got, ref, bnd)


# ---- the filter sets of the tests -------------------------------------------------------------------------------------
FB = np.array([1.0, 0.6, -0.3, 0.2, -0.1, 0.05, 0.3, -0.2, 0.1])      # feed-forward shape for nb = 1 .. 9
POLES = {"0": 0.0, "0.5": 0.5, "-0.5": -0.5, "0.947": 0.947, "0.948": 0.948, "-0.948": -0.948, "0.98": 0.98,
         "slow": 1 - 6.3e-5, "1-2^-20": 1 - 2.0 ** -20, "1": 1.0, "-1": -1.0}


def _gain(c):
    return max(1.0 - abs(c), 1e-3)


def scan_filters():
    """name -> (b, a) float32, every one an IirBlock (na <= 2, nb <= 9)"""
    out = {}
    for pn, c in POLES.items():
        for nb in ((1, 2, 3, 5, 9) if pn in ("0.5", "0.948", "slow") else (2,)):
            b = _gain(c) * FB[:nb] / np.sum(np.abs(FB[:nb]))
            out["p%s_nb%d" % (pn, nb)] = (b.astype(np.float32), np.float32([1.0, -c]))
    out["fir_nb5"] = ((FB[:5] / 2).astype(np.float32), np.float32([1.0]))
    out["deemph"] = tuple(np.asarray(v, np.float32) for v in _designs()["deemph"])
    out["lowpass10"] = tuple(np.asarray(v, np.float32) for v in _designs()["lowpass10"])
    out["highpass1k"] = tuple(np.asarray(v, np.float32) for v in _designs()["highpass1k"])
    # a0 = 4 and -1 keep the normalisation exact
    for a0 in (4.0, -1.0):
        for pn in ("0.5", "slow"):
            b, a = out["p%s_nb2" % pn]
            out["p%s_a0=%g" % (pn, a0)] = ((a0 * b.astype(np.float64)).astype(np.float32), (a0 * a.astype(np.float64)).astype(np.float32))
    return out


def inexact_filters():
    """a0 = 3 and 0.7: fl32(b / a0) and fl32(a / a0) are not the user's filter (see test_coefficient_term)"""
    out = {}
    base = scan_filters()
    for a0 in (3.0, 0.7):
        for pn in ("0.5", "slow"):
            b, a = base["p%s_nb2" % pn]
            out["p%s_a0=%g" % (pn, a0)] = ((a0 * b.astype(np.float64)).astype(np.float32), (a0 * a.astype(np.float64)).astype(np.float32))
        b, a = general_filters()["butter4_lowpass"]
        out["butter4_a0=%g" % a0] = ((a0 * b.astype(np.float64)).astype(np.float32), (a0 * a.astype(np.float64)).astype(np.float32))
    return out


def _designs():
    from oracle import lr_oracle as O
    return {"deemph": O.fm_deemphasis_taps(75e-6, 220500.0), "lowpass10": O.singlepole_lowpass_taps(10.0, 1e6),
            "highpass1k": O.singlepole_highpass_taps(1e3, 48e3)}


def _stable(a32):
    return bool(np.all(np.abs(np.roots(np.asarray(a32, np.float64))) < 1.0))


def resonator(r, w=0.05):
    a = np.array([1.0, -2 * r * np.cos(2 * np.pi * w), r * r, 0.0])
    return np.float32([0.5 * (1 - r), 0.0, -0.5 * (1 - r)]), a.astype(np.float32)


def general_filters():
    """name -> (b, a) float32, every one an IirGeneralBlock: low-pass and band-pass designs of order 2 .. 9 (na <= 10),
    a narrow one included, kept only where the float32 taps are stable; nb = 10 with na = 2; two resonators padded to
    na = 4, one whose W lands just under the 65536-sample limit and one that does not decay within it (W = -1).
    Left out: butter(3, 0.02), ellip(4, [0.3, 0.45]) and butter(4, [0.25, 0.28]) band-pass.  Their direct form in
    float32 amplifies rounding so much that the bound on uniform noise is 5e-2 .. 40 times the output's RMS: any
    direct-form evaluation in float32 is that far off, so no bound could tell a wrong kernel from a right one."""
    sg = scipy.signal
    out = {}
    designs = {
        "butter2_lowpass": sg.butter(2, 0.3), "butter4_lowpass": sg.butter(4, 0.2), "butter9_lowpass": sg.butter(9, 0.4),
        "cheby1_4_lowpass": sg.cheby1(4, 1.0, 0.2), "cheby1_6_lowpass": sg.cheby1(6, 1.0, 0.3),
        "ellip5_lowpass": sg.ellip(5, 1.0, 60.0, 0.3), "ellip2_narrow": sg.ellip(2, 1.0, 40.0, 0.02),
        "butter2_bandpass": sg.butter(2, [0.2, 0.4], "bandpass"), "cheby1_3_bandpass": sg.cheby1(3, 1.0, [0.3, 0.5], "bandpass"),
    }
    for name, (b, a) in designs.items():
        b32, a32 = np.float32(b), np.float32(a)
        if _stable(a32):
            out[name] = (b32, a32)
    out["fir10_pole"] = ((0.05 * np.concatenate([FB, [0.05]])).astype(np.float32), np.float32([1.0, -0.9]))
    out["resonator_w64k"] = resonator(RES_W64K)
    out["resonator_nodecay"] = resonator(1 - 1e-6)
    return out


# a pole radius whose W (warm_length) is just under 65536 (tests/test_iir_small_ref.py checks it)
RES_W64K = 0.99964


# mutants that cannot differ from the truth for a filter, and why
def scan_mutant_applies(mutant, b, a, n_tiles, D=1):
    bh, c = scan_coefs(b, a)
    local = is_local(c)
    if mutant == "xhist":
        return len(bh) > 1                              # no input history to drop
    if mutant == "ystate":
        return c != 0.0                                 # no feedback, no carried output
    if mutant == "phase":
        return D > 1
    if mutant == "a0":
        return float(np.float64(a[0])) != 1.0
    if mutant == "power":
        return c not in (0.0, 1.0)                      # every power of 0 (or of 1) is the same
    if mutant == "lookback":
        # LOCAL has no look-back; with |c^4096| below u32 a prefix and its aggregate differ by less than one rounding
        # of the carry (0.98^4096 = 1e-36; 0.948^4096 underflows to 0)
        return not local and abs(float(_f32(float(np.longdouble(c) ** 4096)))) > U32
    if mutant == "dead":
        # the raised cut-off kills a predecessor the true one keeps only if some weight cT^d of the stream's tiles lies in
        # [1e-12, 1e-6)
        if local:
            return False
        w = abs(float(np.longdouble(c) ** 4096))
        return any(1e-12 <= w ** d < 1e-6 for d in range(1, n_tiles))
    if mutant == "warm":
        # the halved warm-up differs only if the carried state survives 256 steps above float32's smallest subnormal
        if not local:
            return False
        gain = float(np.sum(np.abs(bh))) / max(1e-30, 1 - abs(c))
        return abs(c) ** 256 * gain >= 2.0 ** -149
    return True


def general_mutant_applies(mutant, b, a, n):
    m = GeneralModel(b, a, False)
    nb, na = len(m.b), len(m.a)
    if mutant in ("halfw", "decay", "first"):
        W = m.W
        if mutant == "decay":                            # the calls' chunking must change
            return m.plan(n) != GeneralModel(b, a, False, "decay").plan(n)
        return 0 <= W < n                                # one chunk from the carried state: no warm-up to shorten
    if mutant == "xhist":
        return nb > 1
    if mutant == "yrev":
        return na > 2                                    # one carried output reads the same either way
    return True
