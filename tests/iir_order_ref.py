"""A numpy model of iir_order.cu (IIRFilterBlock with 11..64 taps on either side) and the per-output error bound the GPU
outputs are held to.

Model: the kernel's decomposition in double, call by call -- FIR part u = (b / a0) * x; per thread V = 32 samples of the
recurrence from a zero state; per tile of P = 64 threads a serial chain of the thread end states with M^V (the tile's
aggregate); the kernel's fixed look-back walk (the aggregates of the LBW - 1 nearest predecessors weighted M^(T (d-1)),
the prefix of the tile LBW back or of tile 0); a second chain from the tile's carry gives each thread's incoming state
s_t; the outputs are yl[i] + hom[:, i] . s_t.  The tables are computed in extended precision and rounded once, as on the
host.

Bound, per output n, against the float64 recurrence y_ref (scipy lfilter):

    |y_gpu[n] - y_ref[n]| <= 2 u32 |y_ref[n]| + C u64 (E_alg[n] + E_ref[n]),     C = 2

u32 = 2^-24 covers the one rounding of each output to float32 (2 u32: the rounding of a value that is itself off by the
double-precision error).  E_alg is a running first-order rounding analysis of the model's own operations, with the
matrices and tables the kernel applies (u64 = 2^-53; a sum of m products is off by at most (m + 1) u64 times the sum of
the products' magnitudes, one more u64 for a coefficient or table entry rounded once; complex values are measured by
|re| + |im|):
  - an operation that produces a sample of the recurrence (the FIR sum, each zero-state step) injects an error that
    later outputs see through the impulse response h of 1/A: input-like, weight |h[n - t]|;
  - an operation that produces a state vector (each chain step with |M^V|, each look-back step with |M^(T d)|, the
    prefix with |M^T|, the carried last outputs of a call) injects an error eps_c in component c at state time t0; the
    zero-input response of unit state e_c is g_c[m] = -sum_(j>c) a_j h[m-j+c+1], so it acts as input-like errors
    sum_c eps_c |a_(c+1+k)| at t0 + k;
  - the final correction yl + hom . s (error bounded with |hom|) is added to its own output only.
E_alg = (|h| * injections) + direct terms.  E_ref bounds the reference's own sequential evaluation in the same way:
(nb + q + 3) u64 times the largest product-magnitude sum within the filter's length either side, through |h|.
C = 2 absorbs gamma_m = m u / (1 - m u) and the second-order products for m u << 1.  Nothing is fitted to observed
errors; `test_iir_order_ref.py::test_bound_is_tight` shows the double-precision term stays below 1e-6 of the signal
for every filter of the set.
"""
import numpy as np
import scipy.ndimage
import scipy.signal

P, V, LBW = 64, 32, 8
T = P * V
U32, U64 = 2.0 ** -24, 2.0 ** -53
C_BOUND = 2.0


def _norm(b, a, mutant=None):
    a64, b64 = np.asarray(a, np.float64), np.asarray(b, np.float64)
    a0 = 1.0 if mutant == "a0" else a64[0]
    return b64 / a0, -a64[1:] / a0


def homogeneous(cdiv, L):
    """g[c, m]: zero-input response from y[-1-c] = 1, in extended precision, rounded once."""
    q = len(cdiv)
    cl = cdiv.astype(np.longdouble)
    yv = np.zeros((q, q + L), np.longdouble)
    for c in range(q):
        yv[c, q - 1 - c] = 1
    for m in range(L):
        yv[:, q + m] = yv[:, m:q + m][:, ::-1] @ cl
    return yv[:, q:].astype(np.float64)


def power(g, k):
    """M^k in the state coordinates s = (y[-1], .., y[-q]): [r, c] = g_c[k-1-r] for k > r, else [c == r - k]."""
    q = g.shape[0]
    W = np.zeros((q, q))
    for r in range(q):
        if k > r:
            W[r, :] = g[:, k - 1 - r]
        elif 0 <= r - k < q:
            W[r, r - k] = 1.0
    return W


class OrderModel:
    """mutant: None, 'power' (M^(V+1) for M^V in the chains), 'lookback' (a predecessor's aggregate taken for its
    inclusive prefix), 'xhist' (input history dropped across calls), 'ystate32' (carried outputs rounded to float32),
    'a0' (a0 not divided out), 'hom' (homogeneous table shifted by one sample)."""

    def __init__(self, b, a, cplx, mutant=None):
        self.b, self.c = _norm(b, a, mutant)
        self.q, self.nb, self.cplx, self.mutant = len(self.c), len(self.b), cplx, mutant
        dt = np.complex128 if cplx else np.float64
        self.xh = np.zeros(self.nb - 1, dt)
        self.ys = np.zeros(self.q, dt)
        if self.q:
            g = homogeneous(self.c, T * (LBW - 1) + 2)
            self.MV = power(g, V + 1 if mutant == "power" else V)
            self.W = [power(g, T * e) for e in range(LBW)]
            self.hom = g[:, 1:V + 1] if mutant == "hom" else g[:, :V]      # hom[c, i] = g_c[i]

    def process(self, x):
        """The outputs of one call (double).  Also sets self.err_inj (per-sample rounding injections that propagate
        through h, see the module docstring) and self.err_direct (per-output injections that do not)."""
        x = np.asarray(x)
        n, q, nh, nb = len(x), self.q, self.nb - 1, self.nb
        dt = self.ys.dtype
        self.err_inj, self.err_direct = np.zeros(n), np.zeros(n)
        if n == 0:
            return np.zeros(0, dt)
        tiles = -(-n // T)
        xx = np.concatenate([self.xh, x.astype(dt), np.zeros(tiles * T - n, dt)])
        inj = np.zeros(tiles * T + q + 1)
        direct = np.zeros(tiles * T)
        ab, ac = np.abs(self.b), np.abs(self.c)
        u = np.zeros(tiles * T, dt)
        fir_m = np.zeros(tiles * T)
        for j in range(nb):
            u += self.b[j] * xx[nh - j:nh - j + tiles * T]
            fir_m += ab[j] * mag(xx[nh - j:nh - j + tiles * T])
        inj[:tiles * T] += (nb + 1) * fir_m
        yl = u.reshape(tiles * P, V).copy()
        rec_m = mag(u).reshape(tiles * P, V)
        for i in range(V):
            for j in range(1, min(i, q) + 1):
                rec_m[:, i] += ac[j - 1] * mag(yl[:, i - j])
                yl[:, i] += self.c[j - 1] * yl[:, i - j]
        inj[:tiles * T] += (q + 2) * rec_m.reshape(-1)
        if q == 0:
            y = yl.reshape(-1)[:n]
        else:
            # Acoef[c, k] = |a_(c+1+k)|: a state error eps_c at state time t0 acts as input errors sum_c eps_c Acoef[c, k]
            # at t0 + k (g_c[m] = -sum_(j>c) a_j h[m-j+c+1])
            Acoef = np.zeros((q, q))
            for c in range(q):
                Acoef[c, :q - c] = ac[c:]

            def state_err(eps, t0):                       # eps [.., q] at state times t0 [..]
                add = (eps.reshape(-1, q) @ Acoef)
                idx = np.asarray(t0).reshape(-1, 1) + np.arange(q)
                np.add.at(inj, idx.reshape(-1), add.reshape(-1))

            aMV, aW = np.abs(self.MV), [np.abs(w) for w in self.W]
            tb = np.arange(tiles) * T
            z = np.zeros((tiles, P, q), dt)
            k = min(q, V)
            z[:, :, :k] = yl.reshape(tiles, P, V)[:, :, ::-1][:, :, :k]
            e = np.zeros((tiles, q), dt)
            for t in range(P):
                state_err((q + 2) * (mag(z[:, t]) + mag(e) @ aMV.T), tb + (t + 1) * V)
                e = z[:, t] + e @ self.MV.T
            agg, pfx = e, np.zeros((tiles, q), dt)
            carry = np.zeros((tiles, q), dt)
            for t in range(tiles):
                if t == 0:
                    cin = self.ys.copy()
                else:
                    cin = np.zeros(q, dt)
                    lb_m = np.zeros(q)
                    dlast = min(t, LBW)
                    for d in range(1, dlast + 1):
                        v = pfx[t - d] if d == dlast and self.mutant != "lookback" else agg[t - d]
                        cin += self.W[d - 1] @ v
                        lb_m += aW[d - 1] @ mag(v)
                    state_err((dlast * q + 2) * lb_m, tb[t])
                carry[t] = cin
                pfx[t] = agg[t] + self.W[1] @ cin
                state_err((q + 2) * (mag(agg[t]) + aW[1] @ mag(cin)), tb[t] + T)
            s = np.zeros((tiles, P, q), dt)
            cur = carry
            for t in range(P):
                s[:, t] = cur
                state_err((q + 2) * (mag(z[:, t]) + mag(cur) @ aMV.T), tb + (t + 1) * V)
                cur = z[:, t] + cur @ self.MV.T
            y = (yl.reshape(tiles, P, V) + np.einsum("tpc,ci->tpi", s, self.hom)).reshape(-1)
            direct = (q + 2) * (mag(yl.reshape(-1)) + np.einsum("tpc,ci->tpi", mag(s), np.abs(self.hom)).reshape(-1))
            y = y[:n]
            ys = np.concatenate([y[::-1][:q], self.ys[:max(0, q - n)]])
            # the carried outputs' own errors reach the next call as a state error
            eps = np.concatenate([direct[:n][::-1][:q], np.zeros(max(0, q - n))])
            state_err(eps, n)
            self.ys = ys.astype(np.complex64 if self.cplx else np.float32).astype(dt) if self.mutant == "ystate32" else ys
        if self.mutant != "xhist":
            self.xh = np.concatenate([self.xh, x.astype(dt)])[len(self.xh) + n - nh:] if nh else self.xh
        self.err_inj, self.err_direct = inj[:n], direct[:n]
        return y


def mag(v):
    """|re| + |im| for complex values (bounds each component's and the modulus's error), |v| for real ones"""
    return np.abs(v.real) + np.abs(v.imag) if np.iscomplexobj(v) else np.abs(v)


def reference(b, a, xs):
    """float64 outputs of the recurrence over the calls xs (scipy lfilter with carried state)."""
    b64, a64 = np.asarray(b, np.float64), np.asarray(a, np.float64)
    x = np.concatenate([np.asarray(c) for c in xs]) if xs else np.zeros(0)
    if len(x) == 0:
        return x.astype(np.float64)
    return scipy.signal.lfilter(b64, a64, x.astype(np.complex128 if np.iscomplexobj(x) else np.float64))


def impulse(cn, N):
    """h of 1/A (taps normalised, cn[j-1] = -a_j / a0) over N samples"""
    imp = np.zeros(max(N, 1))
    imp[0] = 1.0
    return scipy.signal.lfilter([1.0], np.concatenate([[1.0], -np.asarray(cn)]), imp)


def _causal_conv(h, w):
    """(|h| * w)[:len(w)] for non-negative sequences, never below the exact value by more than FFT rounding"""
    if len(w) == 0:
        return w
    r = scipy.signal.fftconvolve(np.abs(h[:len(w)]), w)[:len(w)]
    return np.maximum(r, 0.0) * (1 + 1e-9) + 1e-12 * float(np.max(r))


def ref_error(bn, cn, x, ref, cplx, through):
    """E_ref in units of u64: the float64 reference's own rounding.  Per sample the products of bn with L inputs and of
    cn with L outputs (L the longer side), (nb + q + 3) times the largest such magnitude sum within L either side, taken
    through the filter's |h| by `through`."""
    N = len(x)
    L = max(len(bn), len(cn) + 1)
    tm = np.convolve(mag(np.asarray(x).astype(np.complex128 if cplx else np.float64)), np.abs(bn))[:N]
    if len(cn):
        tm += np.convolve(mag(np.concatenate([[0.0], ref[:-1]])), np.abs(cn))[:N]
    tw = scipy.ndimage.maximum_filter1d(tm, 2 * L - 1) if N else tm      # terms of the samples within L either side
    return through((len(bn) + len(cn) + 3) * tw)


def bound(b, a, xs, cplx):
    """(model outputs, float64 reference, per-output bound) of the stream of calls xs (see the module docstring)"""
    m = OrderModel(b, a, cplx)
    ys, inj, direct = [], [], []
    for x in xs:
        ys.append(m.process(x))
        inj.append(m.err_inj)
        direct.append(m.err_direct)
    y, inj, direct = np.concatenate(ys), np.concatenate(inj), np.concatenate(direct)
    ref = reference(b, a, xs)
    x = np.concatenate([np.asarray(v) for v in xs]) if xs else np.zeros(0)
    N = len(x)
    bn, cn = _norm(b, a)
    h = impulse(cn, N)
    e_ref = ref_error(bn, cn, x, ref, cplx, lambda w: _causal_conv(h, w))
    e_alg = _causal_conv(h, inj) + direct
    bnd = 2 * U32 * np.abs(ref) + C_BOUND * U64 * (e_alg + e_ref)
    return y, ref, bnd


def excess(got, ref, bnd):
    """max over n of |got - ref| / bound (<= 1 passes; an overflowing output counts as infinitely far off)"""
    if len(ref) == 0:
        return 0.0
    err = np.abs(np.asarray(got, np.complex128) - ref)
    err = np.where(np.isfinite(err), err, np.inf)
    return float(np.max(err / bnd))


# ---- the filter set of the GPU tests ----------------------------------------------------------------------------------
def _stable(a32):
    return bool(np.all(np.abs(np.roots(np.asarray(a32, np.float64))) < 1.0))


def filters():
    """name -> (b, a) in float32.  Every design is scaled by 2 so that a0 = 2 (exact in float32).  Kept only where the
    float32 feedback taps are stable (pole radii checked in float64) and where the direct form is well enough
    conditioned that the double-precision term of the bound stays below 1e-6 of the output on uniform noise
    (`test_iir_order_ref.py::test_bound_is_tight`): band designs centred on [0.3, 0.7] of Nyquist up to order 8
    (17 taps), low-pass designs up to 17 taps.  Wider or narrower bands, higher orders and longer low-pass designs
    either lose stability in float32 or amplify rounding beyond that in any direct-form evaluation, the reference's
    included."""
    sg = scipy.signal
    out = {}
    for order in (5, 6, 8):
        for kind, fn in (("butter", lambda o, w, bt: sg.butter(o, w, bt)),
                         ("cheby1", lambda o, w, bt: sg.cheby1(o, 1.0, w, bt)),
                         ("ellip", lambda o, w, bt: sg.ellip(o, 1.0, 60.0, w, bt))):
            for bt in ("bandpass", "bandstop"):
                b, a = fn(order, [0.3, 0.7], bt)
                b32, a32 = (2 * b).astype(np.float32), (2 * a).astype(np.float32)
                if _stable(a32):
                    out["%s%d_%s" % (kind, order, bt)] = (b32, a32)
    for name, (b, a) in (("butter10_lowpass", sg.butter(10, 0.6)), ("cheby2_10_lowpass", sg.cheby2(10, 60.0, 0.6)),
                         ("butter16_lowpass", sg.butter(16, 0.6))):
        b32, a32 = (2 * b).astype(np.float32), (2 * a).astype(np.float32)
        if _stable(a32):
            out[name] = (b32, a32)
    # nb = 1, na = 40: 39 poles, radii 0.6 .. 0.9, spread over the circle (one real pole)
    rr = np.linspace(0.6, 0.9, 19)
    th = np.pi * (np.arange(19) + 0.5) / 19
    poles = np.concatenate([rr * np.exp(1j * th), rr * np.exp(-1j * th), [0.8]])
    out["allpole40"] = (np.float32([2.0]), (2 * np.poly(poles).real).astype(np.float32))
    out["fir64"] = ((2 * sg.firwin(64, 0.3)).astype(np.float32), np.float32([2.0]))
    # a resonator with pole radius 1 - 1e-5, padded to 11 taps on both sides
    r, w = 1 - 1e-5, 2 * np.pi * 0.05
    res_a = np.concatenate([[1.0, -2 * r * np.cos(w), r * r], np.zeros(8)])
    out["resonator"] = ((2e-3 * 0.5 ** np.arange(11)).astype(np.float32), (2 * res_a).astype(np.float32))
    comb = np.zeros(33, np.float32)
    comb[0], comb[-1] = 2.0, -2.0
    out["comb33"] = (np.float32([2.0]), comb)
    return out


# mutants that cannot differ from the truth for a filter, and why
def mutant_applies(mutant, b, a):
    _, cn = _norm(b, a)
    q, nb = len(cn), len(b)
    if mutant == "xhist":
        return nb > 1                 # no input history to drop
    if mutant in ("power", "ystate32", "hom"):
        return q > 0                  # a pure FIR has no recurrence, carries or homogeneous response
    if mutant == "lookback":
        # the prefix LBW tiles back enters the carry through M^(T LBW); where every row of that power sums to less than
        # the double rounding unit, the aggregate differs from the prefix by less than one rounding of the state
        if q == 0:
            return False
        g = homogeneous(cn, T * LBW + 1)
        return float(np.max(np.sum(np.abs(power(g, T * LBW)), axis=1))) > U64
    return True
