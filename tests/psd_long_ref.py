"""Float32 model, per-bin error bound and deliberately wrong variants ("mutants") of the long-frame PSD kernels
(psd_long.cu), frames of 8192 <= N <= 2^20 points.

Decomposition.  Every transform is a Stockham autosort FFT of length L = 16^k * rem (rem in 1, 2, 4, 8; radix-16
passes first, the remainder last).  A pass of radix R over the span Ns (1, R0, R0 R1, ...) takes, for each j < L / R,
the R inputs a[j + r L/R], multiplies input r by W_L^((j mod Ns) r L / (Ns R)), runs an R-point DFT and writes output q
to b[(j div Ns) Ns R + (j mod Ns) + q Ns]; the last pass leaves the DFT in natural order.

  * N <= 16384: one CTA per frame, the whole frame is one such transform (psd_long_single_kernel).
  * N >= 32768: N = N1 N2 with N2 = 2^ceil(log2(N) / 2).  Pass 1 (psd_long_col_kernel) transforms the N2 columns
    x[n1 N2 + n2] over n1 and writes Y[k1, n2] W_N^(n2 k1) to a scratch buffer; the twiddle is the product of two
    float32 table entries, W_N^(m mod 1024) W_N^(1024 (m div 1024)).  Pass 2 (psd_long_row_kernel) transforms the rows
    Y[k1, :] over n2 and stores X[k1 + N1 k2].  A CTA holds a tile of TILE = 8192 points: TILE / N1 adjacent columns
    in pass 1, TILE / N2 adjacent rows in pass 2.  A call is cut into batches of BATCH_SAMPLES / N frames, so that the
    scratch buffer stays at 256 MiB.

The window is applied where the kernels load x, |X|^2 / scale (and 10 log10 of it) is computed in double from the
float32 X and rounded once.  Real input is carried as complex with a zero imaginary part.

Per-bin bound.  With u = 2^-24 and xw the windowed frame,

    delta_k = C_BOUND u log2(N) (N^(1/4) ||xw||_2 + |X_k|)

bounds the error of the computed X_k, and then

    |P^_k - P_k| <= (2 |X_k| delta_k + delta_k^2) / scale + ulp(P_k)

and in dB the same interval, converted, on the bins where P_k exceeds the linear bound; bins at or below it need only
be finite or -inf (the reference's 10 log10(0)).  The FFT's error is normwise (Higham, Accuracy and Stability of
Numerical Algorithms, 2nd ed., Thm 24.2: ||X^ - X||_2 <= c u log2(N) ||X||_2, ||X||_2 = sqrt(N) ||xw||_2).  On noise
it spreads over all N bins, u log2(N) ||xw||_2 each; a strong tone does not spread it so far: its rounding errors after
the first sub-transforms reach only the bins of one row, about sqrt(N) of them, hence N^(1/4) ||xw||_2, and the tone's
own bin carries a relative error of a few u per stage, hence |X_k|.  C_BOUND is taken from this model:
tests/test_psd_long_ref.py shows that the model stays within half of it for every N, with noise, tones and a tone
60 dB below another, while each mutant breaks it."""
import math

import numpy as np

U = 2.0 ** -24
C_BOUND = 4.0
SINGLE_MAX = 16384
TILE = 8192
BATCH_SAMPLES = 1 << 25            # 256 MiB of complex64 scratch
MAX_N = 1 << 20
LONG_SIZES = [1 << m for m in range(13, 21)]


def radices(L):
    out = []
    while L >= 16:
        out.append(16)
        L //= 16
    if L > 1:
        out.append(L)
    return out


def split(N):
    """(N1, N2): column length and row length of the two-pass form."""
    m = N.bit_length() - 1
    N2 = 1 << ((m + 1) // 2)
    return N // N2, N2


def batch_frames(N):
    return max(1, BATCH_SAMPLES // N)


def twiddles(L):
    """W_L^m, m < L, computed in double and rounded to float32 (as PsdLongPlan does on the host)."""
    m = np.arange(L, dtype=np.float64)
    return (np.cos(2 * np.pi * m / L) - 1j * np.sin(2 * np.pi * m / L)).astype(np.complex64)


def _dft_matrix(R):
    q, r = np.meshgrid(np.arange(R), np.arange(R), indexing="ij")
    return np.exp(-2j * np.pi * (q * r) / R).astype(np.complex64)


def stockham(a, mutant=None):
    """Float32 Stockham FFT over axis 1 of a (batch, L, S) complex64 array; returns a new array."""
    B, L, S = a.shape
    tw = twiddles(L)
    Ns = 1
    for p, R in enumerate(radices(L)):
        v = a.reshape(B, R, L // R, S)
        j = np.arange(L // R)
        k = j % Ns
        e = (k[None, :] * np.arange(R)[:, None]) * (L // (Ns * R))
        w = tw[e]
        if mutant == "twiddle_sign" and p == 1:
            w = np.conj(w)
        v = v * w[None, :, :, None]
        out = np.einsum("qr,brjs->bqjs", _dft_matrix(R), v).astype(np.complex64)
        b = np.empty_like(a)
        dst = ((j // Ns) * Ns * R + k)[None, :] + np.arange(R)[:, None] * Ns
        b[:, dst, :] = out
        a = b
        Ns *= R
    return a


def _epilogue(X, scale, logarithmic, mutant):
    if mutant == "scale":
        scale = scale * 2.0
    p = (X.real.astype(np.float64) ** 2 + X.imag.astype(np.float64) ** 2) * (1.0 / scale)
    if logarithmic:
        with np.errstate(divide="ignore"):
            p = 10.0 * np.log10(p)
    return p.astype(np.float32)


def _windowed(x, w, N, mutant):
    """Frames of x times the window, as complex64 (batch, N); the 'window' mutant leaves one tile's share out."""
    F = len(x) // N
    xf = np.asarray(x).reshape(F, N)
    ww = np.broadcast_to(w, (F, N)).copy()
    if mutant == "window":
        if N <= SINGLE_MAX:
            ww[:, N // 4:N // 2] = 1.0                 # one quarter of the CTA's threads
        else:
            N1, N2 = split(N)
            C1 = TILE // N1
            ww.reshape(F, N1, N2)[:, :, C1:2 * C1] = 1.0  # the second column tile of pass 1
    if np.iscomplexobj(xf):
        return (xf * ww).astype(np.complex64)
    return (xf * ww).astype(np.float32).astype(np.complex64)


def model_psd(x, window, scale, logarithmic, mutant=None):
    """The kernels' decomposition on whole frames of x (complex64 or float32) in float32 arithmetic."""
    w = np.asarray(window, np.float32)
    N = len(w)
    assert SINGLE_MAX < N <= MAX_N or N in (8192, 16384)
    x = np.asarray(x)
    F = len(x) // N
    if N <= SINGLE_MAX:
        X = stockham(_windowed(x, w, N, mutant)[:, :, None], mutant)[:, :, 0]
        return _epilogue(X, scale, logarithmic, mutant).reshape(-1)
    N1, N2 = split(N)
    C2 = TILE // N2
    lo = twiddles(N)[:1024]
    hi = twiddles(N)[::1024]
    out = np.empty(F * N, np.float32)
    BF = batch_frames(N)
    for f0 in range(0, F, BF):
        f1 = min(F, f0 + BF)
        xw = _windowed(x[f0 * N:f1 * N], w, N, mutant).reshape(f1 - f0, N1, N2)
        Y = stockham(xw, mutant)                                       # (batch, k1, n2)
        m = np.arange(N1)[:, None] * np.arange(N2)[None, :]            # k1 n2 < N
        Y = (Y * (lo[m % 1024] * hi[m // 1024])[None]).astype(np.complex64)
        Z = stockham(np.ascontiguousarray(np.swapaxes(Y, 1, 2)))       # (batch, k2, k1): rows transformed over n2
        if mutant == "transpose" and f0 == 0:
            g = 1                                                      # the second row tile stores one k2 too far
            Z[:, :, g * C2:(g + 1) * C2] = np.roll(Z[:, :, g * C2:(g + 1) * C2], 1, axis=1)
        X = Z.reshape(f1 - f0, N)                                      # X[k1 + N1 k2] = Z[k2, k1]
        out[f0 * N:f1 * N] = _epilogue(X, scale, logarithmic, mutant).reshape(-1)
    return out


# ---- the per-bin bound -------------------------------------------------------------------------------------------------
def _frames64(x, window):
    N = len(window)
    xf = np.asarray(x).reshape(-1, N)
    w = np.asarray(window, np.float32).astype(np.float64)
    if np.iscomplexobj(xf):
        xw = (xf.astype(np.complex128) * w).astype(np.complex64)
    else:
        xw = (xf.astype(np.float64) * w).astype(np.float32)
    return xw.astype(np.complex128)


def linear_tolerance(x, window, scale, ref_lin, c=C_BOUND):
    """Per-bin tolerance of the linear PSD, from the reference P_k (float32, as oracle.psd returns it)."""
    N = len(window)
    xw = _frames64(x, window)
    norm = np.sqrt(np.sum(np.abs(xw) ** 2, axis=1))                    # ||x w||_2 per frame
    P = np.asarray(ref_lin, np.float32).reshape(-1, N)
    absX = np.sqrt(P.astype(np.float64) * scale)
    d = c * U * math.log2(N) * (N ** 0.25 * norm[:, None] + absX)
    return ((2 * absX * d + d * d) / scale + np.spacing(np.abs(P)).astype(np.float64)).reshape(-1)


def check(got, x, window, scale, ref_lin, ref_log=None, logarithmic=False, c=C_BOUND, what=""):
    """Raises AssertionError when a bin of `got` is outside the bound; returns the worst |err| / tol."""
    got = np.asarray(got)
    P = np.asarray(ref_lin, np.float32).astype(np.float64)
    tol = linear_tolerance(x, window, scale, ref_lin, c)
    assert got.shape == P.shape, "%s: length %s != %s" % (what, got.shape, P.shape)
    if not logarithmic:
        err = np.abs(got.astype(np.float64) - P)
        bad = np.flatnonzero(~(err <= tol))
        assert not bad.size, "%s: bin %d: |%.9g - %.9g| > %.3g (%d bins)" % (what, bad[0], got[bad[0]], P[bad[0]], tol[bad[0]], bad.size)
        return float(np.max(err / np.maximum(tol, 1e-300))) if err.size else 0.0
    L = np.asarray(ref_log, np.float32).astype(np.float64)
    g = got.astype(np.float64)
    above = P > tol
    hi = 10 * np.log10((P[above] + tol[above]) / P[above])
    lo = -10 * np.log10(np.maximum(P[above] - tol[above], 1e-300) / P[above])
    # dB values are float32: the reference's rounding and the kernel's, a few ulp of the dB value
    slack = 4 * np.spacing(np.abs(L[above]).astype(np.float32)).astype(np.float64)
    d = g[above] - L[above]
    ok = (d <= hi + slack) & (-d <= lo + slack)
    bad = np.flatnonzero(~ok)
    assert not bad.size, "%s: dB bin %d: %.9g vs %.9g (%d bins)" % (what, np.flatnonzero(above)[bad[0]], g[above][bad[0]],
                                                                      L[above][bad[0]], bad.size)
    low = g[~above]
    assert np.all(np.isfinite(low) | (low == -np.inf)), "%s: NaN or +inf below the bound" % what
    return float(np.max(np.abs(d) / (np.maximum(hi, lo) + slack))) if d.size else 0.0
