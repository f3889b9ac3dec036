"""Numpy model of the compute phase of the interior tuner+discriminator kernel (tuner.cu: polyphase_crcf_kernel<5, 26,
ROT, DISC> on the bulk-copy path), which runs the polyphase FIR in two-parallel fast-FIR form.

It mirrors the kernel's indexing: the host's reversed taps with the alignment spare (hr, T = Q*D + 1 entries) and the
float32 sum taps hs; tiles of TS = PT_TO - DISC_OV - DISC_TAIL outputs, whose first DISC_OV slots overlap the previous
tile and whose last DISC_TAIL slots are not stored; thread t of a tile reading blocks u_j = X[B + (t*R + j)*D .. +D); the
A_k, B_k (k < R/2) and S_k sub-filters over V_i = u_2i+1 + u_2i+2; the last pair's A_{R/2} taken from the next thread's
A_0 (the tile's last thread gets its own A_0, as lane 31's shuffle does, and that output is not stored); and the spare tap
added as output r is formed at block Q + r.  Every accumulator is a float32 FMA chain in the kernel's order (blocks
ascending, then taps), or exact in float64."""
import numpy as np

D, Q, R, THREADS, DISC_OV, DISC_TAIL = 5, 26, 8, 64, 4, 4
TO = THREADS * R                    # outputs per tile
TS = TO - DISC_OV - DISC_TAIL       # tile stride
T = Q * D + 1


def host_taps(h, shift):
    """launch_shape: hr'[i] = hr_base[i - shift] with hr_base[i] = h[Q*D-1-i]; hs[q*D+p] = hr'[2qD+p] + hr'[(2q+1)D+p]."""
    hr_base = np.zeros(Q * D, np.float32)
    for i in range(Q * D):
        k = Q * D - 1 - i
        if k < len(h):
            hr_base[i] = h[k]
    hr = np.zeros(T, np.float32)
    hr[shift:shift + Q * D] = hr_base[:T - shift]
    hs = np.array([hr[2 * q * D + p] + hr[(2 * q + 1) * D + p] for q in range(Q // 2) for p in range(D)], np.float32)
    return hr, hs


def _fma(acc, h, x, exact):
    if exact:
        return acc + np.float64(h) * x
    # float32 FMA on each lane: the product of two float32 values is exact in float64, the sum is rounded once more
    a = acc.astype(np.complex128) + np.float64(h) * x.astype(np.complex128)
    return a.astype(np.complex64)


def _add(a, b, exact):
    return a + b if exact else (a.astype(np.complex64) + b.astype(np.complex64)).astype(np.complex64)


def _sub(a, b, exact):
    return a - b if exact else (a.astype(np.complex64) - b.astype(np.complex64)).astype(np.complex64)


def tile_outputs(Xt, hr, hs, exact):
    """Xt: [tiles, LOADED] rotated samples of each tile.  Returns the TO filter outputs of every tile, slot order."""
    dt = np.complex128 if exact else np.complex64
    Xt = Xt.astype(dt)
    nt = Xt.shape[0]
    KP, QH = R // 2, Q // 2
    zero = np.zeros((nt, THREADS), dt)
    fa = [zero.copy() for _ in range(KP)]
    an = None
    fb = [zero.copy() for _ in range(KP)]
    fs = [zero.copy() for _ in range(KP)]
    acc = [None] * R
    uo = None
    base = np.arange(THREADS) * R * D
    hq = hr[Q * D]
    for j in range(R + Q):
        xs = [Xt[:, base + j * D + p] for p in range(D if j < R + Q - 1 else 1)]
        if j == R + Q - 1:
            pass
        elif j % 2 == 0:
            i = j // 2
            for k in range(KP):
                q = i - k
                if 0 <= q < QH:
                    for p in range(D):
                        fa[k] = _fma(fa[k], hr[2 * q * D + p], xs[p], exact)
            if 1 <= i and i - 1 <= KP - 1 + QH - 1:
                v = [_add(uo[p], xs[p], exact) for p in range(D)]
                for k in range(KP):
                    q = i - 1 - k
                    if 0 <= q < QH:
                        for p in range(D):
                            fs[k] = _fma(fs[k], hs[q * D + p], v[p], exact)
        else:
            i = (j - 1) // 2
            for k in range(KP):
                q = i - k
                if 0 <= q < QH:
                    for p in range(D):
                        fb[k] = _fma(fb[k], hr[(2 * q + 1) * D + p], xs[p], exact)
            uo = xs
        if j == 2 * QH - 1:
            # the next thread's A_0; the last thread keeps its own (shuffle down from lane 31)
            an = np.concatenate([fa[0][:, 1:], fa[0][:, -1:]], axis=1)
        if j >= Q:
            r = j - Q
            k = r // 2
            if r % 2 == 0:
                acc[r] = _fma(_add(fa[k], fb[k], exact), hq, xs[0], exact)
            else:
                a1 = fa[k + 1] if k + 1 < KP else an
                acc[r] = _fma(_sub(_sub(fs[k], a1, exact), fb[k], exact), hq, xs[0], exact)
    # slot s = t*R + r
    return np.stack(acc, axis=-1).reshape(nt, TO)


def direct_outputs(Xt, hr):
    """Direct form in float64: y[slot s] = sum_{i' < T} hr[i'] X[B + s*D + i']."""
    Xt = Xt.astype(np.complex128)
    s = np.arange(TO)
    return sum(np.float64(hr[i]) * Xt[:, s * D + i] for i in range(T))


def stream(xr, h, first, tiles, exact):
    """The filter outputs y[m], m = DISC_OV-th slot of tile 0 onward, of a rotated stream xr (zero before index 0)
    through `tiles` tiles, as the launcher lays them out (off, shift, tile stride TS), by the model and by direct form."""
    off = first - DISC_OV * D - (Q * D - 1)
    shift = off % 2
    off -= shift
    hr, hs = host_taps(h, shift)
    if exact:
        # the algebra alone: the sum taps unrounded (the kernel's float32 hs is part of its float32 error)
        hs = np.array([np.float64(hr[2 * q * D + p]) + hr[(2 * q + 1) * D + p] for q in range(Q // 2) for p in range(D)])
    span = (TO - 1) * D + T
    lead = max(0, -off)
    xp = np.concatenate([np.zeros(lead, xr.dtype), xr, np.zeros(span, xr.dtype)])
    B = off + np.arange(tiles) * TS * D + lead
    Xt = np.stack([xp[b:b + span] for b in B])
    got = tile_outputs(Xt, hr, hs, exact)[:, DISC_OV:TO - DISC_TAIL].reshape(-1)
    ref = direct_outputs(Xt, hr)[:, DISC_OV:TO - DISC_TAIL].reshape(-1)
    return got, ref
