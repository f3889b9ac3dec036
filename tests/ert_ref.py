"""Reference model for the ERT receiver's signal path (composites/ertreceiver.lua:38-43):

  * `manchester_matched_filter`: the oracle of ManchesterMatchedFilterBlock (manchestermatchedfilter.lua:36-51), the
    oracle FIR with floor(rate / baudrate) taps of -1 then as many of +1 (the Lua loop `for i=1, symbol_period` runs
    floor(symbol_period) times), both signs flipped with `invert`;
  * `MagFirModel` / `MagCase`: the overlap-save kernel's fused-magnitude mode (fir_fft.cu IN = 3, the stage graph.cu
    fuse_magnitude_fir makes): complex input, |x| at the load, then the packed-real geometry of the rrrf mode.  The fused
    stage runs the overlap-save kernel on every call whatever its FIR's algorithm (FirBlock::path: no other kernel has the
    magnitude prologue), so its geometry is the rrrf mode's with the FFT forced;
  * `MAG_REL`: the float32 magnitude's relative rounding, the one term the fused stage adds to the rrrf bound of
    tests/fft_fir_ref.py."""
import numpy as np

from oracle import lr_oracle as O
from tests import fft_fir_ref as F

# |x| = sqrt(fl(fl(im^2) + re^2)) then a correctly rounded square root: the radicand carries gamma_2, its root half of that,
# and the root's own rounding one u (Higham Lemma 3.1 and 3.3)
MAG_REL = F.gamma(2) / 2 + F.U


def manchester_taps(baudrate, rate, invert=False):
    period = int(np.floor(rate / baudrate))
    assert period >= 1, "Sample rate %g is below the baud rate %g" % (rate, baudrate)
    h = np.array([-1.0] * period + [1.0] * period)
    return O.f32_taps(-h if invert else h)


def manchester_matched_filter(baudrate, rate, invert=False):
    return O.FIRFilter(manchester_taps(baudrate, rate, invert), False)


class MagFirModel(F.FirModel):
    """FirBlock's choices for the fused stage: M real taps, decimation D (M <= 513: the single-block plan)."""

    def __init__(self, M, D):
        F.FirModel.__init__(self, "rrrf", M, D, algo="fft")
        self.kind, self.poly, self.gen_poly = "mag", False, False
        assert self.fast and self.nparts == 1, "the fused magnitude needs the single-block overlap-save plan (M <= 513)"


class MagCase(F.Case):
    """One fused stage (taps h, decimation D) and its streams; the input is complex, the output real."""

    def __init__(self, name, h, D, streams=(), sig="noise", seed=0):
        F.Case.__init__(self, name, "rrrf", h, D, None, "fft", streams, sig, seed)
        self.model = MagFirModel(self.M, D)
        self.cplx_in = True
        self.burst = F.burst_length(self.model)

    def full(self, x, n0, h=None, turns=0):
        return F.Case.full(self, np.abs(np.asarray(x).astype(np.complex128)), n0, h, turns)

    def expect(self, x, n0, calls):
        """tests/fft_fir_ref.py Case.expect over |x|, plus the magnitude's rounding: MAG_REL sum_k |h_k| |x_(o-k)|."""
        ref, bound, callno, k = F.Case.expect(self, x, n0, calls)
        ax = np.abs(np.asarray(x).astype(np.complex128))
        S = np.maximum(F.fir_ref(np.abs(self.h.astype(np.float64)), ax, wide=True), 0.0)
        return ref, bound + MAG_REL * S[k], callno, k
