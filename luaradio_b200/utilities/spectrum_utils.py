"""Power spectral density on the GPU.  Mirrors radio/utilities/spectrum_utils.lua:524-642 (class PSD): the engine of the
reference's spectrum sinks (gnuplotspectrum / gnuplotwaterfall call PSD:compute once per frame).

    psd = PSD(num_samples, complex_input, window_type="hamming", sample_rate=2, logarithmic=True)
    out = psd.compute(samples)          # any whole number of num_samples-frames -> as many PSD frames

window -> DFT -> |X_k|^2 / (sample_rate * window energy) [-> 10*log10], frames of a power of two from 2 to 2^20 points
(lrb200_psd_create): up to 16384 points one CTA per frame, longer frames in two passes through a device scratch buffer.
Other even lengths, which the reference accepts, raise.  fftshift() is the host-side reordering of
spectrum_utils.lua:646-667."""
import ctypes

import numpy as np

from .. import _lib
from . import window_utils


class PSD:
    def __init__(self, num_samples, complex_input=True, window_type=None, sample_rate=None, logarithmic=None):
        if num_samples % 2:
            raise ValueError("PSD length must be even.")
        self.num_samples = int(num_samples)
        self.window_type = window_type or "hamming"
        self.sample_rate = 2 if sample_rate is None else sample_rate
        self.logarithmic = True if logarithmic is None else bool(logarithmic)
        self.complex_input = bool(complex_input)
        # spectrum_utils.lua:545-551: periodic window as float32, energy summed from the float32 values
        self.window = np.array(window_utils.window(self.num_samples, self.window_type, True), np.float32)
        self.window_energy = float(np.sum(self.window.astype(np.float64) ** 2))
        lib = self._lib = _lib.require_device()
        scale = float(self.sample_rate) * self.window_energy
        self._handle = _lib.check_handle(lib.lrb200_psd_create(self.num_samples, self.window.ctypes.data, scale, 1 if self.logarithmic else 0,
                                                               1 if self.complex_input else 0, _lib.LRB200_HOST), "lrb200 psd object")

    def compute(self, samples):
        x = np.ascontiguousarray(samples, np.complex64 if self.complex_input else np.float32)
        if len(x) % self.num_samples:
            raise ValueError("PSD input must be a whole number of %d-sample frames." % self.num_samples)
        out = np.empty(len(x), np.float32)
        n_out = ctypes.c_size_t(0)
        _lib.check(self._lib.lrb200_block_execute(self._handle, x.ctypes.data, len(x), out.ctypes.data, ctypes.byref(n_out)), "psd")
        return out

    def close(self):
        if self._handle:
            self._lib.lrb200_block_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def fftshift(samples):
    """spectrum_utils.lua:646-667: swap the two halves (in a copy)."""
    x = np.asarray(samples)
    h = len(x) // 2
    return np.concatenate([x[h:], x[:h]])
