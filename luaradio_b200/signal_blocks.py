"""The hot-path signal blocks, same constructors / type signatures / process() contract as the
reference's radio/blocks/signal/*.lua, with process() executed by libluaradio_b200.so on the GPU.

Each block keeps the reference's structure: instantiate() registers type signatures,
initialize() designs taps from get_rate() and creates the native handle (the analogue of
`ffi.gc(libliquid.firfilt_crcf_create(...), destroy)`, firfilter.lua:186-202), process() hands the
input Vector's pointer to the library and returns the block-owned, reusable output Vector.
There is no non-GPU implementation: without the library/GPU, initialize() raises.
"""
import ctypes
import math

import numpy as np

from . import _lib
from .block import Block, Input, Output, factory
from .types import ComplexFloat32, Float32, Vector
from .utilities import filter_utils


class GPUBlock(Block):
    """Common process() for blocks backed by one lrb200 handle."""
    _handle = None

    def _make_handle(self, flags):
        raise NotImplementedError

    def initialize(self):
        lib = _lib.require_device()
        self._lib = lib
        self._handle = self._make_handle(_lib.LRB200_HOST)
        self.out = self.get_output_type().vector()

    def make_device_handle(self):
        """A second native handle in LRB200_DEVICE mode, for the GPU flow graph (ownership passes to the graph)."""
        _lib.require_device()
        return self._make_handle(_lib.LRB200_DEVICE)

    def process(self, x):
        lib = self._lib
        n = x.length
        out = self.out.resize(lib.lrb200_block_max_output(self._handle, n))
        n_out = ctypes.c_size_t(0)
        rc = lib.lrb200_block_execute(self._handle, x.ctypes_ptr(), n, out.ctypes_ptr(), ctypes.byref(n_out))
        if rc != 0:
            raise _lib.LibraryError("%s: %s" % (self.name, _lib.last_error()))
        return out.resize(n_out.value)

    def reset(self):
        if self._handle:
            _lib.check(self._lib.lrb200_block_reset(self._handle), "reset")

    def cleanup(self):
        if self._handle:
            self._lib.lrb200_block_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.cleanup()
        except Exception:
            pass


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def _c64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.complex64))


# ---------------------------------------------------------------------------------------------
# FIRFilterBlock and its design wrappers (firfilter.lua:43-82 and *filter.lua)
# ---------------------------------------------------------------------------------------------
class FIRFilterBlock(GPUBlock):
    name = "FIRFilterBlock"

    def instantiate(self, taps, use_fft=None):
        assert taps is not None, "Missing argument #1 (taps)"
        if isinstance(taps, Vector):
            self.taps = taps
        elif isinstance(taps, np.ndarray) and np.iscomplexobj(taps):
            self.taps = ComplexFloat32.vector_from_array(taps)
        elif isinstance(taps, (list, tuple, np.ndarray)):
            self.taps = Float32.vector_from_array(taps)
        else:
            raise TypeError("Unsupported taps type")
        # use_fft: True forces the fused overlap-save kernel, False the direct form, None = library choice.
        # (The GPU block is length-preserving in both cases, unlike the reference's chunked process_fft.)
        self.use_fft = use_fft
        if self.taps.data_type is ComplexFloat32:
            self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
        else:
            self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
            self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])

    def _make_handle(self, flags, decim=1):
        lib = _lib.load()
        cin = self.get_input_type() is ComplexFloat32
        t = self.taps
        if t.data_type is ComplexFloat32:
            h = lib.lrb200_fir_create_cccf(t.ctypes_ptr(), t.length, decim, flags)
        elif cin:
            h = lib.lrb200_fir_create_crcf(t.ctypes_ptr(), t.length, decim, flags)
        else:
            h = lib.lrb200_fir_create_rrrf(t.ctypes_ptr(), t.length, decim, flags)
        _lib.check_handle(h, "lrb200 fir object")
        if self.use_fft is not None:
            _lib.check(lib.lrb200_fir_set_algorithm(h, _lib.FIR_FFT if self.use_fft else _lib.FIR_DIRECT), "fir_set_algorithm")
        return h


class LowpassFilterBlock(FIRFilterBlock):
    name = "LowpassFilterBlock"

    def instantiate(self, num_taps, cutoff, nyquist=None, window=None):
        assert num_taps is not None, "Missing argument #1 (num_taps)"
        assert cutoff is not None, "Missing argument #2 (cutoff)"
        self.cutoff, self.window, self.nyquist = cutoff, window or "hamming", nyquist
        FIRFilterBlock.instantiate(self, Float32.vector(num_taps))

    def design(self, nyquist):
        return filter_utils.firwin_lowpass(self.taps.length, self.cutoff / nyquist, self.window)

    def initialize(self):
        nyquist = self.nyquist or (self.get_rate() / 2.0)
        self.taps = self.taps.data_type.vector_from_array(self.design(nyquist))
        FIRFilterBlock.initialize(self)


class HighpassFilterBlock(LowpassFilterBlock):
    name = "HighpassFilterBlock"

    def design(self, nyquist):
        return filter_utils.firwin_highpass(self.taps.length, self.cutoff / nyquist, self.window)


class BandpassFilterBlock(LowpassFilterBlock):
    name = "BandpassFilterBlock"

    def instantiate(self, num_taps, cutoffs, nyquist=None, window=None):
        assert num_taps is not None, "Missing argument #1 (num_taps)"
        assert cutoffs is not None, "Missing argument #2 (cutoffs)"
        self.cutoffs, self.window, self.nyquist = cutoffs, window or "hamming", nyquist
        FIRFilterBlock.instantiate(self, Float32.vector(num_taps))

    def design(self, nyquist):
        return filter_utils.firwin_bandpass(self.taps.length, [c / nyquist for c in self.cutoffs], self.window)


class BandstopFilterBlock(BandpassFilterBlock):
    name = "BandstopFilterBlock"

    def design(self, nyquist):
        return filter_utils.firwin_bandstop(self.taps.length, [c / nyquist for c in self.cutoffs], self.window)


class ComplexBandpassFilterBlock(BandpassFilterBlock):
    name = "ComplexBandpassFilterBlock"

    def instantiate(self, num_taps, cutoffs, nyquist=None, window=None):
        assert num_taps is not None, "Missing argument #1 (num_taps)"
        assert cutoffs is not None, "Missing argument #2 (cutoffs)"
        self.cutoffs, self.window, self.nyquist = cutoffs, window or "hamming", nyquist
        FIRFilterBlock.instantiate(self, ComplexFloat32.vector(num_taps))

    def design(self, nyquist):
        return filter_utils.firwin_complex_bandpass(self.taps.length, [c / nyquist for c in self.cutoffs], self.window)


class ComplexBandstopFilterBlock(ComplexBandpassFilterBlock):
    name = "ComplexBandstopFilterBlock"

    def design(self, nyquist):
        return filter_utils.firwin_complex_bandstop(self.taps.length, [c / nyquist for c in self.cutoffs], self.window)


# ---------------------------------------------------------------------------------------------
class HilbertTransformBlock(GPUBlock):
    """hilberttransform.lua:27-37."""
    name = "HilbertTransformBlock"

    def instantiate(self, num_taps, window=None):
        assert num_taps is not None, "Missing argument #1 (num_taps)"
        assert num_taps % 2 == 1, "Number of taps must be odd"
        taps = filter_utils.fir_hilbert_transform(num_taps, window or "hamming")
        self.hilbert_taps = Float32.vector_from_array(taps)
        self.add_type_signature([Input("in", Float32)], [Output("out", ComplexFloat32)])

    def _make_handle(self, flags):
        t = self.hilbert_taps
        return _lib.check_handle(_lib.load().lrb200_hilbert_create(t.ctypes_ptr(), t.length, flags), "lrb200 hilbert object")


class FrequencyTranslatorBlock(GPUBlock):
    """frequencytranslator.lua:26-31: y[n] = x[n] exp(j 2 pi (offset/rate) n)."""
    name = "FrequencyTranslatorBlock"

    def instantiate(self, offset):
        assert offset is not None, "Missing argument #1 (offset)"
        self.offset = offset
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])

    def _make_handle(self, flags):
        turns = float(self.offset) / float(self.get_rate())
        return _lib.check_handle(_lib.load().lrb200_rotator_create(turns, flags), "lrb200 rotator object")


class FrequencyDiscriminatorBlock(GPUBlock):
    """frequencydiscriminator.lua:25-38."""
    name = "FrequencyDiscriminatorBlock"

    def instantiate(self, modulation_index):
        assert modulation_index is not None, "Missing argument #1 (modulation_index)"
        self.gain = 2 * math.pi * modulation_index
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", Float32)])

    def _make_handle(self, flags):
        return _lib.check_handle(_lib.load().lrb200_discrim_create(self.gain, flags), "lrb200 discriminator object")


class DownsamplerBlock(GPUBlock):
    """downsampler.lua:29-56."""
    name = "DownsamplerBlock"

    def instantiate(self, factor):
        assert factor is not None, "Missing argument #1 (factor)"
        self.factor = int(factor)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
        self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])

    def get_rate(self):
        return Block.get_rate(self) / self.factor

    def _make_handle(self, flags):
        return _lib.check_handle(_lib.load().lrb200_downsample_create(self.factor, self.get_input_type().size, flags),
                                 "lrb200 downsampler object")


class IIRFilterBlock(GPUBlock):
    """iirfilter.lua:39-61."""
    name = "IIRFilterBlock"

    def instantiate(self, b_taps, a_taps):
        assert b_taps is not None, "Missing argument #1 (b_taps)"
        assert a_taps is not None, "Missing argument #2 (a_taps)"
        self.b_taps = b_taps if isinstance(b_taps, Vector) else Float32.vector_from_array(b_taps)
        self.a_taps = a_taps if isinstance(a_taps, Vector) else Float32.vector_from_array(a_taps)
        assert self.a_taps.length >= 1, "Feedback taps must be at least length 1"
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
        self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])

    def _make_handle(self, flags):
        lib = _lib.load()
        fn = lib.lrb200_iir_create_crcf if self.get_input_type() is ComplexFloat32 else lib.lrb200_iir_create_rrrf
        return _lib.check_handle(fn(self.b_taps.ctypes_ptr(), self.b_taps.length, self.a_taps.ctypes_ptr(), self.a_taps.length, flags),
                                 "lrb200 iir object")


class SinglepoleLowpassFilterBlock(IIRFilterBlock):
    """singlepolelowpassfilter.lua:29-67."""
    name = "SinglepoleLowpassFilterBlock"

    def instantiate(self, cutoff):
        assert cutoff is not None, "Missing argument #1 (cutoff)"
        self.cutoff = cutoff
        IIRFilterBlock.instantiate(self, Float32.vector(2), Float32.vector(2))

    def _design(self, rate):
        tau = 1.0 / (2 * math.pi * self.cutoff)
        tau = 1.0 / (2 * rate * math.tan(1.0 / (2 * rate * tau)))
        b = [1 / (1 + 2 * tau * rate), 1 / (1 + 2 * tau * rate)]
        a = [1.0, (1 - 2 * tau * rate) / (1 + 2 * tau * rate)]
        return b, a

    def initialize(self):
        b, a = self._design(self.get_rate())
        self.b_taps = Float32.vector_from_array(b)
        self.a_taps = Float32.vector_from_array(a)
        IIRFilterBlock.initialize(self)

    def make_device_handle(self):
        b, a = self._design(self.get_rate())
        self.b_taps = Float32.vector_from_array(b)
        self.a_taps = Float32.vector_from_array(a)
        return IIRFilterBlock.make_device_handle(self)


class SinglepoleHighpassFilterBlock(SinglepoleLowpassFilterBlock):
    name = "SinglepoleHighpassFilterBlock"

    def _design(self, rate):
        tau = 1.0 / (2 * math.pi * self.cutoff)
        tau = 1.0 / (2 * rate * math.tan(1.0 / (2 * rate * tau)))
        b = [(2 * tau * rate) / (1 + 2 * tau * rate), -(2 * tau * rate) / (1 + 2 * tau * rate)]
        a = [1.0, (1 - 2 * tau * rate) / (1 + 2 * tau * rate)]
        return b, a


class FMDeemphasisFilterBlock(SinglepoleLowpassFilterBlock):
    """fmdeemphasisfilter.lua:24-27."""
    name = "FMDeemphasisFilterBlock"

    def instantiate(self, tau):
        assert tau is not None, "Missing argument #1 (tau)"
        SinglepoleLowpassFilterBlock.instantiate(self, 1.0 / (2 * math.pi * tau))


class ComplexMagnitudeBlock(GPUBlock):
    """complexmagnitude.lua:28-36."""
    name = "ComplexMagnitudeBlock"

    def instantiate(self):
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", Float32)])

    def _make_handle(self, flags):
        return _lib.check_handle(_lib.load().lrb200_cmag_create(flags), "lrb200 cmag object")


class ComplexToRealBlock(GPUBlock):
    """complextoreal.lua:27-35."""
    name = "ComplexToRealBlock"

    def instantiate(self):
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", Float32)])

    def _make_handle(self, flags):
        return _lib.check_handle(_lib.load().lrb200_c2r_create(flags), "lrb200 c2r object")


# ---------------------------------------------------------------------------------------------
# Resampling family (SURVEY 8f row 4)
# ---------------------------------------------------------------------------------------------
class MultiplyConstantBlock(GPUBlock):
    """multiplyconstant.lua: y = x * constant; a complex constant only accepts complex input."""
    name = "MultiplyConstantBlock"

    def instantiate(self, constant):
        assert constant is not None, "Missing argument #1 (constant)"
        if isinstance(constant, (complex, np.complexfloating)):
            self.constant, self.complex_constant = complex(constant), True
            self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
        elif isinstance(constant, (int, float, np.integer, np.floating)):
            self.constant, self.complex_constant = float(constant), False
            self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])
            self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
        else:
            raise TypeError("Unsupported constant type")

    def _make_handle(self, flags):
        c = complex(self.constant)
        cdata = 1 if self.get_input_type() is ComplexFloat32 else 0
        return _lib.check_handle(_lib.load().lrb200_mulconst_create(c.real, c.imag, cdata, 1 if self.complex_constant else 0, flags),
                                 "lrb200 mulconst object")


class UpsamplerBlock(GPUBlock):
    """upsampler.lua:29-52: y[i*L] = x[i], zeros in between; rate * L."""
    name = "UpsamplerBlock"

    def instantiate(self, factor):
        assert factor is not None, "Missing argument #1 (factor)"
        self.factor = int(factor)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
        self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])

    def get_rate(self):
        return Block.get_rate(self) * self.factor

    def _make_handle(self, flags):
        return _lib.check_handle(_lib.load().lrb200_upsample_create(self.factor, self.get_input_type().size, flags),
                                 "lrb200 upsampler object")


# ---------------------------------------------------------------------------------------------
# Blocks the WBFM-stereo / AM-synchronous chains add to the hot path (SURVEY 8f row 3)
# ---------------------------------------------------------------------------------------------
class GPUMultiBlock(GPUBlock):
    """A GPU block with several input and/or output ports: process(x1, x2, ...) -> (y1, y2, ...) through
    lrb200_block_execute_multi.  All inputs have the same length (block.lua:516-532)."""
    out_types = None              # data types of the output ports (default: the signature's)

    def initialize(self):
        lib = _lib.require_device()
        self._lib = lib
        self._handle = self._make_handle(_lib.LRB200_HOST)
        self.outs = [self.get_output_type(i + 1).vector() for i in range(len(self.outputs))]

    def process(self, *xs):
        lib, n = self._lib, xs[0].length
        cap = lib.lrb200_block_max_output(self._handle, n)
        for o in self.outs:
            o.resize(cap)
        ins = (ctypes.c_void_p * len(xs))(*[x.ctypes_ptr() for x in xs])
        outs = (ctypes.c_void_p * len(self.outs))(*[o.ctypes_ptr() for o in self.outs])
        n_out = ctypes.c_size_t(0)
        rc = lib.lrb200_block_execute_multi(self._handle, ins, len(xs), n, outs, len(self.outs), ctypes.byref(n_out))
        if rc != 0:
            raise _lib.LibraryError("%s: %s" % (self.name, _lib.last_error()))
        res = tuple(o.resize(n_out.value) for o in self.outs)
        return res[0] if len(res) == 1 else res


class _BinaryBlock(GPUMultiBlock):
    op = None
    real_too = True

    def instantiate(self):
        self.add_type_signature([Input("in1", ComplexFloat32), Input("in2", ComplexFloat32)], [Output("out", ComplexFloat32)])
        if self.real_too:
            self.add_type_signature([Input("in1", Float32), Input("in2", Float32)], [Output("out", Float32)])

    def _make_handle(self, flags):
        cplx = 1 if self.get_input_type() is ComplexFloat32 else 0
        return _lib.check_handle(_lib.load().lrb200_binary_create(self.op.encode(), cplx, flags), "lrb200 %s object" % self.op)


class MultiplyBlock(_BinaryBlock):
    """multiply.lua:26-60: out = in1 * in2 (complex or real)."""
    name, op = "MultiplyBlock", "multiply"


class MultiplyConjugateBlock(_BinaryBlock):
    """multiplyconjugate.lua:26-51: out = in1 * conj(in2)."""
    name, op, real_too = "MultiplyConjugateBlock", "multiplyconjugate", False


class AddBlock(_BinaryBlock):
    """add.lua:23-60: out = in1 + in2."""
    name, op = "AddBlock", "add"


class SubtractBlock(_BinaryBlock):
    """subtract.lua:23-60: out = in1 - in2."""
    name, op = "SubtractBlock", "subtract"


class DelayBlock(GPUBlock):
    """delay.lua:26-60: out[n] = in[n - num_samples], zeros first (ComplexFloat32 / Float32)."""
    name = "DelayBlock"

    def instantiate(self, num_samples):
        assert num_samples is not None, "Missing argument #1 (num_samples)"
        assert num_samples > 0, "Number of samples must be greater than 0"
        self.num_samples = int(num_samples)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
        self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])

    def _make_handle(self, flags):
        return _lib.check_handle(_lib.load().lrb200_delay_create(self.num_samples, self.get_input_type().size, flags), "lrb200 delay object")


class PLLBlock(GPUMultiBlock):
    """pll.lua:27-170: in -> out (exp(j * multiplied phase)), error (phase detector output)."""
    name = "PLLBlock"

    # True: chunk-parallel form for long vectors (lrb200_pll_set_mode(h, 1)); every chunk whose speculated start misses the
    # carried loop state is run again in order, so it agrees with the sequential form on any input, locked or not
    parallel = False

    def instantiate(self, loop_bandwidth, frequency_min, frequency_max, multiplier=None):
        assert loop_bandwidth is not None, "Missing argument #1 (loop_bandwidth)"
        assert frequency_min is not None, "Missing argument #2 (frequency_min)"
        assert frequency_max is not None, "Missing argument #3 (frequency_max)"
        self.loop_bw, self.freq_min, self.freq_max = float(loop_bandwidth), float(frequency_min), float(frequency_max)
        self.multiplier = 1.0 if multiplier is None else float(multiplier)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32), Output("error", Float32)])

    def _make_handle(self, flags):
        lib = _lib.load()
        h = _lib.check_handle(lib.lrb200_pll_create(self.loop_bw, self.freq_min, self.freq_max, self.multiplier, self.get_rate(), flags),
                              "lrb200 pll object")
        if self.parallel:
            _lib.check(lib.lrb200_pll_set_mode(h, 1), "pll_set_mode")
        return h


# ---------------------------------------------------------------------------------------------
# Level control (the reference's "Level Control" category)
# ---------------------------------------------------------------------------------------------
class AGCBlock(GPUBlock):
    """agc.lua:41-115: feed-forward automatic gain control towards `target` dBFS, gated by `threshold` dBFS.
    gain_tau is 0.1 s ("fast"), 3.0 s ("slow") or options["gain_tau"] ("custom"); power_tau is options["power_tau"] or
    1.0 s."""
    name = "AGCBlock"

    def instantiate(self, mode=None, target=None, threshold=None, options=None):
        assert mode is not None, 'Missing argument #1 (mode), can be "fast", "slow", or "custom"'
        self.mode = mode
        self.target = -35 if target is None else target
        self.threshold = -75 if threshold is None else threshold
        self.options = options or {}
        gain_tau = {"fast": 0.1, "slow": 3.0}.get(mode) if isinstance(mode, str) else None
        self.gain_tau = gain_tau if gain_tau is not None else self.options.get("gain_tau")
        power_tau = self.options.get("power_tau")
        self.power_tau = 1.0 if power_tau is None else power_tau
        assert mode in ("fast", "slow", "custom"), 'Invalid mode "%s"' % (mode,)
        assert self.gain_tau is not None, 'Missing gain_tau parameter for "custom" mode'
        self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])

    def _make_handle(self, flags):
        cdata = 1 if self.get_input_type() is ComplexFloat32 else 0
        return _lib.check_handle(_lib.load().lrb200_agc_create(float(self.target), float(self.threshold), float(self.gain_tau),
                                                               float(self.power_tau), float(self.get_rate()), cdata, flags),
                                 "lrb200 agc object")


class PowerSquelchBlock(GPUBlock):
    """powersquelch.lua:24-75: y = x while the average power is at least `threshold` dBFS, else 0.

    The power estimator's time constant is always 0.001 s: the reference's instantiate assigns `tau or 0.001` from an
    undefined global `tau` (powersquelch.lua:26), so its second argument is accepted and ignored.  This block does the
    same, because the reference's outputs are the contract."""
    name = "PowerSquelchBlock"

    def instantiate(self, threshold=None, cutoff=None):
        assert threshold is not None, "Missing argument #1 (threshold)"
        self.threshold = threshold
        self.tau = 0.001
        self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])

    def _make_handle(self, flags):
        cdata = 1 if self.get_input_type() is ComplexFloat32 else 0
        return _lib.check_handle(_lib.load().lrb200_powersquelch_create(float(self.threshold), float(self.tau), float(self.get_rate()),
                                                                        cdata, flags),
                                 "lrb200 powersquelch object")


# ---------------------------------------------------------------------------------------------
# Digital: the RDS / BPSK31 front ends up to clock recovery
# ---------------------------------------------------------------------------------------------
class RootRaisedCosineFilterBlock(FIRFilterBlock):
    """rootraisedcosinefilter.lua:29-45: an FIR filter with root raised cosine taps (filter_utils.fir_root_raised_cosine),
    designed in initialize() from get_rate()."""
    name = "RootRaisedCosineFilterBlock"

    def instantiate(self, num_taps, beta=None, symbol_rate=None):
        assert num_taps is not None, "Missing argument #1 (num_taps)"
        assert beta is not None, "Missing argument #2 (beta)"
        assert symbol_rate is not None, "Missing argument #3 (symbol_rate)"
        self.beta, self.symbol_rate = beta, symbol_rate
        FIRFilterBlock.instantiate(self, Float32.vector(num_taps))

    def initialize(self):
        taps = filter_utils.fir_root_raised_cosine(self.taps.length, self.get_rate(), self.beta, 1 / self.symbol_rate)
        self.taps = Float32.vector_from_array(taps)
        FIRFilterBlock.initialize(self)


class ManchesterMatchedFilterBlock(FIRFilterBlock):
    """manchestermatchedfilter.lua:27-51: an FIR filter matched to a Manchester-coded symbol, floor(rate / baudrate) taps of
    -1 then as many of +1 (both signs flipped with `invert`), designed in initialize() from get_rate().  Its output peaks
    positive at 1 -> 0 transitions and negative at 0 -> 1 transitions."""
    name = "ManchesterMatchedFilterBlock"

    def instantiate(self, baudrate, invert=False):
        assert baudrate is not None, "Missing argument #1 (baudrate)"
        self.baudrate, self.invert = baudrate, bool(invert)
        self.taps, self.use_fft = Float32.vector(32), None          # designed in initialize()
        self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])

    @staticmethod
    def design(rate, baudrate, invert):
        """The taps: the reference's `for i=1, symbol_period` loop runs floor(symbol_period) times."""
        period = int(math.floor(rate / baudrate))
        assert period >= 1, "Sample rate %g is below the baud rate %g" % (rate, baudrate)
        sign = -1.0 if invert else 1.0
        return np.concatenate([np.full(period, -sign), np.full(period, sign)]).astype(np.float32)

    def initialize(self):
        self.taps = Float32.vector_from_array(self.design(self.get_rate(), self.baudrate, self.invert))
        FIRFilterBlock.initialize(self)


class BinaryPhaseCorrectorBlock(GPUBlock):
    """binaryphasecorrector.lua:28-77: rotates a BPSK signal against the moving average of its phase, folded into
    (-pi/2, pi/2], measured every `sample_interval` samples over the last `num_samples` measurements."""
    name = "BinaryPhaseCorrectorBlock"

    def instantiate(self, num_samples=None, sample_interval=None):
        assert num_samples is not None, "Missing argument #1 (num_samples)"
        self.num_samples = num_samples
        self.sample_interval = 32 if sample_interval is None else sample_interval
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])

    def _make_handle(self, flags):
        return _lib.check_handle(_lib.load().lrb200_phasecorrector_create(int(self.num_samples), int(self.sample_interval), flags),
                                 "lrb200 phasecorrector object")
