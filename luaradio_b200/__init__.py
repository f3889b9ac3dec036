"""luaradio_b200: the H100 (sm_90a) implementation of LuaRadio's sample-stream DSP hot path.

The namespace mirrors the reference's `radio` module (radio/init.lua:16-50) for the blocks on the hot
path, so a flow graph reads the same:

    import luaradio_b200 as radio
    top = radio.CompositeBlock()
    top.connect(source, radio.TunerBlock(-250e3, 200e3, 5), radio.FrequencyDiscriminatorBlock(1.25),
                radio.LowpassFilterBlock(128, 15e3), radio.FMDeemphasisFilterBlock(75e-6),
                radio.DownsamplerBlock(5), sink)
    top.run()

All arithmetic runs in libluaradio_b200.so (hand-written CUDA, include/lrb200.h); there is no CPU path.
"""
from . import _lib, block, types
from .block import Block, Input, Output, factory
from .composite import (AMEnvelopeDemodulator, ArraySink, ArraySource, CompositeBlock, DecimatorBlock, InterpolatorBlock,
                        IQFileSink, IQFileSource, NBFMDemodulator, RationalResamplerBlock, RawFileSink, RawFileSource,
                        RealFileSink, RealFileSource, SSBDemodulator, TunerBlock, WAVFileSink, WBFMMonoDemodulator,
                        WBFMStereoDemodulator, AMSynchronousDemodulator, GPUChainBlock)
from .signal_blocks import (MultiplyConstantBlock, UpsamplerBlock, BandpassFilterBlock, BandstopFilterBlock, ComplexBandpassFilterBlock,
                            ComplexBandstopFilterBlock, ComplexMagnitudeBlock, ComplexToRealBlock,
                            DownsamplerBlock, FIRFilterBlock, FMDeemphasisFilterBlock,
                            FrequencyDiscriminatorBlock, FrequencyTranslatorBlock, GPUBlock,
                            HighpassFilterBlock, HilbertTransformBlock, IIRFilterBlock, LowpassFilterBlock,
                            SinglepoleHighpassFilterBlock, SinglepoleLowpassFilterBlock,
                            MultiplyBlock, MultiplyConjugateBlock, AddBlock, SubtractBlock, DelayBlock, PLLBlock, GPUMultiBlock,
                            AGCBlock, PowerSquelchBlock, RootRaisedCosineFilterBlock, BinaryPhaseCorrectorBlock,
                            ManchesterMatchedFilterBlock)
from .types import ComplexFloat32, Float32, Vector
from .utilities import filter_utils, spectrum_utils, window_utils

__version__ = "0.1.0"
