---
-- The remaining hot-path blocks: each b200.install() below is the `if platform.features.cuda then` branch for
-- the file named in its comment.  Apply with  require('radio_b200.blocks_patch')(require('radio')).
-- Every block gets initialize() (HOST-pointer handle for its own process()) and make_device_handle() (the same
-- create call with DEVICE pointers, used by the scheduler in composite_patch.lua).

local ffi = require('ffi')
local platform = require('radio.core.platform')
local types = require('radio.types')
local b200 = require('radio_b200.platform')

return function (radio)
    if not platform.features.cuda then return end
    local lib = platform.libs.cuda
    local function in_type(self) return self:get_input_type() end
    local function complex_out() return types.ComplexFloat32 end
    local function real_out() return types.Float32 end
    local function elem_size(self) return self:get_input_type() == types.ComplexFloat32 and 8 or 4 end

    require('radio_b200.firfilter_patch')(radio.FIRFilterBlock)

    -- radio/blocks/signal/frequencytranslator.lua:32 (before the volk branch)
    b200.install(radio.FrequencyTranslatorBlock, "rotator", function (self, flags)
        return lib.lrb200_rotator_create(self.offset / self:get_rate(), flags)
    end, complex_out)
    radio.FrequencyTranslatorBlock.process = b200.process

    -- radio/blocks/signal/frequencydiscriminator.lua:33-40
    b200.install(radio.FrequencyDiscriminatorBlock, "discriminator", function (self, flags)
        return lib.lrb200_discrim_create(self.gain, flags)
    end, real_out)
    radio.FrequencyDiscriminatorBlock.process = b200.process

    -- radio/blocks/signal/downsampler.lua:40-56
    b200.install(radio.DownsamplerBlock, "downsampler", function (self, flags)
        return lib.lrb200_downsample_create(self.factor, elem_size(self), flags)
    end, in_type)
    radio.DownsamplerBlock.process = b200.process

    -- radio/blocks/signal/iirfilter.lua:63 (before the liquid branch); Singlepole*/FMDeemphasis inherit it
    b200.install(radio.IIRFilterBlock, "iir", function (self, flags)
        local create = self:get_input_type() == types.ComplexFloat32 and lib.lrb200_iir_create_crcf or lib.lrb200_iir_create_rrrf
        return create(self.b_taps.data, self.b_taps.length, self.a_taps.data, self.a_taps.length, flags)
    end, in_type)
    radio.IIRFilterBlock.process_complex = b200.process
    radio.IIRFilterBlock.process_real = b200.process

    -- radio/blocks/signal/hilberttransform.lua:39
    b200.install(radio.HilbertTransformBlock, "hilbert", function (self, flags)
        return lib.lrb200_hilbert_create(self.hilbert_taps.data, self.hilbert_taps.length, flags)
    end, complex_out)
    radio.HilbertTransformBlock.process = b200.process

    -- radio/blocks/signal/complexmagnitude.lua:24-36, complextoreal.lua:23-35
    b200.install(radio.ComplexMagnitudeBlock, "cmag", function (self, flags) return lib.lrb200_cmag_create(flags) end, real_out)
    radio.ComplexMagnitudeBlock.process = b200.process
    b200.install(radio.ComplexToRealBlock, "c2r", function (self, flags) return lib.lrb200_c2r_create(flags) end, real_out)
    radio.ComplexToRealBlock.process = b200.process

    -- radio/blocks/signal/upsampler.lua:36-52 and multiplyconstant.lua:44-70 (resampling family, SURVEY 8f row 4).
    -- InterpolatorBlock / RationalResamplerBlock stay the composites they are; in a GPU sub-graph the three or four
    -- handles are committed to one polyphase kernel (composite_patch.lua -> lrb200_graph_commit).
    b200.install(radio.UpsamplerBlock, "upsampler", function (self, flags)
        return lib.lrb200_upsample_create(self.factor, elem_size(self), flags)
    end, in_type)
    radio.UpsamplerBlock.process = b200.process
    b200.install(radio.MultiplyConstantBlock, "mulconst", function (self, flags)
        local cplx_data = self:get_input_type() == types.ComplexFloat32
        local c = self.constant
        local cplx_const = ffi.istype(types.ComplexFloat32, c)
        return lib.lrb200_mulconst_create(cplx_const and c.real or c.value, cplx_const and c.imag or 0,
                                          cplx_data and 1 or 0, cplx_const and 1 or 0, flags)
    end, function (self) return self:get_output_type() end)
    radio.MultiplyConstantBlock.process = b200.process
    radio.MultiplyConstantBlock.process_complex_by_real = b200.process

    -- Two-input element-wise blocks, DelayBlock and PLLBlock (SURVEY 8f row 3: the WBFM stereo / AM synchronous chains).
    -- multiply.lua:27-28 registers process_complex / process_real per signature; add.lua:32, subtract.lua:32 and
    -- multiplyconjugate.lua:41,51 define a plain process().
    local function same_type_out(self) return {self:get_output_type()} end
    for name, op in pairs({MultiplyBlock = "multiply", MultiplyConjugateBlock = "multiplyconjugate", AddBlock = "add", SubtractBlock = "subtract"}) do
        b200.install_multi(radio[name], op, function (self, flags)
            return lib.lrb200_binary_create(op, self:get_input_type() == types.ComplexFloat32 and 1 or 0, flags)
        end, same_type_out)
        radio[name].process = b200.process_multi
    end
    radio.MultiplyBlock.process_complex = b200.process_multi
    radio.MultiplyBlock.process_real = b200.process_multi
    -- radio/blocks/signal/delay.lua:26-60 (ComplexFloat32 / Float32; the Bit and Byte signatures keep the Lua loop)
    local delay_initialize, delay_process = radio.DelayBlock.initialize, radio.DelayBlock.process
    b200.install(radio.DelayBlock, "delay", function (self, flags)
        return lib.lrb200_delay_create(self.num_samples, elem_size(self), flags)
    end, in_type)
    local gpu_delay_initialize = radio.DelayBlock.initialize
    local function float_delay(self)
        local t = self:get_input_type()
        return t == types.ComplexFloat32 or t == types.Float32
    end
    function radio.DelayBlock:initialize()
        self.on_gpu = float_delay(self)
        if self.on_gpu then return gpu_delay_initialize(self) end
        return delay_initialize(self)
    end
    function radio.DelayBlock:process(x)
        if self.on_gpu then return b200.process(self, x) end
        return delay_process(self, x)
    end
    function radio.DelayBlock:gpu_capable() return float_delay(self) end      -- the scheduler leaves a Bit / Byte delay line on the host
    -- radio/blocks/signal/pll.lua:113-170: loop constants are derived in the library from the Hz arguments (the reference's
    -- initialize() overwrites self.loop_bw / freq_min / freq_max with rad/sample; this initialize() leaves them in Hz)
    b200.install_multi(radio.PLLBlock, "pll", function (self, flags)
        return lib.lrb200_pll_create(self.loop_bw, self.freq_min, self.freq_max, self.multiplier, self:get_rate(), flags)
    end, function () return {types.ComplexFloat32, types.Float32} end)
    radio.PLLBlock.process = b200.process_multi

    -- File sample formats (SURVEY 8f row 1).  Sources keep their fread(); the swap + (value - offset)/scale loop of
    -- radio/blocks/sources/iqfile.lua:96-108 / realfile.lua:86-104 becomes one call on the raw chunk.
    local function source_process(create, what)
        return function (self)
            local n = tonumber(ffi.C.fread(self.raw_samples.data, ffi.sizeof(self.raw_samples.data_type), self.raw_samples.length, self.file))
            if n == 0 then
                if ffi.C.feof(self.file) ~= 0 and self.repeat_on_eof then ffi.C.rewind(self.file) else return nil end
            end
            self.handle = self.handle or b200.own(create(self.format_name, b200.HOST), what)
            local out, n_out = self.out:resize(n), ffi.new("size_t[1]")
            if lib.lrb200_block_execute(self.handle, self.raw_samples.data, n, out.data, n_out) ~= 0 then
                b200.fail(what)
            end
            return out
        end
    end
    radio.IQFileSource.process = source_process(lib.lrb200_iqconv_create, "iqconv")
    radio.RealFileSource.process = source_process(lib.lrb200_realconv_create, "realconv")
    -- a source read by a device DAG alone is absorbed into it: the converter is the DAG's first node (composite_patch.lua)
    local function converter(self, create, what)
        local h = create(self.format_name, b200.DEVICE)
        if h == nil then b200.fail("Creating lrb200 " .. what .. " object") end
        return h
    end
    function radio.IQFileSource:make_converter_handle() return converter(self, lib.lrb200_iqconv_create, "iqconv") end
    function radio.RealFileSource:make_converter_handle() return converter(self, lib.lrb200_realconv_create, "realconv") end
    -- Sinks (radio/blocks/sinks/iqfile.lua:66-88, realfile.lua, wavfile.lua:170-194 for one channel): convert, then fwrite.
    local function sink_process(create, what)
        return function (self, x)
            self.handle = self.handle or b200.own(create(self.format_name, b200.HOST), what)
            self.raw_samples:resize(x.length)
            local n_out = ffi.new("size_t[1]")
            if lib.lrb200_block_execute(self.handle, x.data, x.length, self.raw_samples.data, n_out) ~= 0 then
                b200.fail(what)
            end
            if ffi.C.fwrite(self.raw_samples.data, ffi.sizeof(self.raw_samples.data_type), x.length, self.file) ~= x.length then
                error("fwrite(): " .. ffi.string(ffi.C.strerror(ffi.errno())))
            end
            self.count = (self.count or 0) + x.length           -- WAVFileSink:cleanup() fills the header sizes from it
        end
    end
    radio.IQFileSink.process = sink_process(lib.lrb200_iqsink_create, "iqsink")
    radio.RealFileSink.process = sink_process(lib.lrb200_realsink_create, "realsink")
    -- format_name: the reference's instantiate() keeps only the format TABLE (sources/iqfile.lua:48); the library wants the
    -- format's name, so each constructor is wrapped to remember it (second argument in all four signatures)
    for _, class in ipairs({radio.IQFileSource, radio.RealFileSource, radio.IQFileSink, radio.RealFileSink}) do
        local instantiate = class.instantiate
        class.instantiate = function (self, file, format, ...)
            self.format_name = format
            return instantiate(self, file, format, ...)
        end
    end

    -- the scheduler: connected GPU blocks share one device-resident flow graph (composite_patch.lua)
    require('radio_b200.composite_patch').install(radio)
end
