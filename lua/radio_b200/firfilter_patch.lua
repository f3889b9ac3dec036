---
-- FIRFilterBlock on the H100: the extra branch a maintainer adds at the TOP of the backend ladder in
-- radio/blocks/signal/firfilter.lua (:88 `if platform.features.volk then`), mechanically identical to
-- the liquid branch (:165-226).  Lowpass/Highpass/Bandpass/Bandstop/ComplexBandpass/ComplexBandstop, RootRaisedCosine
-- and ManchesterMatchedFilter inherit it unchanged because they only design taps and call FIRFilterBlock.initialize.
--
--   if platform.features.cuda then  <this file's body>  elseif platform.features.volk then ...

local platform = require('radio.core.platform')
local types = require('radio.types')
local b200 = require('radio_b200.platform')

return function (FIRFilterBlock)
    if not platform.features.cuda then return end
    local lib = platform.libs.cuda

    b200.install(FIRFilterBlock, "fir", function (self, flags)
        local data_type = self:get_input_type()
        local h
        if data_type == types.ComplexFloat32 and self.taps.data_type == types.Float32 then
            h = lib.lrb200_fir_create_crcf(self.taps.data, self.taps.length, 1, flags)
        elseif data_type == types.Float32 and self.taps.data_type == types.Float32 then
            h = lib.lrb200_fir_create_rrrf(self.taps.data, self.taps.length, 1, flags)
        else
            h = lib.lrb200_fir_create_cccf(self.taps.data, self.taps.length, 1, flags)
        end
        -- FIRFilterBlock(taps, use_fft): true -> fused overlap-save, false -> direct form, nil -> automatic
        if h ~= nil and self.use_fft ~= nil then
            lib.lrb200_fir_set_algorithm(h, self.use_fft and b200.FIR_FFT or b200.FIR_DIRECT)
        end
        return h
    end, function (self) return self:get_input_type() end)

    -- length-preserving for every algorithm (the GPU block never delays/chunks like process_fft)
    FIRFilterBlock.process_complex_input_complex_taps = b200.process
    FIRFilterBlock.process_complex_input_real_taps = b200.process
    FIRFilterBlock.process_real_input_real_taps = b200.process
    FIRFilterBlock.process_fft_complex_input_complex_taps = b200.process
    FIRFilterBlock.process_fft_complex_input_real_taps = b200.process
    FIRFilterBlock.process_fft_real_input_real_taps = b200.process
end
