---
-- Level control (radio/blocks/signal/agc.lua, powersquelch.lua) on the GPU: each b200.install() below is the
-- `if platform.features.cuda then` branch for the file named in its comment.  Apply with
-- require('radio_b200.level_patch')(require('radio')), as radio_b200/init.lua does after blocks_patch.lua.
--
-- install() replaces the reference's initialize(), which would overwrite self.target / self.threshold with linear values
-- (agc.lua:65-67, powersquelch.lua:38): they stay in dBFS here, and the library linearises them and derives the alphas
-- from the time constants and the rate, in the reference's expression order (as for the PLL in blocks_patch.lua).

local platform = require('radio.core.platform')
local types = require('radio.types')
local b200 = require('radio_b200.platform')

return function (radio)
    if not platform.features.cuda then return end
    local lib = platform.libs.cuda
    local function in_type(self) return self:get_input_type() end
    local function complex_flag(self) return self:get_input_type() == types.ComplexFloat32 and 1 or 0 end

    -- radio/blocks/signal/agc.lua:57-115
    b200.install(radio.AGCBlock, "agc", function (self, flags)
        return lib.lrb200_agc_create(self.target, self.threshold, self.gain_tau, self.power_tau, self:get_rate(),
                                     complex_flag(self), flags)
    end, in_type)
    radio.AGCBlock.process_real = b200.process
    radio.AGCBlock.process_complex = b200.process

    -- radio/blocks/signal/powersquelch.lua:32-75 (self.tau is always 0.001: powersquelch.lua:26 reads an undefined global)
    b200.install(radio.PowerSquelchBlock, "powersquelch", function (self, flags)
        return lib.lrb200_powersquelch_create(self.threshold, self.tau, self:get_rate(), complex_flag(self), flags)
    end, in_type)
    radio.PowerSquelchBlock.process_real = b200.process
    radio.PowerSquelchBlock.process_complex = b200.process
end
