---
-- The digital front-end blocks (radio/blocks/signal/binaryphasecorrector.lua) on the GPU: the b200.install() below is
-- the `if platform.features.cuda then` branch for that file.  Apply with
-- require('radio_b200.digital_patch')(require('radio')), as radio_b200/init.lua does after blocks_patch.lua.
--
-- RootRaisedCosineFilterBlock needs nothing here: it is a FIRFilterBlock that designs its taps in initialize()
-- (rootraisedcosinefilter.lua:38-44) and then calls FIRFilterBlock.initialize, which firfilter_patch.lua gives its GPU form.

local platform = require('radio.core.platform')
local types = require('radio.types')
local b200 = require('radio_b200.platform')

return function (radio)
    if not platform.features.cuda then return end
    local lib = platform.libs.cuda

    -- radio/blocks/signal/binaryphasecorrector.lua:28-77 (num_samples, sample_interval from instantiate)
    b200.install(radio.BinaryPhaseCorrectorBlock, "phasecorrector", function (self, flags)
        return lib.lrb200_phasecorrector_create(self.num_samples, self.sample_interval, flags)
    end, function () return types.ComplexFloat32 end)
    radio.BinaryPhaseCorrectorBlock.process = b200.process
end
