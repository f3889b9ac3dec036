---
-- Entry point of the H100 backend:
--
--   local radio = require('radio')
--   require('radio_b200')(radio)      -- before any block is created
--
-- Probes libluaradio_b200.so (radio_b200/platform.lua), gives the hot-path block classes their GPU form
-- (radio_b200/blocks_patch.lua, firfilter_patch.lua, level_patch.lua, digital_patch.lua) and installs the scheduler
-- (radio_b200/composite_patch.lua).
-- Without a CUDA device, or with LUARADIO_DISABLE_CUDA=1, nothing is patched and the stock backends run.
-- Returns true when the CUDA backend is active.

local platform = require('radio.core.platform')

return function (radio)
    require('radio_b200.blocks_patch')(radio)
    require('radio_b200.level_patch')(radio)
    require('radio_b200.digital_patch')(radio)
    return platform.features.cuda == true
end
