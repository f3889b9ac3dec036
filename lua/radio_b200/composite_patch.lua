---
-- GPU scheduler hook for radio/core/composite.lua.  A CUDA context does not survive fork(), and
-- _initialize() runs in the parent before the fork loop (composite.lua:443 then :568-636), so when the CUDA
-- backend is active the top block runs through the single-process path (composite.lua:647-707) and every
-- MAXIMAL LINEAR RUN of GPU blocks in the crawled connection graph is collapsed into ONE lrb200 flow graph:
-- one process() call per source vector, device-resident intermediates, fused kernels, H2D/D2H only at the
-- two ends of the run.  Before that, every connected NON-linear set of GPU blocks with a single outside feed (the WBFM
-- stereo demodulator: two-input blocks, the PLL's two outputs, fan-outs), and every group of sets that share one outside
-- feed (several receivers on one source), becomes ONE device DAG (GPUDagBlock, lrb200_dag_*), with the raw file source
-- that feeds it alone absorbed as its first node.
-- CPU blocks, and multi-input blocks or fan-out points outside such a set, stay ordinary blocks at the edges.
--
--   local top = radio.CompositeBlock(); top:connect(...); top:run()   -- unchanged user code
--
-- install(radio) wraps five methods of CompositeBlock:
--   _crawl_connections (composite.lua:343-381)  the top-level call returns the flat input-port -> output-port map;
--                                               GPU sub-graphs are substituted there, before _connect_pipes (:383-393)
--   _connect_pipes (composite.lua:383-393)      members of a sub-graph get a rate-only link in place of their pipe
--   _initialize (composite.lua:416-424)         initialises the substitutes after the original blocks
--   _prepare_to_run (composite.lua:426-466)     hands the global evaluation order to the substitutes (EOF flush)
--   start (composite.lua:534-545)               forces multiprocess = false
-- Set LUARADIO_B200_SUPERCHUNK=<samples> to pack the per-vector calls into pinned super-chunks
-- (lrb200_graph_set_superchunk, lrb200_dag_set_superchunk): throughput of the reference's 8192-sample vectors goes from launch-bound to
-- memcpy-bound; outputs then arrive in bursts, and the last partial super-chunk is only pushed out by cleanup().

local ffi = require('ffi')
local platform = require('radio.core.platform')
local block = require('radio.core.block')
local b200 = require('radio_b200.platform')

--- A block that stands for a run of connected GPU blocks [first .. last].
local GPUChainBlock = block.factory("GPUChainBlock")

function GPUChainBlock:instantiate(blocks, edges)
    self.blocks = blocks
    self.edges = edges or {}                 -- member input port -> the output port that fed it in the crawled graph
    self:add_type_signature({block.Input("in", blocks[1]:get_input_type())},
                            {block.Output("out", blocks[#blocks]:get_output_type())})
end

function GPUChainBlock:get_rate()
    return self.blocks[#self.blocks]:get_rate()
end

function GPUChainBlock:initialize()
    local lib = platform.libs.cuda
    self.graph = ffi.gc(lib.lrb200_graph_create(), lib.lrb200_graph_destroy)
    if self.graph == nil then b200.fail("graph_create") end
    for _, b in ipairs(self.blocks) do
        -- make_device_handle(): the block's own create call with DEVICE pointers (radio_b200/platform.lua install)
        local h = b:make_device_handle()
        if lib.lrb200_graph_append(self.graph, h) ~= 0 then b200.fail("graph_append") end
    end
    if lib.lrb200_graph_commit(self.graph, 1) ~= 0 then b200.fail("graph_commit") end
    local sc = tonumber(os.getenv('LUARADIO_B200_SUPERCHUNK') or 0)
    if sc > 0 and lib.lrb200_graph_set_superchunk(self.graph, sc) ~= 0 then b200.fail("graph_set_superchunk") end
    self.out = self:get_output_type().vector()
end

local n_out = ffi.new("size_t[1]")
function GPUChainBlock:process(x)
    local lib = platform.libs.cuda
    local out = self.out:resize(tonumber(lib.lrb200_graph_max_output(self.graph, x.length)))
    if lib.lrb200_graph_execute(self.graph, x.data, x.length, out.data, n_out) ~= 0 then b200.fail("graph_execute") end
    return out:resize(tonumber(n_out[0]))
end

--- Hand flushed super-chunk outputs (outs[k] for output port k) to the downstream pipes before they are closed.
local function hand_on_flushed(self, outs)
    local any = false
    for k, out in ipairs(outs) do
        if out.length > 0 then
            any = true
            for _, p in ipairs(self.outputs[k].pipes) do p:write(out) end
        end
    end
    if any then
        -- The run loop has already ended (the source's EOF stops it at once, composite.lua:662-681) and cleanup() runs in
        -- evaluation order, so the blocks downstream are still alive: let each of them take one more turn on the flushed tail.
        local downstream, todo = {}, {self}
        while #todo > 0 do
            local b = table.remove(todo)
            for _, port in ipairs(b.outputs) do
                for _, p in ipairs(port.pipes) do
                    local consumer = p.input.owner
                    if not downstream[consumer] then
                        downstream[consumer] = true
                        todo[#todo + 1] = consumer
                    end
                end
            end
        end
        for _, b in ipairs(self.evaluation_order or {}) do
            if downstream[b] then b:run_once() end
        end
    end
end

function GPUChainBlock:cleanup()
    -- super-chunk mode: hand the pending samples to the downstream pipes before they are closed
    local lib = platform.libs.cuda
    local out = self.out:resize(tonumber(lib.lrb200_graph_max_output(self.graph, 0)))
    if lib.lrb200_graph_flush(self.graph, out.data, n_out) ~= 0 then b200.fail("graph_flush") end
    hand_on_flushed(self, {out:resize(tonumber(n_out[0]))})
end

local M = {GPUChainBlock = GPUChainBlock}

--- Does `b` have a GPU form in its differentiated type (blocks_patch.lua)?
local function on_gpu(b)
    return b.make_device_handle ~= nil and (b.gpu_capable == nil or b:gpu_capable())
end

--- Is `b` a concrete GPU block that can sit inside a linear run?
local function is_gpu(b)
    return on_gpu(b) and #b.inputs == 1 and #b.outputs == 1
end

--- Substitute every maximal linear run (length >= 2) of GPU blocks in the crawled connection map.
-- connections: InputPort -> OutputPort over concrete blocks (composite.lua:343-381).
function M.collapse_gpu_runs(connections, substitutes)
    -- consumers per output port
    local consumers = {}
    for input, output in pairs(connections) do
        consumers[output] = consumers[output] or {}
        table.insert(consumers[output], input)
    end
    local function next_in_run(b)          -- the single GPU consumer of b's output, if the edge is 1:1
        local c = consumers[b.outputs[1]]
        if c and #c == 1 and is_gpu(c[1].owner) then return c[1].owner end
        return nil
    end
    local function prev_in_run(b)
        local up = connections[b.inputs[1]]
        if up and is_gpu(up.owner) and next_in_run(up.owner) == b then return up.owner end
        return nil
    end
    -- plan first, rewrite afterwards: adding keys to a table while pairs() walks it is undefined in Lua
    local seen, runs = {}, {}
    for input, _ in pairs(connections) do
        local b = input.owner
        if is_gpu(b) and not seen[b] and prev_in_run(b) == nil then
            local run = {b}
            seen[b] = true
            local nb = next_in_run(b)
            while nb do
                run[#run + 1] = nb
                seen[nb] = true
                nb = next_in_run(nb)
            end
            if #run >= 2 then runs[#runs + 1] = run end
        end
    end
    for _, run in ipairs(runs) do
        local edges = {}
        for _, rb in ipairs(run) do edges[rb.inputs[1]] = connections[rb.inputs[1]] end
        local chain = GPUChainBlock(run, edges)
        chain:differentiate({run[1]:get_input_type()})
        if substitutes then substitutes[#substitutes + 1] = chain end
        local first_in, last_out = run[1].inputs[1], run[#run].outputs[1]
        -- upstream edge now ends at the chain's input; edges inside the run disappear
        connections[chain.inputs[1]] = connections[first_in]
        for _, rb in ipairs(run) do connections[rb.inputs[1]] = nil end
        -- downstream consumers now read the chain's output
        for _, cin in ipairs(consumers[last_out] or {}) do connections[cin] = chain.outputs[1] end
    end
    return connections
end

--- A connected, NON-linear set of GPU blocks (a two-input block, PLLBlock's two outputs or a fan-out inside the set) fed by
-- ONE outside output port, or the sets that share one such port, as one device DAG (lrb200_dag_*): every edge between the members is a device buffer, the only
-- host traffic is the set's input and its outputs.  Linear runs inside the set become fused flow graphs
-- (lrb200_dag_add_graph), everything else single nodes (lrb200_dag_add_block).  A node's output k is referenced as
-- node * 4 + k, the DAG's own input as -1 (include/lrb200.h).  An absorbed raw file source (IQFileSource, RealFileSource
-- read by the set alone) makes it a source block: it freads the file's bytes itself and the source's converter is the
-- DAG's first node.  LUARADIO_B200_SUPERCHUNK switches on super-chunk mode (lrb200_dag_set_superchunk) as for the chains.
local GPUDagBlock = block.factory("GPUDagBlock")
GPUDagBlock.RAW_READ = 524288            -- samples per fread from an absorbed source (the reference's 8192 is launch-bound)

function GPUDagBlock:instantiate(members, ext_in, ext_out, edges, raw_source)
    self.blocks, self.ext_in, self.ext_out, self.edges, self.raw_source = members, ext_in, ext_out, edges, raw_source
    local outputs = {}
    for k, p in ipairs(ext_out) do outputs[k] = block.Output("out" .. k, p.data_type) end
    self:add_type_signature(raw_source and {} or {block.Input("in", ext_in.data_type)}, outputs)
end

function GPUDagBlock:get_rate()
    return self.ext_out[1].owner:get_rate()
end

function GPUDagBlock:initialize()
    local lib = platform.libs.cuda
    local edges = self.edges                              -- member input port -> producing output port (snapshot)
    self.dag = ffi.gc(lib.lrb200_dag_create(), lib.lrb200_dag_destroy)
    if self.dag == nil then b200.fail("dag_create") end
    local member, consumers = {}, {}
    for _, b in ipairs(self.blocks) do member[b] = true end
    for input, output in pairs(edges) do
        consumers[output] = consumers[output] or {}
        table.insert(consumers[output], input)
    end
    local function simple(b) return #b.inputs == 1 and #b.outputs == 1 end
    local function next_in_run(b)                         -- the single member consumer of a simple block, if the edge is 1:1
        local c = consumers[b.outputs[1]]
        if c and #c == 1 and member[c[1].owner] and simple(c[1].owner) then return c[1].owner end
        return nil
    end
    local ref, done = {}, {}
    ref[self.ext_in] = -1
    if self.raw_source then                               -- node 0: the file format converter, fed the raw bytes
        local h = self.raw_source:make_converter_handle()
        local ins = ffi.new("int[?]", 1)
        ins[0] = -1
        if lib.lrb200_dag_add_block(self.dag, h, ins, 1) < 0 then
            lib.lrb200_block_destroy(h)
            b200.fail("dag_add_block")
        end
        ref[self.ext_in] = 0
    end
    for _, b in ipairs(self.blocks) do                    -- evaluation (topological) order
        if not done[b] then
            local run = {}
            if simple(b) then
                run[1] = b
                local nb = next_in_run(b)
                while nb and not done[nb] do
                    run[#run + 1] = nb
                    nb = next_in_run(nb)
                end
            end
            if #run >= 2 then
                local g = lib.lrb200_graph_create()
                if g == nil then b200.fail("graph_create") end
                for _, rb in ipairs(run) do
                    if lib.lrb200_graph_append(g, rb:make_device_handle()) ~= 0 then b200.fail("graph_append") end
                end
                if lib.lrb200_graph_commit(g, 1) ~= 0 then b200.fail("graph_commit") end
                local node = lib.lrb200_dag_add_graph(self.dag, g, ref[edges[run[1].inputs[1]]])
                if node < 0 then
                    lib.lrb200_graph_destroy(g)
                    b200.fail("dag_add_graph")
                end
                ref[run[#run].outputs[1]] = node * 4
                for _, rb in ipairs(run) do done[rb] = true end
            else
                local ins = ffi.new("int[?]", #b.inputs)
                for i, p in ipairs(b.inputs) do ins[i - 1] = ref[edges[p]] end
                local h = b:make_device_handle()
                local node = lib.lrb200_dag_add_block(self.dag, h, ins, #b.inputs)
                if node < 0 then
                    lib.lrb200_block_destroy(h)
                    b200.fail("dag_add_block")
                end
                for k, p in ipairs(b.outputs) do ref[p] = node * 4 + (k - 1) end
                done[b] = true
            end
        end
    end
    local outs = ffi.new("int[?]", #self.ext_out)
    for k, p in ipairs(self.ext_out) do outs[k - 1] = ref[p] end
    if lib.lrb200_dag_set_outputs(self.dag, outs, #self.ext_out) ~= 0 then b200.fail("dag_set_outputs") end
    self.superchunk = tonumber(os.getenv('LUARADIO_B200_SUPERCHUNK') or 0)
    if self.superchunk > 0 and lib.lrb200_dag_set_superchunk(self.dag, self.superchunk) ~= 0 then b200.fail("dag_set_superchunk") end
    self.fed = false                                      -- samples went in since the last flush (super-chunk mode)
    self.outs, self.out_ptrs, self.n_outs = {}, ffi.new("void*[?]", #self.ext_out), ffi.new("size_t[?]", #self.ext_out)
    for k, p in ipairs(self.ext_out) do self.outs[k] = p.data_type.vector() end
    -- the source was initialised with the original blocks (its file is open); read bigger chunks than its own
    if self.raw_source then self.raw_source.raw_samples:resize(math.max(self.raw_source.chunk_size or 0, self.RAW_READ)) end
end

function GPUDagBlock:execute(data, n, flush)
    local lib = platform.libs.cuda
    for k, o in ipairs(self.outs) do
        self.out_ptrs[k - 1] = o:resize(tonumber(lib.lrb200_dag_max_output(self.dag, k - 1, n))).data
    end
    if flush then
        if lib.lrb200_dag_flush(self.dag, self.out_ptrs, self.n_outs) ~= 0 then b200.fail("dag_flush") end
    elseif lib.lrb200_dag_execute(self.dag, data, n, self.out_ptrs, self.n_outs) ~= 0 then
        b200.fail("dag_execute")
    end
    self.fed = self.superchunk > 0 and not flush
    for k, o in ipairs(self.outs) do o:resize(tonumber(self.n_outs[k - 1])) end
    return unpack(self.outs)
end

function GPUDagBlock:process(x)
    if self.raw_source then
        local src = self.raw_source
        local n = tonumber(ffi.C.fread(src.raw_samples.data, ffi.sizeof(src.raw_samples.data_type), src.raw_samples.length, src.file))
        if n == 0 then
            if ffi.C.feof(src.file) ~= 0 and src.repeat_on_eof then ffi.C.rewind(src.file) else return nil end
        end
        return self:execute(src.raw_samples.data, n)
    end
    return self:execute(x.data, x.length)
end

function GPUDagBlock:cleanup()
    -- super-chunk mode: hand the pending samples of every port to the downstream pipes before they are closed
    if self.fed then
        self:execute(nil, 0, true)
        hand_on_flushed(self, self.outs)
    end
end

M.GPUDagBlock = GPUDagBlock

--- Planning step: the connected sets of GPU blocks with exactly one outside feed that are not a straight line, and the
-- sets (straight lines and single blocks included) that share one outside feed, merged into one: several receivers on
-- one source become one DAG, so the source's samples cross PCIe once.  Returns an array of {members = {blocks in evaluation order}, ext_in = OutputPort, ext_out = {OutputPort, ...}}.
function M.plan_gpu_dags(connections)
    local gpu, order = {}, {}                             -- set of GPU blocks; all of them in a stable order
    local function note(b)
        if not gpu[b] and on_gpu(b) and #b.inputs >= 1 and #b.outputs >= 1 then
            gpu[b] = true
            order[#order + 1] = b
        end
    end
    for input, output in pairs(connections) do
        note(input.owner)
        note(output.owner)
    end
    local adj = {}
    for _, b in ipairs(order) do adj[b] = {} end
    for input, output in pairs(connections) do
        local a, c = input.owner, output.owner
        if gpu[a] and gpu[c] then
            adj[a][c] = true
            adj[c][a] = true
        end
    end
    local seen, feeds_in_order, by_feed = {}, {}, {}      -- the sets with one outside feed, grouped by that feed
    for _, b in ipairs(order) do
        if not seen[b] then
            -- connected component
            local comp, todo, count = {}, {b}, 0
            while #todo > 0 do
                local c = table.remove(todo)
                if not comp[c] then
                    comp[c] = true
                    count = count + 1
                    for nbr, _ in pairs(adj[c]) do
                        if not comp[nbr] then todo[#todo + 1] = nbr end
                    end
                end
            end
            for c, _ in pairs(comp) do seen[c] = true end
            -- shape: a multi-port member or a fan-out inside the set
            local nonlinear = false
            local internal_consumers = {}
            for input, output in pairs(connections) do
                if comp[input.owner] and comp[output.owner] then
                    internal_consumers[output] = (internal_consumers[output] or 0) + 1
                    if internal_consumers[output] > 1 then nonlinear = true end
                end
            end
            for c, _ in pairs(comp) do
                if #c.inputs > 1 or #c.outputs > 1 then nonlinear = true end
            end
            -- outside feeds
            local feeds, nfeeds, ext_in = {}, 0, nil
            for input, output in pairs(connections) do
                if comp[input.owner] and not comp[output.owner] and not feeds[output] then
                    feeds[output] = true
                    nfeeds = nfeeds + 1
                    ext_in = output
                end
            end
            if nfeeds == 1 then
                if not by_feed[ext_in] then
                    by_feed[ext_in] = {}
                    feeds_in_order[#feeds_in_order + 1] = ext_in
                end
                table.insert(by_feed[ext_in], {comp = comp, nonlinear = count >= 2 and nonlinear})
            end
        end
    end
    -- one candidate per feed: a non-linear set, or the sets (receivers) that share it; a lone straight line is left to
    -- collapse_gpu_runs and several outside feeds to the host scheduler
    local plans = {}
    for _, ext_in in ipairs(feeds_in_order) do
        local sets = by_feed[ext_in]
        if #sets >= 2 or sets[1].nonlinear then
            local comp = {}
            for _, s in ipairs(sets) do
                for c, _ in pairs(s.comp) do comp[c] = true end
            end
            -- members in evaluation order: depth-first over the producers inside the set
            local members, placed = {}, {}
            local function place(c)
                if placed[c] then return end
                placed[c] = true
                for _, p in ipairs(c.inputs) do
                    local up = connections[p].owner
                    if comp[up] then place(up) end
                end
                members[#members + 1] = c
            end
            for _, c in ipairs(order) do
                if comp[c] then place(c) end
            end
            local read_outside = {}
            for input, output in pairs(connections) do
                if comp[output.owner] and not comp[input.owner] then read_outside[output] = true end
            end
            local ext_out = {}
            for _, c in ipairs(members) do
                for _, p in ipairs(c.outputs) do
                    if read_outside[p] then ext_out[#ext_out + 1] = p end
                end
            end
            if #ext_out > 0 then plans[#plans + 1] = {members = members, ext_in = ext_in, ext_out = ext_out} end
        end
    end
    return plans
end

--- Substitute every planned set by one GPUDagBlock in the crawled connection map (before the linear runs are collapsed).
-- A raw file source whose output only the set reads is absorbed (the rule CompositeBlock._collapse_gpu_runs applies).
function M.collapse_gpu_dags(connections, substitutes)
    local plans = M.plan_gpu_dags(connections)
    for _, plan in ipairs(plans) do
        local member, edges = {}, {}
        for _, b in ipairs(plan.members) do member[b] = true end
        for _, b in ipairs(plan.members) do
            for _, p in ipairs(b.inputs) do edges[p] = connections[p] end
        end
        local src = plan.ext_in.owner
        if src.make_converter_handle == nil then src = nil end
        for input, output in pairs(connections) do
            if output == plan.ext_in and not member[input.owner] then src = nil end
        end
        local dag = GPUDagBlock(plan.members, plan.ext_in, plan.ext_out, edges, src)
        dag:differentiate(src and {} or {plan.ext_in.data_type})
        if substitutes then substitutes[#substitutes + 1] = dag end
        -- outside readers of a member output now read the matching DAG output; the members' own edges disappear
        local rewire = {}
        for input, output in pairs(connections) do
            if not member[input.owner] then
                for k, p in ipairs(plan.ext_out) do
                    if output == p then rewire[input] = dag.outputs[k] end
                end
            end
        end
        for input, output in pairs(rewire) do connections[input] = output end
        for p, _ in pairs(edges) do connections[p] = nil end
        if not src then connections[dag.inputs[1]] = plan.ext_in end
    end
    return connections
end

function M.install(radio)
    if not platform.features.cuda then return end
    local CompositeBlock = radio.CompositeBlock
    local crawl, start = CompositeBlock._crawl_connections, CompositeBlock.start
    local connect_pipes, initialize = CompositeBlock._connect_pipes, CompositeBlock._initialize
    -- _prepare_to_run (composite.lua:426-466) = _differentiate, _crawl_connections, _connect_pipes(all_connections),
    -- _validate_rates, _initialize, then the global evaluation order and the control sockets from all_connections.
    -- _validate_rates and _initialize walk the ORIGINAL blocks (self._connections), the run loop walks all_connections.
    function CompositeBlock:_crawl_connections(crawled_connections, composite_stack)
        local top_level = crawled_connections == nil
        local connections = crawl(self, crawled_connections, composite_stack)
        if top_level then
            self._b200_substitutes = {}
            M.collapse_gpu_dags(connections, self._b200_substitutes)
            M.collapse_gpu_runs(connections, self._b200_substitutes)
        end
        return connections
    end
    function CompositeBlock:_connect_pipes(all_connections)
        connect_pipes(self, all_connections)
        -- the members of a sub-graph have no pipes any more, but _validate_rates (composite.lua:394-414) and the members'
        -- own initialize() (LowpassFilterBlock:initialize -> self:get_rate(), block.lua:383-390) ask their input pipe for
        -- the rate: a rate-only link to the port that fed the member in the crawled graph
        for _, sub in ipairs(self._b200_substitutes or {}) do
            for input, output in pairs(sub.edges) do
                input.pipe = {get_rate = function () return output.owner:get_rate() end}
            end
            for _, b in ipairs(sub.blocks) do b.in_gpu_subgraph = true end
        end
    end
    function CompositeBlock:_initialize()
        -- the original blocks first (members: their subclass initialize() designs the taps, the patched base initialize()
        -- then skips the HOST handle), the substitutes afterwards: they take DEVICE handles from the initialised members
        initialize(self)
        for _, sub in ipairs(self._b200_substitutes or {}) do sub:initialize() end
    end
    local prepare = CompositeBlock._prepare_to_run
    function CompositeBlock:_prepare_to_run()
        local all_connections, evaluation_order = prepare(self)
        for _, sub in ipairs(self._b200_substitutes or {}) do sub.evaluation_order = evaluation_order end
        return all_connections, evaluation_order
    end
    function CompositeBlock:start(multiprocess)
        return start(self, false)       -- one process: the CUDA context cannot be forked (composite.lua:568-636)
    end
end

return M
