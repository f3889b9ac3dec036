"""CompositeBlock: flow-graph construction and the single-process GPU scheduler.

Graph building mirrors radio/core/composite.lua:111-216 (connect / aliasing), :302-424 (validate,
differentiate in evaluation order, crawl hierarchical blocks down to concrete ports, connect pipes,
validate rates, initialize).  Running differs by design (north_star): instead of fork-per-block over
socketpairs (composite.lua:568-636) the graph runs in ONE process on ONE CUDA stream.  Every MAXIMAL LINEAR
RUN of GPU blocks in the flattened graph -- wherever it sits in an arbitrary DAG -- is replaced by one
GPUChainBlock backed by the library's flow graph (lrb200_graph_*), where the blocks share device-resident
buffers and adjacent blocks are fused; host<->device copies happen only at the two ends of each run.  The
reduced graph (sources, chains, CPU blocks, multi-input blocks, sinks) runs in evaluation order like the
reference's run(false) round-robin (composite.lua:647-707).  start()/wait()/stop()/status() have the
reference's meaning (composite.lua:534-545, 858-913) on a scheduler thread.
"""
import ctypes
import sys
import threading

import numpy as np

from . import _lib
from .block import Block, Input, Output, Pipe, Port
from .signal_blocks import (MultiplyConstantBlock, UpsamplerBlock, ComplexBandpassFilterBlock, ComplexMagnitudeBlock, ComplexToRealBlock,
                            SinglepoleHighpassFilterBlock, DownsamplerBlock, FMDeemphasisFilterBlock, FrequencyDiscriminatorBlock,
                            FrequencyTranslatorBlock, GPUBlock, LowpassFilterBlock, HilbertTransformBlock, DelayBlock, PLLBlock,
                            MultiplyConjugateBlock, AddBlock, SubtractBlock)
from .types import ComplexFloat32, Float32, Vector


# -------------------------------------------------------------------------------------------------
# Minimal host-side sources/sinks for the boundary (the reference analogues are RawFileSource/Sink,
# radio/blocks/sources/rawfile.lua:75-108, radio/blocks/sinks/rawfile.lua:60-67, on in-memory buffers)
# -------------------------------------------------------------------------------------------------
class ArraySource(Block):
    name = "ArraySource"

    def instantiate(self, array, rate, chunk=1 << 22):
        a = np.ascontiguousarray(array)
        self.data_type = ComplexFloat32 if np.iscomplexobj(a) else Float32
        self.array = a.astype(self.data_type.dtype, copy=False)
        self.rate = float(rate)
        self.chunk = int(chunk)
        self.pos = 0
        self.add_type_signature([], [Output("out", self.data_type)])

    def get_rate(self):
        return self.rate

    def process(self):
        if self.pos >= len(self.array):
            return None    # EOF (block.lua:588)
        v = Vector.cast(self.array[self.pos:self.pos + self.chunk])
        self.pos += v.length
        return v


class IQFileSource(Block):
    """radio/blocks/sources/iqfile.lua:27-116: interleaved I/Q in one of 14 sample formats -> ComplexFloat32.
    `file` is a path, an open binary file, or a bytes-like object.  The format conversion (byte swap, offset,
    scale; iqfile.lua:96-108) runs on the GPU: process() converts one chunk through the C ABI; inside a GPU flow
    graph the converter becomes the graph's first stage and the RAW bytes cross PCIe (2 B/sample for "u8")."""
    name = "IQFileSource"
    raw_source = True                      # CompositeBlock: feed the graph read_raw() bytes, converter = stage 0
    components = 2
    create_fn = "lrb200_iqconv_create"
    out_type = ComplexFloat32
    FORMATS = {"u8": 1, "s8": 1, "u16le": 2, "u16be": 2, "s16le": 2, "s16be": 2, "u32le": 4, "u32be": 4,
               "s32le": 4, "s32be": 4, "f32le": 4, "f32be": 4, "f64le": 8, "f64be": 8}

    def instantiate(self, file, format, rate, repeat_on_eof=False, chunk=8192):
        assert file is not None, "Missing argument #1 (file)"
        assert format is not None, "Missing argument #2 (format)"
        assert format in self.FORMATS, 'Unsupported format ("%s")' % format
        assert rate is not None, "Missing argument #3 (rate)"
        self.file, self.format, self.rate, self.repeat_on_eof = file, format, float(rate), repeat_on_eof
        self.sample_bytes = self.components * self.FORMATS[format]
        self.chunk_size = int(chunk)          # samples per read; the reference uses 8192 (iqfile.lua:52)
        self._handle = None
        self.add_type_signature([], [Output("out", self.out_type)])

    def get_rate(self):
        return self.rate

    def initialize(self):
        # like the reference (fread() of chunk_size samples per process(), iqfile.lua:82-95) the file is read
        # incrementally, so a pipe (rtl_sdr | ...) streams and a capture larger than RAM works
        self._buf, self._fh, self._own_fh = None, None, False
        if isinstance(self.file, (bytes, bytearray, memoryview, np.ndarray)):
            self._buf = np.frombuffer(bytes(self.file) if not isinstance(self.file, np.ndarray) else self.file.tobytes(), np.uint8)
        elif isinstance(self.file, str):
            self._fh, self._own_fh = open(self.file, "rb"), True
        else:
            self._fh = self.file
        self._pos = 0
        self._tail = b""
        self.out = self.out_type.vector()

    def read_raw(self, samples=None):
        """Next chunk of raw file bytes (whole samples; `samples` overrides chunk_size), or None at EOF."""
        nbytes = (samples or self.chunk_size) * self.sample_bytes
        if self._buf is not None:
            if self._pos >= len(self._buf) - self.sample_bytes + 1:
                if not self.repeat_on_eof or len(self._buf) < self.sample_bytes:
                    return None
                self._pos = 0
            raw = self._buf[self._pos:self._pos + nbytes]
            raw = raw[:len(raw) // self.sample_bytes * self.sample_bytes]
            self._pos += len(raw)
            return np.ascontiguousarray(raw)
        data = self._tail + (self._fh.read(nbytes - len(self._tail)) or b"")
        if len(data) < self.sample_bytes and self.repeat_on_eof and self._fh.seekable():
            self._fh.seek(0)                                   # iqfile.lua:90-93
            data = self._fh.read(nbytes) or b""
        whole = len(data) // self.sample_bytes * self.sample_bytes
        self._tail = data[whole:]
        if whole == 0:
            return None
        return np.frombuffer(data[:whole], np.uint8)

    def make_device_handle(self):
        lib = _lib.require_device()
        return _lib.check_handle(getattr(lib, self.create_fn)(self.format.encode(), _lib.LRB200_DEVICE), "lrb200 file-format object")

    def process(self):
        raw = self.read_raw()
        if raw is None:
            return None
        lib = _lib.require_device()
        if self._handle is None:
            self._handle = _lib.check_handle(getattr(lib, self.create_fn)(self.format.encode(), _lib.LRB200_HOST), "lrb200 file-format object")
        n = len(raw) // self.sample_bytes
        out = self.out.resize(n)
        n_out = ctypes.c_size_t(0)
        _lib.check(lib.lrb200_block_execute(self._handle, raw.ctypes.data, n, out.ctypes_ptr(), ctypes.byref(n_out)), "file-format conversion")
        return out.resize(n_out.value)

    def cleanup(self):
        if self._handle:
            _lib.load().lrb200_block_destroy(self._handle)
            self._handle = None
        if getattr(self, "_own_fh", False) and self._fh is not None:
            self._fh.close()
            self._fh = None


class RealFileSource(IQFileSource):
    """radio/blocks/sources/realfile.lua:27-110: real samples in one of the 14 formats -> Float32, converted on the GPU."""
    name = "RealFileSource"
    components = 1
    create_fn = "lrb200_realconv_create"
    out_type = Float32


class RawFileSource(Block):
    """radio/blocks/sources/rawfile.lua:75-108: a file of raw `data_type` elements (host byte order) -> that type.
    Pure I/O: in a GPU flow graph the chunks go straight into the graph's pinned H2D staging."""
    name = "RawFileSource"

    def instantiate(self, file, data_type, rate, repeat_on_eof=False, chunk=8192):
        assert file is not None, "Missing argument #1 (file)"
        assert data_type is not None, "Missing argument #2 (data_type)"
        assert rate is not None, "Missing argument #3 (rate)"
        self.file, self.data_type, self.rate, self.repeat_on_eof, self.chunk_size = file, data_type, float(rate), repeat_on_eof, int(chunk)
        self.add_type_signature([], [Output("out", data_type)])

    def get_rate(self):
        return self.rate

    def initialize(self):
        dt = self.data_type.dtype
        if isinstance(self.file, str):
            self._buf = np.fromfile(self.file, dt)
        else:
            b = self.file if isinstance(self.file, (bytes, bytearray, memoryview)) else self.file.read()
            self._buf = np.frombuffer(bytes(b)[:len(b) // dt.itemsize * dt.itemsize], dt)
        self._pos = 0

    def process(self):
        if self._pos >= len(self._buf):
            if not self.repeat_on_eof or len(self._buf) == 0:
                return None
            self._pos = 0
        x = self._buf[self._pos:self._pos + self.chunk_size]
        self._pos += len(x)
        return Vector.cast(np.ascontiguousarray(x))


class _FileSinkBase(Block):
    """Shared by IQFileSink / RealFileSink / WAVFileSink: float samples -> the file's sample format on the GPU
    (lrb200_iqsink_create / lrb200_realsink_create).  process() converts one chunk through the C ABI; as the sink of a GPU
    flow graph the converter is the graph's last stage and write_raw() receives the file bytes from the D2H copy."""
    raw_sink = True
    components = 1
    create_fn = "lrb200_realsink_create"
    in_type = Float32
    FORMATS = IQFileSource.FORMATS

    def _setup(self, file, format):
        assert file is not None, "Missing argument #1 (file)"
        assert format in self.FORMATS, 'Unsupported format ("%s")' % format
        self.file, self.format = file, format
        self.raw_sample_bytes = self.components * self.FORMATS[format]
        self._handle, self._fh, self._own = None, None, False
        self.count = 0

    def initialize(self):
        if isinstance(self.file, str):
            self._fh, self._own = open(self.file, "wb"), True
        else:
            self._fh = self.file

    def make_device_handle(self):
        lib = _lib.require_device()
        return _lib.check_handle(getattr(lib, self.create_fn)(self.format.encode(), _lib.LRB200_DEVICE), "lrb200 file-format object")

    def convert(self, x):
        """samples (numpy / Vector) -> file bytes (uint8 array), through the C ABI in host-pointer mode."""
        lib = _lib.require_device()
        if self._handle is None:
            self._handle = _lib.check_handle(getattr(lib, self.create_fn)(self.format.encode(), _lib.LRB200_HOST), "lrb200 file-format object")
        a = np.ascontiguousarray(x.data if isinstance(x, Vector) else x, dtype=self.in_type.dtype)
        raw = np.zeros(len(a) * self.raw_sample_bytes, np.uint8)
        n_out = ctypes.c_size_t(0)
        _lib.check(lib.lrb200_block_execute(self._handle, a.ctypes.data, len(a), raw.ctypes.data, ctypes.byref(n_out)), "file-format conversion")
        return raw

    def write_raw(self, raw, num_samples):
        self.count += num_samples
        self._fh.write(raw.tobytes())

    def process(self, x):
        self.write_raw(self.convert(x), x.length)

    def cleanup(self):
        if self._handle:
            _lib.load().lrb200_block_destroy(self._handle)
            self._handle = None
        if self._fh is not None:
            self._fh.flush()
            if self._own:
                self._fh.close()
            self._fh = None


class IQFileSink(_FileSinkBase):
    """radio/blocks/sinks/iqfile.lua:25-100: ComplexFloat32 -> interleaved I/Q in one of the 14 formats."""
    name = "IQFileSink"
    components = 2
    create_fn = "lrb200_iqsink_create"
    in_type = ComplexFloat32

    def instantiate(self, file, format):
        self._setup(file, format)
        self.add_type_signature([Input("in", ComplexFloat32)], [])


class RealFileSink(_FileSinkBase):
    """radio/blocks/sinks/realfile.lua: Float32 -> real samples in one of the 14 formats."""
    name = "RealFileSink"

    def instantiate(self, file, format):
        self._setup(file, format)
        self.add_type_signature([Input("in", Float32)], [])


class RawFileSink(Block):
    """radio/blocks/sinks/rawfile.lua:60-67: any type, raw element bytes (host byte order).  Pure I/O."""
    name = "RawFileSink"

    def instantiate(self, file):
        assert file is not None, "Missing argument #1 (file)"
        self.file = file
        self.add_type_signature([Input("in", lambda t: True)], [])

    def initialize(self):
        self._own = isinstance(self.file, str)
        self._fh = open(self.file, "wb") if self._own else self.file

    def process(self, x):
        self._fh.write(np.ascontiguousarray(x.data).tobytes())

    def cleanup(self):
        self._fh.flush()
        if self._own:
            self._fh.close()


class WAVFileSink(_FileSinkBase):
    """radio/blocks/sinks/wavfile.lua:58-225: Float32 channel(s) -> PCM WAV (8/16/32 bits = u8/s16le/s32le).  The 44-byte
    RIFF/fmt/data headers are written on cleanup() with the final sizes (:196-218).  One channel: the conversion is the
    last stage of the GPU flow graph; two or more: channels are interleaved on the host, then converted."""
    name = "WAVFileSink"
    WAVE_FORMATS = {8: "u8", 16: "s16le", 32: "s32le"}

    def instantiate(self, file, num_channels, bits_per_sample=16):
        assert num_channels is not None, "Missing argument #2 (num_channels)"
        assert bits_per_sample in self.WAVE_FORMATS, "Unsupported bits per sample (%s)" % str(bits_per_sample)
        self._setup(file, self.WAVE_FORMATS[bits_per_sample])
        self.num_channels, self.bits_per_sample = int(num_channels), bits_per_sample
        self.raw_sink = self.num_channels == 1
        if self.num_channels == 1:
            self.add_type_signature([Input("in", Float32)], [])
        else:
            self.add_type_signature([Input("in%d" % (i + 1), Float32) for i in range(self.num_channels)], [])

    def header(self):
        import struct
        bps = self.bits_per_sample // 8
        data, rate = self.count * self.num_channels * bps, int(self.get_rate())
        return (b"RIFF" + struct.pack("<I", 36 + data) + b"WAVE" + b"fmt " +
                struct.pack("<IHHIIHH", 16, 1, self.num_channels, rate, rate * self.num_channels * bps,
                            self.num_channels * bps, self.bits_per_sample) + b"data" + struct.pack("<I", data))

    def initialize(self):
        _FileSinkBase.initialize(self)
        self._fh.write(b"\0" * 44)            # seek past the headers for now (wavfile.lua:162-165)

    def process(self, *channels):
        if self.num_channels == 1:
            return _FileSinkBase.process(self, channels[0])
        n = channels[0].length
        inter = np.stack([np.asarray(c.data[:n], np.float32) for c in channels], axis=1).reshape(-1)
        self.count += n
        self._fh.write(self.convert(inter).tobytes())

    def cleanup(self):
        if self._fh is not None:
            self._fh.seek(0)
            self._fh.write(self.header())
            self._fh.seek(0, 2)
        _FileSinkBase.cleanup(self)


class ArraySink(Block):
    name = "ArraySink"

    def instantiate(self):
        self.chunks = []
        self.add_type_signature([Input("in", lambda t: True)], [])

    def process(self, x):
        self.chunks.append(np.array(x.data, copy=True))

    def result(self):
        if not self.chunks:
            return np.zeros(0, dtype=self.get_input_type().dtype if self.signature else np.float32)
        return np.concatenate(self.chunks)


# -------------------------------------------------------------------------------------------------
def _evaluation_order(connections, blocks):
    deps = {b: set() for b in blocks}
    for inp, outp in connections.items():
        if inp.aliased or outp.aliased:
            continue
        deps.setdefault(inp.owner, set()).add(outp.owner)
        deps.setdefault(outp.owner, set())
    order = []
    while len(order) < len(deps):
        progressed = False
        for b, d in deps.items():
            if b not in order and all(x in order for x in d):
                order.append(b)
                progressed = True
                break
        if not progressed:
            raise AssertionError("Flow graph has a cycle.")
    return order


class CompositeBlock(Block):
    name = "CompositeBlock"

    def instantiate(self):
        self._blocks = []
        self._connections = {}      # input port (or aliased output) -> output port (or aliased input)
        self._order = None
        self._gpu_graph = None

    def add_type_signature(self, inputs, outputs, *a):
        Block.add_type_signature(self, inputs, outputs)
        for p in self.inputs + self.outputs:
            p.aliased = True

    # -- composite.lua:111-131
    def connect(self, *args):
        if all(isinstance(a, Block) for a in args):
            first = args[0]
            for i, second in enumerate(args[1:], start=2):
                assert len(first.outputs) == 1, 'Unexpected number of output ports in block %d "%s": found %d, expected 1.' % (i - 1, first.name, len(first.outputs))
                assert len(second.inputs) == 1, 'Unexpected number of input ports in block %d "%s": found %d, expected 1.' % (i, second.name, len(second.inputs))
                self._connect_by_name(first, first.outputs[0].name, second, second.inputs[0].name)
                first = second
        else:
            self._connect_by_name(*args)
        return self

    # -- composite.lua:133-187
    def _connect_by_name(self, src, src_port_name, dst, dst_port_name):
        find = lambda blk, nm: next((p for p in (blk.outputs or []) + (blk.inputs or []) if p.name == nm), None)
        src_port, dst_port = find(src, src_port_name), find(dst, dst_port_name)
        assert src_port, 'Output port "%s" of block "%s" not found.' % (src_port_name, src.name)
        assert dst_port, 'Input port "%s" of block "%s" not found.' % (dst_port_name, dst.name)
        self._order = None
        if src is not self and dst is not self:
            assert src_port.kind == "out", "Source port %s.%s is not an output port." % (src.name, src_port.name)
            assert dst_port.kind == "in", "Destination port %s.%s is not an input port." % (dst.name, dst_port.name)
            assert dst_port not in self._connections, 'Input port "%s" of block "%s" already connected.' % (dst_port.name, dst.name)
            self._connections[dst_port] = src_port
            for b in (src, dst):
                if b not in self._blocks:
                    self._blocks.append(b)
        else:
            alias_port = src_port if src is self else dst_port
            target_port = dst_port if src is self else src_port
            if alias_port.kind == "in" and target_port.kind == "in":
                assert target_port not in self._connections, "Input port %s.%s already connected." % (target_port.owner.name, target_port.name)
                self._connections[target_port] = alias_port
            elif alias_port.kind == "out" and target_port.kind == "out":
                assert alias_port not in self._connections, "Output port %s.%s already connected." % (alias_port.owner.name, alias_port.name)
                self._connections[alias_port] = target_port
            else:
                raise AssertionError("Malformed port connection.")
            if target_port.owner not in self._blocks:
                self._blocks.append(target_port.owner)

    def _eval_order(self):
        if self._order is None:
            self._order = _evaluation_order(self._connections, self._blocks)
        return self._order

    # -- composite.lua:302-341
    def _validate_inputs(self):
        for b in self._blocks:
            for p in b.inputs or []:
                assert p in self._connections, 'Block "%s" input "%s" is unconnected.' % (b.name, p.name)
            if isinstance(b, CompositeBlock):
                b._validate_inputs()

    def _differentiate(self):
        for b in self._eval_order():
            b.differentiate([self._connections[p].data_type for p in b.inputs])
            if isinstance(b, CompositeBlock):
                b._differentiate()
        for out in self.outputs or []:
            src = self._connections[out]
            assert out.data_type is src.data_type, "Invalid type signature, composite output %s.%s data type does not match block output %s.%s." % (self.name, out.name, src.owner.name, src.name)

    # -- composite.lua:343-379: flatten hierarchical blocks to concrete (input port -> output port)
    def _crawl_connections(self, crawled=None, stack=()):
        crawled = {} if crawled is None else crawled

        def resolve(port):
            if port.kind == "out" and not port.aliased:
                return port
            if port.kind == "out" and port.aliased:
                return resolve(port.owner._connections[port])
            for comp in stack:
                if port in comp._connections:
                    return resolve(comp._connections[port])
            raise AssertionError("Unexpected disconnected composite input port %s.%s" % (port.owner.name, port.name))

        for b in self._eval_order():
            if isinstance(b, CompositeBlock):
                b._crawl_connections(crawled, (self,) + tuple(stack))
            else:
                for p in b.inputs:
                    crawled[p] = resolve(self._connections[p])
        return crawled

    def _prepare_to_run(self, initialize=True):
        self._validate_inputs()
        self._differentiate()
        self._all_connections = self._crawl_connections()
        for inp, outp in self._all_connections.items():      # a second run() starts from clean ports
            outp.pipes = []
            inp.pipe = None
        for inp, outp in self._all_connections.items():
            pipe = Pipe(outp, inp)
            outp.pipes.append(pipe)
            inp.pipe = pipe
        concrete = []
        for inp, outp in self._all_connections.items():
            for b in (outp.owner, inp.owner):
                if b not in concrete:
                    concrete.append(b)
        self._concrete_order = _evaluation_order(self._all_connections, concrete)
        for b in self._concrete_order:           # rate validation, composite.lua:394-414
            rates = [p.pipe.get_rate() for p in b.inputs]
            assert all(r == rates[0] for r in rates), 'Block "%s" input sample rate mismatch.' % b.name
        if initialize:
            for b in self._concrete_order:       # composite.lua:416-424: initialize every block
                b.initialize()

    # ---------------------------------------------------------------------------------------------
    # GPU scheduler: maximal linear GPU runs -> GPUChainBlock, then round-robin over the reduced graph
    # ---------------------------------------------------------------------------------------------
    def _plan_gpu_dags(self):
        """Pure planning step: the candidates for ONE device DAG (lrb200_dag_*), every edge in device memory.  A connected
        set of GPU blocks fed by exactly one external output port is one when it is NOT a straight line (it contains a
        multi-port block or an internal fan-out); the sets that share one such feed -- receivers on one source, straight
        lines and single blocks included -- are merged into one candidate, so the shared input crosses PCIe once.  Sets
        with several external feeds stay on the host scheduler.  Returns [(members in evaluation order, external producer
        port, [member output ports read from outside])]."""
        orig = self._all_connections
        gpu = [b for b in self._concrete_order if isinstance(b, GPUBlock) and b.inputs and b.outputs]
        gset = set(gpu)
        adj = {b: set() for b in gpu}
        for inp, outp in orig.items():
            if inp.owner in gset and outp.owner in gset:
                adj[inp.owner].add(outp.owner)
                adj[outp.owner].add(inp.owner)
        seen, by_feed = set(), {}                            # external feed -> [(set, non-linear)]
        for b in gpu:
            if b in seen:
                continue
            comp, todo = set(), [b]
            while todo:
                c = todo.pop()
                if c in comp:
                    continue
                comp.add(c)
                todo.extend(adj[c] - comp)
            seen |= comp
            ext_in = {orig[p] for m in comp for p in m.inputs if orig[p].owner not in comp}
            if len(ext_in) != 1:
                continue                                     # several external feeds: stays a host-level graph
            fan_out = any(sum(1 for i, o in orig.items() if o is p and i.owner in comp) > 1 for m in comp for p in m.outputs)
            nonlinear = len(comp) >= 2 and (fan_out or any(len(m.inputs) > 1 or len(m.outputs) > 1 for m in comp))
            by_feed.setdefault(next(iter(ext_in)), []).append((comp, nonlinear))
        plans = []
        for ext_in, sets in by_feed.items():
            if len(sets) == 1 and not sets[0][1]:
                continue                                     # a lone straight line: the chain planner's business
            comp = set().union(*(s for s, _ in sets))
            members = [m for m in self._concrete_order if m in comp]
            ext_out = []
            for m in members:
                for p in m.outputs:
                    if any(o is p and i.owner not in comp for i, o in orig.items()):
                        ext_out.append(p)
            if not ext_out:
                continue
            plans.append((members, ext_in, ext_out))
        return plans

    def _plan_gpu_runs(self, exclude=()):
        """Pure planning step (no device needed): every maximal linear run of GPU blocks in the flattened graph, as
        [(blocks, absorbed raw file source or None, absorbed raw file sink or None)].  A run of ONE block is only kept
        when it borders a raw file source / sink (otherwise the block's own handle does the same work).  Blocks in
        `exclude` (members of a device DAG) are not considered."""
        orig = self._all_connections
        consumers = {}
        for inp, outp in orig.items():
            consumers.setdefault(outp, []).append(inp)
        exclude = set(exclude)

        def is_gpu(b):
            return isinstance(b, GPUBlock) and len(b.inputs) == 1 and len(b.outputs) == 1 and b not in exclude

        def next_in_run(b):
            c = consumers.get(b.outputs[0], [])
            return c[0].owner if len(c) == 1 and is_gpu(c[0].owner) else None

        def prev_in_run(b):
            up = orig[b.inputs[0]].owner
            return up if is_gpu(up) and next_in_run(up) is b else None

        plan = []
        for b in list(self._concrete_order):
            if not is_gpu(b) or prev_in_run(b) is not None:
                continue
            run, nb = [b], next_in_run(b)
            while nb is not None:
                run.append(nb)
                nb = next_in_run(nb)
            up_port = orig[run[0].inputs[0]]
            src = up_port.owner if getattr(up_port.owner, "raw_source", False) and len(consumers.get(up_port, [])) == 1 else None
            down = consumers.get(run[-1].outputs[0], [])
            snk = down[0].owner if len(down) == 1 and getattr(down[0].owner, "raw_sink", False) and len(down[0].owner.inputs) == 1 else None
            if len(run) < 2 and src is None and snk is None:
                continue
            plan.append((run, src, snk))
        return plan

    def _collapse_gpu_runs(self, fuse, superchunk, device_dag=True):
        """Rewrite (self._all_connections, self._concrete_order): every planned device DAG becomes one GPUDagBlock, every
        planned run one GPUChainBlock; a raw file source feeding only a run or a DAG (several receivers merged into one DAG
        included), and a raw file sink fed only by a run, are absorbed as its first / last stage."""
        orig = self._all_connections          # lookups use the untouched map; the rewrite goes into `conns`
        conns = dict(orig)
        consumers = {}
        for inp, outp in orig.items():
            consumers.setdefault(outp, []).append(inp)
        chains, dag_members = [], set()
        for members, ext_in, ext_out in (self._plan_gpu_dags() if device_dag else []):
            # a raw file source read by the DAG alone is absorbed: its converter becomes the DAG's first node
            src = ext_in.owner if getattr(ext_in.owner, "raw_source", False) and \
                all(cin.owner in members for cin in consumers.get(ext_in, [])) else None
            dag = GPUDagBlock(members, ext_in, ext_out, orig, fuse, superchunk, src)
            chains.append(dag)
            dag_members.update(members)
            for m in members:
                for p in m.inputs:
                    del conns[p]
            if src is None:
                conns[dag.inputs[0]] = ext_in
                dag.inputs[0].pipe = next(p for m in members for p in m.inputs if orig[p] is ext_in).pipe
            for k, port in enumerate(ext_out):
                for cin in consumers.get(port, []):
                    if cin.owner not in dag_members:
                        conns[cin] = dag.outputs[k]
        for run, src, snk in self._plan_gpu_runs(dag_members):
            up_port = orig[run[0].inputs[0]]
            down = consumers.get(run[-1].outputs[0], [])
            chain = GPUChainBlock(run, src, snk, fuse, superchunk)
            chains.append(chain)
            for rb in run:
                del conns[rb.inputs[0]]
            if src is None:
                conns[chain.inputs[0]] = up_port
                chain.inputs[0].pipe = run[0].inputs[0].pipe          # rate propagation
            if snk is None:
                for cin in down:
                    conns[cin] = chain.outputs[0]
            else:
                del conns[snk.inputs[0]]
        absorbed = set()
        for c in chains:
            absorbed.update(c.blocks)
            absorbed.update(x for x in (getattr(c, "raw_source", None), getattr(c, "raw_sink", None)) if x is not None)
        blocks = [b for b in self._concrete_order if b not in absorbed] + chains
        self._chains = chains
        self._run_connections = conns
        self._run_order = _evaluation_order(conns, blocks) if conns else blocks
        for c in chains:
            c.initialize()

    def describe_gpu_graph(self):
        """The committed device flow graph(s) of the last run: stages separated by ' | ', several runs by ' ; '."""
        return " ; ".join(c.desc for c in getattr(self, "_chains", []) if c.desc)

    def _schedule(self):
        """One process, evaluation order, FIFOs per input port (composite.lua:647-707); at end of stream the chains and
        DAGs are flushed (super-chunk mode) and the graph drains, again while a flush hands samples downstream (a device
        sub-graph behind another one only sees the first one's tail after that drain)."""
        order, conns = self._run_order, self._run_connections
        fifo = {inp: [] for inp in conns}
        consumers = {}
        for inp, outp in conns.items():
            consumers.setdefault(outp, []).append(inp)

        def push(b, outs):
            for port, vec in zip(b.outputs, outs):
                if vec is None or vec.length == 0:
                    continue
                data = np.array(vec.data, copy=True)
                for cin in consumers.get(port, []):
                    fifo[cin].append(data)

        exhausted, flushed, flush_moved = set(), False, False
        while not self._stop_requested:
            live = False
            for b in order:
                if not b.inputs:
                    if b in exhausted:
                        continue
                    v = b.process()
                    if v is None:
                        exhausted.add(b)
                        continue
                    push(b, v if isinstance(v, tuple) else (v,))
                    live = True
                    continue
                if any(len(fifo[p]) == 0 for p in b.inputs):
                    continue
                arrays = [np.concatenate(fifo[p]) if len(fifo[p]) > 1 else fifo[p][0] for p in b.inputs]
                n = min(len(a) for a in arrays)
                if n == 0:
                    continue
                for p, a in zip(b.inputs, arrays):
                    fifo[p] = [a[n:]] if len(a) > n else []
                r = b.process(*[Vector.cast(a[:n]) for a in arrays])
                push(b, () if r is None else (r if isinstance(r, tuple) else (r,)))
                live = True
            if live:
                continue
            if flushed and not flush_moved:
                break
            # every source is at EOF and nothing moved: push the pending super-chunks out and drain once more
            flushed, flush_moved = True, False
            for b in order:
                if isinstance(b, (GPUChainBlock, GPUDagBlock)):
                    r = b.flush()
                    if r is not None:
                        outs = r if isinstance(r, tuple) else (r,)
                        flush_moved = flush_moved or any(v is not None and v.length for v in outs)
                        push(b, outs)

    def _run_body(self, fuse, superchunk, device_dag=True):
        try:
            self._collapse_gpu_runs(fuse, superchunk, device_dag)
            self._schedule()
        finally:
            # composite.lua:693-696: clean up every block, whatever happened (native handles, file sinks, WAV header)
            pending = sys.exc_info()[0] is not None
            first = None
            for b in getattr(self, "_run_order", []) + [x for x in self._concrete_order if x not in getattr(self, "_run_order", [])]:
                try:
                    b.cleanup()
                except Exception as e:          # keep cleaning up; report the first failure unless an error is already in flight
                    first = first or e
            if first is not None and not pending:
                raise first

    # -- composite.lua:534-545 start, :858 status, :886 stop, :913 wait, :937 run
    def start(self, multiprocess=False, fuse=True, superchunk=0, device_dag=True):
        """Prepare the flow graph and start running it on a scheduler thread.  `multiprocess` is accepted for API
        compatibility; the GPU scheduler is always single-process (a CUDA context does not survive fork(), SURVEY.md 7e)."""
        if getattr(self, "_running", False):
            raise RuntimeError("CompositeBlock already running!")
        self._prepare_to_run()
        self._stop_requested, self._error = False, None
        lib = _lib.load()
        device = lib.lrb200_current_device()

        def body():
            try:
                if device >= 0:
                    _lib.check(lib.lrb200_init(device), "lrb200_init")      # the CUDA device is a per-thread setting
                self._run_body(fuse, superchunk, device_dag)
            except BaseException as e:      # surfaced by wait()
                self._error = e
            finally:
                self._running = False

        self._running = True
        self._thread = threading.Thread(target=body, name="luaradio_b200-scheduler", daemon=True)
        self._thread.start()
        return self

    def status(self):
        """{'running': bool} like composite.lua:858-877."""
        return {"running": bool(getattr(self, "_running", False))}

    def stop(self):
        """Ask the scheduler to stop after the vector in flight, then wait for it (composite.lua:886-906)."""
        if getattr(self, "_thread", None) is None:
            return
        self._stop_requested = True
        self.wait()

    def wait(self):
        """Block until the flow graph has finished (sources at EOF or stop()); re-raises a block's error."""
        t = getattr(self, "_thread", None)
        if t is None:
            return
        t.join()
        self._thread = None
        if self._error is not None:
            err, self._error = self._error, None
            raise err

    def run(self, multiprocess=False, fuse=True, superchunk=0, device_dag=True):
        """start() + wait() (composite.lua:937-941), on the calling thread.  device_dag=False keeps non-linear GPU parts as
        host-level graphs of chains and single blocks (a host round trip at every junction)."""
        if getattr(self, "_running", False):
            raise RuntimeError("CompositeBlock already running!")
        self._prepare_to_run()
        self._stop_requested, self._error = False, None
        self._running = True
        try:
            self._run_body(fuse, superchunk, device_dag)
        finally:
            self._running = False
        return self


class GPUChainBlock(Block):
    """A maximal linear run of connected GPU blocks as ONE device-resident flow graph (lrb200_graph_*): the executable
    twin of lua/radio_b200/composite_patch.lua's GPUChainBlock.  An absorbed raw file source makes it a source block (the
    file's own bytes cross PCIe and are converted by the graph's first stage), an absorbed raw file sink a sink block."""
    name = "GPUChainBlock"
    RAW_READ = 1 << 19          # samples per read when the chain pulls from an absorbed file source (the reference's 8192 is launch-bound)

    def instantiate(self, blocks, raw_source=None, raw_sink=None, fuse=True, superchunk=0):
        self.blocks, self.raw_source, self.raw_sink = list(blocks), raw_source, raw_sink
        self.fuse, self.superchunk = fuse, int(superchunk or 0)
        self.graph, self.desc = None, ""
        ins = [] if raw_source is not None else [Input("in", blocks[0].get_input_type())]
        outs = [] if raw_sink is not None else [Output("out", blocks[-1].get_output_type())]
        self.add_type_signature(ins, outs)
        self.differentiate([d.data_type for d in ins])

    def get_rate(self):
        return self.blocks[-1].get_rate()

    def initialize(self):
        lib = self._lib = _lib.require_device()
        g = _lib.check_handle(lib.lrb200_graph_create(), "lrb200 graph")
        self.graph = g
        if self.raw_source is not None:
            _lib.check(lib.lrb200_graph_append(g, self.raw_source.make_device_handle()), "graph_append(file source)")
        for b in self.blocks:
            _lib.check(lib.lrb200_graph_append(g, b.make_device_handle()), "graph_append(%s)" % b.name)
        if self.raw_sink is not None:
            _lib.check(lib.lrb200_graph_append(g, self.raw_sink.make_device_handle()), "graph_append(file sink)")
        _lib.check(lib.lrb200_graph_commit(g, 1 if self.fuse else 0), "graph_commit")
        self.desc = lib.lrb200_graph_describe(g).decode()
        if self.superchunk:
            _lib.check(lib.lrb200_graph_set_superchunk(g, self.superchunk), "graph_set_superchunk")
        self.out = None if self.raw_sink is not None else self.blocks[-1].get_output_type().vector()
        self._raw_out = np.zeros(0, np.uint8)
        self._n_out = ctypes.c_size_t(0)

    def _execute(self, in_ptr, n_in, flush=False):
        lib, g = self._lib, self.graph
        cap = lib.lrb200_graph_max_output(g, n_in)
        if self.raw_sink is not None:
            need = cap * self.raw_sink.raw_sample_bytes
            if len(self._raw_out) < need:
                self._raw_out = np.zeros(need, np.uint8)
            out_ptr = self._raw_out.ctypes.data
        else:
            self.out.resize(cap)
            out_ptr = self.out.ctypes_ptr()
        if flush:
            _lib.check(lib.lrb200_graph_flush(g, out_ptr, ctypes.byref(self._n_out)), "graph_flush")
        else:
            _lib.check(lib.lrb200_graph_execute(g, in_ptr, n_in, out_ptr, ctypes.byref(self._n_out)), "graph_execute")
        n = self._n_out.value
        if self.raw_sink is not None:
            if n:
                self.raw_sink.write_raw(self._raw_out[:n * self.raw_sink.raw_sample_bytes], n)
            return None
        return self.out.resize(n)

    def process(self, x=None):
        if self.raw_source is not None:
            raw = self.raw_source.read_raw(max(self.raw_source.chunk_size, self.RAW_READ))
            if raw is None:
                return None                                   # EOF (block.lua:588)
            r = self._execute(raw.ctypes.data, len(raw) // self.raw_source.sample_bytes)
            return r if r is not None else ()
        return self._execute(x.ctypes_ptr(), x.length)

    def flush(self):
        return self._execute(None, 0, flush=True) if self.graph else None

    def cleanup(self):
        if self.graph:
            self._lib.lrb200_graph_destroy(self.graph)
            self.graph = None


class GPUDagBlock(Block):
    """A connected, non-linear set of GPU blocks, or the sets that share one external feed (receivers on one source), as ONE
    device DAG (lrb200_dag_*): every edge between them is a device buffer; the only host traffic is the single input and
    the outputs.  Linear runs inside the set are added as fused
    lrb200 flow graphs, the rest (two-input blocks, PLL, lone blocks) as single nodes.  An absorbed raw file source makes it
    a source block: the file's own bytes cross PCIe and the source's converter is the DAG's first node.  With `superchunk`
    the host vectors are packed into super-chunks (lrb200_dag_set_superchunk) and flush() drains them at end of stream."""
    name = "GPUDagBlock"
    RAW_READ = GPUChainBlock.RAW_READ

    def instantiate(self, members, ext_in, ext_out, connections, fuse=True, superchunk=0, raw_source=None):
        self.blocks, self.ext_in, self.ext_out, self.fuse = list(members), ext_in, list(ext_out), fuse
        self.superchunk, self.raw_source = int(superchunk or 0), raw_source
        self._conn = connections
        self.dag, self.desc = None, ""
        ins = [] if raw_source is not None else [Input("in", ext_in.data_type)]
        self.add_type_signature(ins, [Output("out%d" % (k + 1), p.data_type) for k, p in enumerate(ext_out)])
        self.differentiate([d.data_type for d in ins])

    def get_rate(self):
        return self.ext_out[0].owner.get_rate()

    def initialize(self):
        lib = self._lib = _lib.require_device()
        d = self.dag = _lib.check_handle(lib.lrb200_dag_create(), "lrb200 dag")
        conn, members = self._conn, set(self.blocks)
        consumers = {}
        for inp, outp in conn.items():
            consumers.setdefault(outp, []).append(inp)
        ref = {self.ext_in: -1}                      # output port -> DAG reference
        if self.raw_source is not None:              # node 0: the file format converter, fed the raw bytes
            h = self.raw_source.make_device_handle()
            if lib.lrb200_dag_add_block(d, h, (ctypes.c_int * 1)(-1), 1) < 0:
                lib.lrb200_block_destroy(h)
                raise _lib.LibraryError("dag_add_block(file source): " + _lib.last_error())
            ref[self.ext_in] = 0

        def simple(b):
            return len(b.inputs) == 1 and len(b.outputs) == 1

        def next_in_run(b):                          # the single member consumer of a simple block, if that edge is 1:1
            c = consumers.get(b.outputs[0], [])
            return c[0].owner if len(c) == 1 and c[0].owner in members and simple(c[0].owner) else None

        done = set()
        for b in self.blocks:                        # evaluation order == topological order
            if b in done:
                continue
            if simple(b):
                run, nb = [b], next_in_run(b)
                while nb is not None and nb not in done:
                    run.append(nb)
                    nb = next_in_run(nb)
                if len(run) >= 2:
                    g = _lib.check_handle(lib.lrb200_graph_create(), "lrb200 graph")
                    for rb in run:
                        _lib.check(lib.lrb200_graph_append(g, rb.make_device_handle()), "graph_append(%s)" % rb.name)
                    _lib.check(lib.lrb200_graph_commit(g, 1 if self.fuse else 0), "graph_commit")
                    node = lib.lrb200_dag_add_graph(d, g, ref[conn[run[0].inputs[0]]])
                    if node < 0:
                        lib.lrb200_graph_destroy(g)
                        raise _lib.LibraryError("dag_add_graph: " + _lib.last_error())
                    ref[run[-1].outputs[0]] = node * 4
                    done.update(run)
                    continue
            ins = (ctypes.c_int * len(b.inputs))(*[ref[conn[p]] for p in b.inputs])
            h = b.make_device_handle()
            node = lib.lrb200_dag_add_block(d, h, ins, len(b.inputs))
            if node < 0:
                lib.lrb200_block_destroy(h)
                raise _lib.LibraryError("dag_add_block(%s): %s" % (b.name, _lib.last_error()))
            for k, p in enumerate(b.outputs):
                ref[p] = node * 4 + k
            done.add(b)
        outs = (ctypes.c_int * len(self.ext_out))(*[ref[p] for p in self.ext_out])
        _lib.check(lib.lrb200_dag_set_outputs(d, outs, len(self.ext_out)), "dag_set_outputs")
        if not self.fuse:                            # else the DAG commits itself, rewrites on, at its first use
            _lib.check(lib.lrb200_dag_commit(d, 0), "dag_commit")
        if self.superchunk:
            _lib.check(lib.lrb200_dag_set_superchunk(d, self.superchunk), "dag_set_superchunk")
        self.desc = "dag{" + lib.lrb200_dag_describe(d).decode() + "}"
        self.outs = [p.data_type.vector() for p in self.ext_out]
        self._n_out = (ctypes.c_size_t * len(self.ext_out))()
        self._fed = False                            # samples went in since the last flush (super-chunk mode)

    def _execute(self, in_ptr, n_in, flush=False):
        lib, d = self._lib, self.dag
        for k, o in enumerate(self.outs):
            o.resize(lib.lrb200_dag_max_output(d, k, n_in))
        ptrs = (ctypes.c_void_p * len(self.outs))(*[o.ctypes_ptr() for o in self.outs])
        if flush:
            _lib.check(lib.lrb200_dag_flush(d, ptrs, self._n_out), "dag_flush")
        else:
            _lib.check(lib.lrb200_dag_execute(d, in_ptr, n_in, ptrs, self._n_out), "dag_execute")
        self._fed = bool(self.superchunk) and not flush
        res = tuple(o.resize(self._n_out[k]) for k, o in enumerate(self.outs))
        return res[0] if len(res) == 1 else res

    def process(self, x=None):
        if self.raw_source is not None:
            raw = self.raw_source.read_raw(max(self.raw_source.chunk_size, self.RAW_READ))
            if raw is None:
                return None                                   # EOF (block.lua:588)
            return self._execute(raw.ctypes.data, len(raw) // self.raw_source.sample_bytes)
        return self._execute(x.ctypes_ptr(), x.length)

    def flush(self):
        """The pending super-chunks' outputs, one vector per port (a vector when there is one port), or None."""
        if not self.dag or not self._fed:
            return None
        return self._execute(None, 0, flush=True)

    def cleanup(self):
        if self.dag:
            self._lib.lrb200_dag_destroy(self.dag)
            self.dag = None


# -------------------------------------------------------------------------------------------------
# Composites on the hot path
# -------------------------------------------------------------------------------------------------
class TunerBlock(CompositeBlock):
    """composites/tuner.lua:32-48: Translator(offset) -> Lowpass(num_taps or 128, bandwidth/2) -> Downsampler(D)."""
    name = "TunerBlock"

    def instantiate(self, offset, bandwidth, decimation, options=None):
        CompositeBlock.instantiate(self)
        assert offset is not None, "Missing argument #1 (offset)"
        assert bandwidth is not None, "Missing argument #2 (bandwidth)"
        assert decimation is not None, "Missing argument #3 (decimation)"
        options = options or {}
        translator = FrequencyTranslatorBlock(offset)
        filt = LowpassFilterBlock(options.get("num_taps", 128), bandwidth / 2.0, None, options.get("window"))
        downsampler = DownsamplerBlock(decimation)
        self.connect(translator, filt, downsampler)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
        self.connect(self, "in", translator, "in")
        self.connect(self, "out", downsampler, "out")


class DecimatorBlock(CompositeBlock):
    """composites/decimator.lua:28-42: Lowpass(num_taps or 128, 1/D, nyquist 1.0) -> Downsampler(D)."""
    name = "DecimatorBlock"

    def instantiate(self, decimation, options=None):
        CompositeBlock.instantiate(self)
        assert decimation is not None, "Missing argument #1 (decimation)"
        options = options or {}
        filt = LowpassFilterBlock(options.get("num_taps", 128), 1.0 / decimation, 1.0, options.get("window"))
        downsampler = DownsamplerBlock(decimation)
        self.connect(filt, downsampler)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
        self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])
        self.connect(self, "in", filt, "in")
        self.connect(self, "out", downsampler, "out")


class WBFMMonoDemodulator(CompositeBlock):
    """composites/wbfmmonodemodulator.lua:22-35."""
    name = "WBFMMonoDemodulator"

    def instantiate(self, tau=None):
        CompositeBlock.instantiate(self)
        tau = tau or 75e-6
        fm_demod = FrequencyDiscriminatorBlock(1.25)
        af_filter = LowpassFilterBlock(128, 15e3)
        af_deemphasis = FMDeemphasisFilterBlock(tau)
        self.connect(fm_demod, af_filter, af_deemphasis)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", Float32)])
        self.connect(self, "in", fm_demod, "in")
        self.connect(self, "out", af_deemphasis, "out")


class NBFMDemodulator(CompositeBlock):
    """composites/nbfmdemodulator.lua:26-41: Lowpass(128, deviation + bandwidth) -> FrequencyDiscriminator(deviation /
    bandwidth) -> Lowpass(128, bandwidth).  Three GPU blocks -> one flow graph (FFT FIR | discriminator | FFT FIR)."""
    name = "NBFMDemodulator"

    def instantiate(self, deviation=None, bandwidth=None):
        CompositeBlock.instantiate(self)
        deviation = deviation or 5e3
        bandwidth = bandwidth or 4e3
        rf_filter = LowpassFilterBlock(128, 2 * (deviation + bandwidth) / 2)
        fm_demod = FrequencyDiscriminatorBlock(deviation / bandwidth)
        af_filter = LowpassFilterBlock(128, bandwidth)
        self.connect(rf_filter, fm_demod, af_filter)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", Float32)])
        self.connect(self, "in", rf_filter, "in")
        self.connect(self, "out", af_filter, "out")


class AMEnvelopeDemodulator(CompositeBlock):
    """composites/amenvelopedemodulator.lua:24-38: ComplexMagnitude -> SinglepoleHighpass(100) -> Lowpass(128, bandwidth)."""
    name = "AMEnvelopeDemodulator"

    def instantiate(self, bandwidth=None):
        CompositeBlock.instantiate(self)
        bandwidth = bandwidth or 5e3
        am_demod = ComplexMagnitudeBlock()
        dcr_filter = SinglepoleHighpassFilterBlock(100)
        af_filter = LowpassFilterBlock(128, bandwidth)
        self.connect(am_demod, dcr_filter, af_filter)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", Float32)])
        self.connect(self, "in", am_demod, "in")
        self.connect(self, "out", af_filter, "out")


class SSBDemodulator(CompositeBlock):
    """composites/ssbdemodulator.lua:25-43: ComplexBandpass(129, {0, +-bandwidth}) -> ComplexToReal -> Lowpass(128, bandwidth)."""
    name = "SSBDemodulator"

    def instantiate(self, sideband, bandwidth=None):
        CompositeBlock.instantiate(self)
        assert sideband, "Missing argument #1 (sideband)"
        assert sideband in ("lsb", "usb"), "Sideband should be 'lsb' or 'usb'"
        bandwidth = bandwidth or 3e3
        sb_filter = ComplexBandpassFilterBlock(129, [0, -bandwidth] if sideband == "lsb" else [0, bandwidth])
        am_demod = ComplexToRealBlock()
        af_filter = LowpassFilterBlock(128, bandwidth)
        self.connect(sb_filter, am_demod, af_filter)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", Float32)])
        self.connect(self, "in", sb_filter, "in")
        self.connect(self, "out", af_filter, "out")


class WBFMStereoDemodulator(CompositeBlock):
    """composites/wbfmstereodemodulator.lua:22-64: discriminator -> Hilbert(129); pilot: ComplexBandpass(129, 18-20 kHz) ->
    PLL(100, 19 kHz +- 50, x2); L+R: Delay(129) -> Lowpass(128, 15e3) -> ComplexToReal; L-R: Delay * conj(PLL) -> Lowpass ->
    ComplexToReal; left = (L+R) + (L-R), right = (L+R) - (L-R), each -> FMDeemphasis(tau).  A DAG: the scheduler turns its
    linear GPU runs (discriminator -> Hilbert; Lowpass -> ComplexToReal twice) into device flow graphs, the two-input
    blocks and the PLL run as single GPU blocks at their junctions."""
    name = "WBFMStereoDemodulator"

    def instantiate(self, tau=None):
        CompositeBlock.instantiate(self)
        tau = tau or 75e-6
        bandwidth = 15e3
        fm_demod = FrequencyDiscriminatorBlock(1.25)
        hilbert = HilbertTransformBlock(129)
        delay = DelayBlock(129)
        pilot_filter = ComplexBandpassFilterBlock(129, [18e3, 20e3])
        pilot_pll = PLLBlock(100, 19e3 - 50, 19e3 + 50, 2)
        mixer = MultiplyConjugateBlock()
        lpr_filter, lpr_am_demod = LowpassFilterBlock(128, bandwidth), ComplexToRealBlock()
        lmr_filter, lmr_am_demod = LowpassFilterBlock(128, bandwidth), ComplexToRealBlock()
        l_sum, left_af_deemphasis = AddBlock(), FMDeemphasisFilterBlock(tau)
        r_sub, right_af_deemphasis = SubtractBlock(), FMDeemphasisFilterBlock(tau)
        self.connect(fm_demod, hilbert)
        self.connect(hilbert, pilot_filter)
        self.connect(pilot_filter, "out", pilot_pll, "in")
        self.connect(hilbert, delay)
        self.connect(delay, "out", mixer, "in1")
        self.connect(pilot_pll, "out", mixer, "in2")
        self.connect(delay, lpr_filter, lpr_am_demod)
        self.connect(mixer, lmr_filter, lmr_am_demod)
        self.connect(lpr_am_demod, "out", l_sum, "in1")
        self.connect(lmr_am_demod, "out", l_sum, "in2")
        self.connect(lpr_am_demod, "out", r_sub, "in1")
        self.connect(lmr_am_demod, "out", r_sub, "in2")
        self.connect(l_sum, left_af_deemphasis)
        self.connect(r_sub, right_af_deemphasis)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("left", Float32), Output("right", Float32)])
        self.connect(self, "in", fm_demod, "in")
        self.connect(self, "left", left_af_deemphasis, "out")
        self.connect(self, "right", right_af_deemphasis, "out")


class AMSynchronousDemodulator(CompositeBlock):
    """composites/amsynchronousdemodulator.lua:25-45: ComplexBandpass(129, ifreq +- bandwidth) -> [PLL(1000, ifreq +- 100)]
    -> MultiplyConjugate(filtered, pll) -> ComplexToReal -> SinglepoleHighpass(100) -> Lowpass(128, bandwidth)."""
    name = "AMSynchronousDemodulator"

    def instantiate(self, ifreq, bandwidth=None):
        CompositeBlock.instantiate(self)
        assert ifreq is not None, "Missing argument #1 (ifreq)"
        bandwidth = bandwidth or 5e3
        rf_filter = ComplexBandpassFilterBlock(129, [ifreq - bandwidth, ifreq + bandwidth])
        pll = PLLBlock(1000, ifreq - 100, ifreq + 100)
        mixer = MultiplyConjugateBlock()
        am_demod = ComplexToRealBlock()
        dcr_filter = SinglepoleHighpassFilterBlock(100)
        af_filter = LowpassFilterBlock(128, bandwidth)
        self.connect(rf_filter, "out", pll, "in")
        self.connect(rf_filter, "out", mixer, "in1")
        self.connect(pll, "out", mixer, "in2")
        self.connect(mixer, am_demod, dcr_filter, af_filter)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", Float32)])
        self.connect(self, "in", rf_filter, "in")
        self.connect(self, "out", af_filter, "out")


class InterpolatorBlock(CompositeBlock):
    """composites/interpolator.lua:25-44: MultiplyConstant(L) -> Upsampler(L) -> Lowpass(num_taps or 128, 1/L, nyquist 1.0).
    The GPU flow graph commits the three blocks to one polyphase kernel (M/L products per output)."""
    name = "InterpolatorBlock"

    def instantiate(self, interpolation, options=None):
        CompositeBlock.instantiate(self)
        assert interpolation is not None, "Missing argument #1 (interpolation)"
        options = options or {}
        scaler = MultiplyConstantBlock(interpolation)
        upsampler = UpsamplerBlock(interpolation)
        filt = LowpassFilterBlock(options.get("num_taps", 128), 1.0 / interpolation, 1.0, options.get("window"))
        self.connect(scaler, upsampler, filt)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
        self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])
        self.connect(self, "in", scaler, "in")
        self.connect(self, "out", filt, "out")


class RationalResamplerBlock(CompositeBlock):
    """composites/rationalresampler.lua:25-49: MultiplyConstant(L) -> Upsampler(L) -> Lowpass(num_taps or 128,
    min(1/L, 1/D), nyquist 1.0) -> Downsampler(D); one polyphase kernel in the GPU flow graph."""
    name = "RationalResamplerBlock"

    def instantiate(self, interpolation, decimation, options=None):
        CompositeBlock.instantiate(self)
        assert interpolation is not None, "Missing argument #1 (interpolation)"
        assert decimation is not None, "Missing argument #2 (decimation)"
        options = options or {}
        cutoff = min(1.0 / interpolation, 1.0 / decimation)
        scaler = MultiplyConstantBlock(interpolation)
        upsampler = UpsamplerBlock(interpolation)
        filt = LowpassFilterBlock(options.get("num_taps", 128), cutoff, 1.0, options.get("window"))
        downsampler = DownsamplerBlock(decimation)
        self.connect(scaler, upsampler, filt, downsampler)
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])
        self.add_type_signature([Input("in", Float32)], [Output("out", Float32)])
        self.connect(self, "in", scaler, "in")
        self.connect(self, "out", downsampler, "out")
