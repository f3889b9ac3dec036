"""The Lua GPUDagBlock's host boundary (super-chunk mode, flush, an absorbed raw file source) executed under the test
interpreter against the mock library, next to the Python GPUDagBlock run against a recording mock of the same library:
both issue the same create / add / set_superchunk / execute / flush sequence for the WBFM-stereo receiver fed by a u8
IQFileSource, and both keep a source that has a second reader out of the DAG."""
import numpy as np
import pytest

from luaradio_b200 import _lib
from tests.test_lua_exec import LUA_GPU_BASE, MockLib, export_graph, patched_radio, vec

SUPERCHUNK = 1 << 20
RAW_READ = 1 << 19


class PyMockLib:
    """libluaradio_b200 as ctypes sees it, for the Python scheduler: records (name, args); handles are fresh integers."""

    def __init__(self):
        self.calls, self._next, self.dag_nodes = [], 100, 0

    def __getattr__(self, name):
        if not name.startswith("lrb200_"):
            raise AttributeError(name)

        def fn(*args):
            self.calls.append((name, args))
            if "_create" in name:
                self._next += 1
                return self._next
            if name.endswith(("_describe", "_name", "last_error")):
                return b"mock"
            if name.endswith("max_output"):
                return args[-1]
            if name in ("lrb200_dag_add_graph", "lrb200_dag_add_block"):
                self.dag_nodes += 1
                return self.dag_nodes - 1
            if name in ("lrb200_dag_execute", "lrb200_dag_flush"):
                n_out = args[-1]
                for k in range(len(n_out)):
                    n_out[k] = args[2] if name == "lrb200_dag_execute" else 3
            return 0
        return fn


def flush_answers_three(orig_getattr):
    """MockLib.__getattr__ with lrb200_dag_flush answering three samples per port, like the mock's graph flush."""
    def getattr_(self, name):
        fn = orig_getattr(self, name)
        if name != "lrb200_dag_flush":
            return fn

        def flush(*args):
            fn(*args)
            for k in (0, 1):
                args[2].hash[k] = 3
            return [0]
        return flush
    return getattr_


def stereo_from_file(second_reader=False):
    import luaradio_b200 as radio
    raw = np.zeros(2 * (RAW_READ + 1000), np.uint8).tobytes()
    src = radio.IQFileSource(raw, "u8", 1102500.0)
    demod = radio.WBFMStereoDemodulator()
    top = radio.CompositeBlock()
    top.connect(src, radio.TunerBlock(-250e3, 200e3, 5), demod)
    top.connect(demod, "left", radio.ArraySink(), "in")
    top.connect(demod, "right", radio.ArraySink(), "in")
    if second_reader:
        top.connect(src, radio.ArraySink())
    return top, src


@pytest.fixture
def py_mock(monkeypatch):
    lib = PyMockLib()
    monkeypatch.setattr(_lib, "_lib", lib)
    return lib


def python_dag(py_mock, second_reader=False):
    from luaradio_b200.composite import GPUDagBlock
    top, src = stereo_from_file(second_reader)
    top._prepare_to_run()
    py_mock.calls.clear()
    top._collapse_gpu_runs(True, SUPERCHUNK)
    dags = [c for c in top._chains if isinstance(c, GPUDagBlock)]
    assert len(dags) == 1
    return top, src, dags[0]


def lua_dag(monkeypatch, top, src):
    monkeypatch.setattr(MockLib, "__getattr__", flush_answers_three(MockLib.__getattr__))
    it, lib, types, radio = patched_radio(monkeypatch)
    lua_gpu = {b: LUA_GPU_BASE[b.name] for b in top._concrete_order if b.name in LUA_GPU_BASE}
    lua_gpu[src] = "IQFileSource"
    lua_of, conns = export_graph(it, radio, types, top, lua_gpu)
    ls = lua_of[src]
    ls.hash.update({"format_name": "u8", "chunk_size": 8192, "file": "FILE*", "raw_samples": vec(types, "ComplexFloat32", 8192)})
    patch = it.require("radio_b200.composite_patch")
    it.call(patch.hash["collapse_gpu_dags"], [conns])
    dags = {id(o.hash["owner"]): o.hash["owner"] for o in conns.hash.values() if "ext_out" in o.hash["owner"].hash}
    assert len(dags) == 1
    return it, lib, next(iter(dags.values())), lua_of, conns


KEEP = ("lrb200_dag_", "lrb200_graph_create", "lrb200_graph_append", "lrb200_graph_commit")


def sequence(calls):
    """The calls that build and drive the DAG, block creations by kind (a FIR's taps type does not matter here)."""
    out = []
    for name, args in calls:
        if name.startswith(("lrb200_fir_create", "lrb200_iir_create")):
            out.append(name.rsplit("_", 1)[0])
        elif "_create" in name or name.startswith(KEEP):
            if name in ("lrb200_dag_describe",):
                continue
            out.append(name)
    return out


def phases(seq):
    """(head up to the first member node, the member nodes as a multiset, tail from set_outputs)"""
    head_end = seq.index("lrb200_dag_add_block") + 1
    tail = seq.index("lrb200_dag_set_outputs")
    return seq[:head_end], sorted(seq[head_end:tail]), seq[tail:]


def test_lua_dag_block_issues_the_python_sequence(monkeypatch, py_mock):
    top, src, dag = python_dag(py_mock)
    assert dag.raw_source is src and not dag.inputs
    dag.process()
    dag.flush()
    assert dag.flush() is None                               # nothing went in since the last flush
    py = sequence(py_mock.calls)
    executes = [a for n, a in py_mock.calls if n == "lrb200_dag_execute"]
    assert len(executes) == 1 and executes[0][2] == RAW_READ
    assert ("lrb200_dag_set_superchunk", (dag.dag, SUPERCHUNK)) in py_mock.calls

    it, lib, ldag, lua_of, conns = lua_dag(monkeypatch, top, src)
    monkeypatch.setenv("LUARADIO_B200_SUPERCHUNK", str(SUPERCHUNK))
    assert ldag.hash["raw_source"] is lua_of[src] and ldag.hash["inputs"].length() == 0
    # the absorbed source's output feeds nothing any more; the DAG is a source block
    assert all(o is not lua_of[src].hash["outputs"].hash[1] for o in conns.hash.values())
    meth = lambda obj, nm, *a: it.call(it.index(obj, nm), [obj] + list(a))
    lib.calls.clear()
    lib.dag_nodes = 0
    meth(ldag, "initialize")
    outs = meth(ldag, "process")
    assert len(outs) == 2 and all(o.hash["length"] == RAW_READ for o in outs)
    meth(ldag, "cleanup")
    lua = sequence(lib.calls)
    h_py, n_py, t_py = phases(py)
    h_lua, n_lua, t_lua = phases(lua)
    assert h_py == h_lua == ["lrb200_dag_create", "lrb200_iqconv_create", "lrb200_dag_add_block"]
    assert n_py == n_lua
    assert t_py == t_lua == ["lrb200_dag_set_outputs", "lrb200_dag_set_superchunk"] + ["lrb200_dag_max_output"] * 2 + \
        ["lrb200_dag_execute"] + ["lrb200_dag_max_output"] * 2 + ["lrb200_dag_flush"]
    # the converter node reads the DAG's input (-1); the file's raw chunk is what execute is handed
    conv = next(a for n, a in lib.calls if n == "lrb200_dag_add_block")
    assert conv[1].what == "lrb200_iqconv_create" and conv[1].args == ("u8", 1) and conv[2].hash[0] == -1
    ex = next(a for n, a in lib.calls if n == "lrb200_dag_execute")
    assert ex[1] == lua_of[src].hash["raw_samples"].hash["data"] and ex[2] == RAW_READ
    assert ("lrb200_dag_set_superchunk", (ldag.hash["dag"], SUPERCHUNK)) in lib.calls


def test_a_source_with_a_second_reader_is_not_absorbed(monkeypatch, py_mock):
    top, src, dag = python_dag(py_mock, second_reader=True)
    assert dag.raw_source is None and len(dag.inputs) == 1 and src in top._run_order
    assert "lrb200_iqconv_create" not in [n for n, _ in py_mock.calls]
    it, lib, ldag, lua_of, conns = lua_dag(monkeypatch, top, src)
    assert ldag.hash.get("raw_source") is None and ldag.hash["inputs"].length() == 1
    assert conns.hash[ldag.hash["inputs"].hash[1]] is lua_of[src].hash["outputs"].hash[1]
