"""Receivers that share one source are planned as ONE device DAG, by CompositeBlock._plan_gpu_dags and by its Lua twin
(lua/radio_b200/composite_patch.lua: plan_gpu_dags), with no device: the connected GPU sets with exactly one outside
feed are grouped by that feed, and two or more sets on one feed become one candidate -- straight lines and single blocks
included -- while a lone straight line stays the chain planner's and sets with several feeds stay on the host
scheduler."""
import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200.block import Block, Input, Output
from luaradio_b200.types import ComplexFloat32
from tests.test_lua_exec import LUA_GPU_BASE, export_graph, patched_radio

RATE = 2.4e6
X = np.zeros(16, np.complex64)


class Host(Block):
    name = "Host"

    def instantiate(self):
        self.add_type_signature([Input("in", ComplexFloat32)], [Output("out", ComplexFloat32)])


def nbfm(top, src, offset):
    top.connect(src, radio.TunerBlock(offset, 25e3, 48), radio.NBFMDemodulator(5e3, 4e3), radio.ArraySink())


def wbfm(top, src, offset):
    top.connect(src, radio.TunerBlock(offset, 200e3, 10), radio.WBFMMonoDemodulator(), radio.ArraySink())


def two_receivers():
    top, src = radio.CompositeBlock(), radio.ArraySource(X, RATE)
    nbfm(top, src, -300e3)
    nbfm(top, src, 200e3)
    return top


def three_receivers():
    top, src = radio.CompositeBlock(), radio.ArraySource(X, RATE)
    nbfm(top, src, -300e3)
    nbfm(top, src, 200e3)
    wbfm(top, src, 600e3)
    return top


def host_in_the_middle():
    top, src = radio.CompositeBlock(), radio.ArraySource(X, RATE)
    top.connect(src, radio.TunerBlock(-300e3, 25e3, 48), Host(), radio.NBFMDemodulator(5e3, 4e3), radio.ArraySink())
    nbfm(top, src, 200e3)
    return top


def source_with_a_host_reader():
    top, src = radio.CompositeBlock(), radio.ArraySource(X, RATE)
    nbfm(top, src, -300e3)
    nbfm(top, src, 200e3)
    top.connect(src, radio.ArraySink())
    return top


def single_block_branch():
    top, src = radio.CompositeBlock(), radio.ArraySource(X, RATE)
    nbfm(top, src, -300e3)
    top.connect(src, radio.FrequencyTranslatorBlock(100e3), radio.ArraySink())
    return top


def two_sources():
    top = radio.CompositeBlock()
    nbfm(top, radio.ArraySource(X, RATE), -300e3)
    nbfm(top, radio.ArraySource(X, RATE), 200e3)
    return top


TOPOLOGIES = {"two_receivers": two_receivers, "three_receivers": three_receivers, "host_in_the_middle": host_in_the_middle,
              "source_with_a_host_reader": source_with_a_host_reader, "single_block_branch": single_block_branch,
              "two_sources": two_sources}

TUNER = ["FrequencyTranslatorBlock", "LowpassFilterBlock", "DownsamplerBlock"]
NBFM = TUNER + ["LowpassFilterBlock", "FrequencyDiscriminatorBlock", "LowpassFilterBlock"]
WBFM = TUNER + ["FrequencyDiscriminatorBlock", "LowpassFilterBlock", "FMDeemphasisFilterBlock"]


def prepared(name):
    top = TOPOLOGIES[name]()
    top._prepare_to_run(initialize=False)
    return top


def receivers(top, members):
    """The members split by the sink (or host block) each one feeds, in evaluation order: one list of names per receiver."""
    out, mset = [], set(members)
    consumers = {}
    for inp, outp in top._all_connections.items():
        consumers.setdefault(outp.owner, []).append(inp.owner)
    for m in members:
        if top._all_connections[m.inputs[0]].owner not in mset:        # the first block of a receiver
            chain, b = [], m
            while b in mset:
                chain.append(b.name)
                b = consumers[b][0]
            out.append(chain)
    return out


@pytest.mark.parametrize("name", ["two_receivers", "three_receivers", "source_with_a_host_reader"])
def test_receivers_on_one_source_are_one_dag(name):
    top = prepared(name)
    dags = top._plan_gpu_dags()
    assert len(dags) == 1
    members, ext_in, ext_out = dags[0]
    want = [NBFM, NBFM] + ([WBFM] if name == "three_receivers" else [])
    assert receivers(top, members) == want
    assert members == [b for b in top._concrete_order if b in set(members)]        # evaluation order
    assert ext_in.owner.name == "ArraySource"
    assert [p.owner.name for p in ext_out] == [r[-1] for r in want]
    assert all(i.owner.name == "ArraySink" for i, o in top._all_connections.items() if o in ext_out)
    assert top._plan_gpu_runs(set(members)) == []


def test_only_the_part_before_a_host_block_merges():
    top = prepared("host_in_the_middle")
    (members, ext_in, ext_out), = top._plan_gpu_dags()
    assert receivers(top, members) == [TUNER, NBFM]
    assert ext_in.owner.name == "ArraySource"
    assert [p.owner.name for p in ext_out] == ["DownsamplerBlock", "LowpassFilterBlock"]
    consumers = [i.owner.name for i, o in top._all_connections.items() if o is ext_out[0]]
    assert consumers == ["Host"]
    # the demodulator behind the host block is still a chain of its own
    assert [[b.name for b in run] for run, _, _ in top._plan_gpu_runs(set(members))] == [NBFM[3:]]


def test_a_single_block_branch_joins_the_dag():
    top = prepared("single_block_branch")
    (members, ext_in, ext_out), = top._plan_gpu_dags()
    assert receivers(top, members) == [NBFM, ["FrequencyTranslatorBlock"]]
    assert [p.owner.name for p in ext_out] == ["LowpassFilterBlock", "FrequencyTranslatorBlock"]
    assert top._plan_gpu_runs(set(members)) == []


def test_two_different_sources_stay_two_chains():
    top = prepared("two_sources")
    assert top._plan_gpu_dags() == []
    assert [[b.name for b in run] for run, _, _ in top._plan_gpu_runs()] == [NBFM, NBFM]


def test_a_lone_receiver_is_still_a_chain():
    top = radio.CompositeBlock()
    nbfm(top, radio.ArraySource(X, RATE), -300e3)
    top._prepare_to_run(initialize=False)
    assert top._plan_gpu_dags() == []
    assert [[b.name for b in run] for run, _, _ in top._plan_gpu_runs()] == [NBFM]


@pytest.mark.parametrize("name", list(TOPOLOGIES))
def test_lua_planner_merges_the_same_receivers(monkeypatch, name):
    """plan_gpu_dags (Lua, executed against the mocks of tests/test_lua_exec.py) returns the members, the outside feed and
    the outside-read outputs of CompositeBlock._plan_gpu_dags, and collapse_gpu_dags leaves no member edge behind."""
    it, lib, types, lradio = patched_radio(monkeypatch)
    top = prepared(name)
    lua_gpu = {b: LUA_GPU_BASE[b.name] for b in top._concrete_order if b.name in LUA_GPU_BASE}
    expected = top._plan_gpu_dags()
    lua_of, conns = export_graph(it, lradio, types, top, lua_gpu)
    patch = it.require("radio_b200.composite_patch")
    plans = it.call(patch.hash["plan_gpu_dags"], [conns])[0].array()
    assert len(plans) == len(expected) == (0 if name == "two_sources" else 1)
    if not expected:
        return
    lua_port = lambda p: lua_of[p.owner].hash["outputs"].hash[p.owner.outputs.index(p) + 1]
    (members_py, ext_in_py, ext_out_py), plan = expected[0], plans[0]
    members = plan.hash["members"].array()
    assert len(members) == len(members_py) and {id(m) for m in members} == {id(lua_of[b]) for b in members_py}
    assert plan.hash["ext_in"] is lua_port(ext_in_py)
    ext_out = plan.hash["ext_out"].array()
    assert len(ext_out) == len(ext_out_py) and {id(p) for p in ext_out} == {id(lua_port(p)) for p in ext_out_py}
    index = {id(m): k for k, m in enumerate(members)}
    for m in members:                                    # evaluation order: producers first
        for p in m.hash["inputs"].array():
            up = conns.hash[p].hash["owner"]
            if id(up) in index:
                assert index[id(up)] < index[id(m)]
    it.call(patch.hash["collapse_gpu_dags"], [conns])
    member_ids = {id(m) for m in members}
    for i, o in conns.hash.items():
        assert id(i.hash["owner"]) not in member_ids and id(o.hash["owner"]) not in member_ids
