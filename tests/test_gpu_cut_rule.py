"""Where a stream can be cut, pinned: lrb200_graph_halo of linear flow graphs (fused and unfused), lrb200_dag_halo and
lrb200_dag_shard_record_bytes of the receivers' DAGs and of a two-node PLL DAG, and the refusal of a block whose memory
is unbounded.  The expected values were recorded from the library before graphs and DAGs shared one cut rule; they are
the contract of that rule (halos are whole output periods and multiples of 4 samples)."""
import ctypes

import numpy as np
import pytest

from luaradio_b200 import _lib
from tests.blocks_util import create_block

pytestmark = pytest.mark.gpu

C1, R1 = [np.zeros(1, np.complex64)], [np.zeros(1, np.float32)]


def _iir(name):
    from tests.iir_order_ref import filters
    b, a = filters()[name]
    return ("IIRFilterBlock", [b, a], R1)


# name: [(rate the block runs at, block, args, a sample of its input type)]
GRAPHS = {
    # examples/rtlsdr_wbfm_mono.lua: tuner -> discriminator -> audio filter -> de-emphasis -> /5
    "wbfm_mono": [(1102500.0, "FrequencyTranslatorBlock", [-250e3], C1), (1102500.0, "LowpassFilterBlock", [128, 100e3], C1),
                  (1102500.0, "DownsamplerBlock", [5], C1), (220500.0, "FrequencyDiscriminatorBlock", [1.25], C1),
                  (220500.0, "LowpassFilterBlock", [128, 15e3], R1), (220500.0, "FMDeemphasisFilterBlock", [75e-6], R1),
                  (220500.0, "DownsamplerBlock", [5], R1)],
    # PowerSquelch in front of the AM envelope demodulator
    "am_envelope_squelch": [(48000.0, "PowerSquelchBlock", [-45], C1), (48000.0, "ComplexMagnitudeBlock", [], C1),
                            (48000.0, "SinglepoleHighpassFilterBlock", [100], R1), (48000.0, "LowpassFilterBlock", [128, 5e3], R1)],
    # the RDS symbol path: the phase corrector's N * I window dominates
    "rds_phase_corrector": [(8000.0, "LowpassFilterBlock", [128, 100], C1), (8000.0, "RootRaisedCosineFilterBlock", [101, 1, 31.25], C1),
                            (8000.0, "BinaryPhaseCorrectorBlock", [50, 32], C1)],
    # state-space IIRs: 11 taps on both sides, and 1 / 40 taps behind a /4
    "iir_order": [(1e5,) + _iir("butter5_bandstop"), (1e5,) + _iir("allpole40"), (1e5, "DownsamplerBlock", [4], R1)],
    # composites/interpolator.lua and rationalresampler.lua (3/5)
    "interpolator": [(1e5, "MultiplyConstantBlock", [3.0], C1), (1e5, "UpsamplerBlock", [3], C1),
                     (3e5, "LowpassFilterBlock", [128, 1.0 / 3, 1.0], C1)],
    "resampler_3_5": [(1e5, "MultiplyConstantBlock", [3.0], R1), (1e5, "UpsamplerBlock", [3], R1),
                      (3e5, "LowpassFilterBlock", [128, 1.0 / 5, 1.0], R1), (3e5, "DownsamplerBlock", [5], R1)],
}

# name: {fuse: lrb200_graph_halo}
EXPECTED_GRAPH_HALO = {
    "wbfm_mono": {1: 3200, 0: 3100},
    "am_envelope_squelch": {1: 3588, 0: 3588},
    "rds_phase_corrector": {1: 1832, 0: 1832},
    "iir_order": {1: 432, 0: 432},
    "interpolator": {1: 48, 0: 48},
    "resampler_3_5": {1: 60, 0: 60},
}


def graph_of(lib, spec, fuse):
    g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
    for rate, cls, args, inp in spec:
        b = create_block(cls, args, inp, rate)
        _lib.check(lib.lrb200_graph_append(g, b.make_device_handle()), "append")
        b.cleanup()
    _lib.check(lib.lrb200_graph_commit(g, fuse), "commit")
    return g


def observe_graph(name, fuse):
    lib = _lib.require_device()
    g = graph_of(lib, GRAPHS[name], fuse)
    try:
        return lib.lrb200_graph_halo(g)
    finally:
        lib.lrb200_graph_destroy(g)


@pytest.mark.parametrize("fuse", [1, 0])
@pytest.mark.parametrize("name", list(GRAPHS))
def test_graph_halo(name, fuse):
    assert observe_graph(name, fuse) == EXPECTED_GRAPH_HALO[name][fuse]


# name: (lrb200_dag_halo, lrb200_dag_shard_record_bytes); the receivers with the PLL in mode 0 and 1, and the PLL DAG of
# test_gpu_dag_shard.py (x -> PLL -> MultiplyConjugate(x, pll.out))
EXPECTED_DAG = {
    ("stereo", 0): (67560, 48),
    ("stereo", 1): (67560, 48),
    ("am_synchronous", 0): (2652, 48),
    ("rds", 0): (1286820, 48),
    ("rds", 1): (1286820, 48),
    ("fanout", 0): (132, 0),
    ("pll", 0): (12636, 48),
    ("pll", 1): (12636, 48),
}


def observe_dag(name, mode):
    from tests.test_gpu_dag_boundary import CASES, release
    from tests.test_gpu_dag_shard import make_dag, pll_dag
    lib = _lib.require_device()
    if name == "pll":
        d = pll_dag(lib, mode)
        try:
            return lib.lrb200_dag_halo(d), lib.lrb200_dag_shard_record_bytes(d)
        finally:
            lib.lrb200_dag_destroy(d)
    top, dag = make_dag(name, CASES[name][1]()[:1 << 16], mode)
    try:
        return lib.lrb200_dag_halo(dag.dag), lib.lrb200_dag_shard_record_bytes(dag.dag)
    finally:
        release(top)


@pytest.mark.parametrize("name,mode", list(EXPECTED_DAG))
def test_dag_halo_and_record_bytes(name, mode):
    assert observe_dag(name, mode) == EXPECTED_DAG[(name, mode)]


def test_unbounded_memory_is_refused_by_name():
    """AGC's gain integrates the whole past: neither a graph nor a DAG holding it can be cut, and the error names it."""
    lib = _lib.require_device()
    agc = create_block("AGCBlock", ["custom", -20, -40, {"gain_tau": 1e-3, "power_tau": 5e-5}], C1, 48000.0)
    g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
    try:
        _lib.check(lib.lrb200_graph_append(g, agc.make_device_handle()), "append")
        _lib.check(lib.lrb200_graph_commit(g, 1), "commit")
        assert lib.lrb200_graph_halo(g) == -1
        assert "agc_cc has unbounded memory, the stream cannot be cut" in _lib.last_error(), _lib.last_error()
    finally:
        lib.lrb200_graph_destroy(g)
    d = _lib.check_handle(lib.lrb200_dag_create(), "dag")
    try:
        assert lib.lrb200_dag_add_block(d, agc.make_device_handle(), (ctypes.c_int * 1)(-1), 1) == 0
        _lib.check(lib.lrb200_dag_set_outputs(d, (ctypes.c_int * 1)(0), 1), "set_outputs")
        assert lib.lrb200_dag_halo(d) == -1
        assert "agc_cc has unbounded memory, the stream cannot be cut" in _lib.last_error(), _lib.last_error()
        assert lib.lrb200_dag_shard_record_bytes(d) == 0
    finally:
        lib.lrb200_dag_destroy(d)
        agc.cleanup()
