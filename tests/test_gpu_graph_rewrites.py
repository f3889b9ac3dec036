"""The flow graph's fusion rules, pinned: each block sequence below is committed with fuse = 1 and fuse = 0, and the test
checks the exact lrb200_graph_describe string, lrb200_graph_num_stages and the kernels one lrb200_graph_execute of N
samples launches.  The table covers every rewrite and each fall-through between them (an unsupported tuner shape, the
overlap-save tap limit, a complex constant or complex taps in front of the interpolator, a composed noble-identity tap
count the polyphase kernel lacks, the Hilbert FIR, a general-order IIR)."""
import ctypes

import numpy as np
import pytest

import luaradio_b200 as radio
from luaradio_b200 import _lib
from luaradio_b200.types import ComplexFloat32, Float32

pytestmark = pytest.mark.gpu

N = 100000
C, R = ComplexFloat32, Float32


def mk(cls, args, in_type, rate=1e6):
    b = cls(*args)
    b.get_rate = lambda: rate
    b.differentiate([in_type])
    b.initialize()
    return b


def _rot(rate=1e6):
    return mk(radio.FrequencyTranslatorBlock, (-1e5,), C, rate)


def _lp(taps, in_type, rate=1e6, cutoff=1e5):
    return mk(radio.LowpassFilterBlock, (taps, cutoff), in_type, rate)


def _fir(taps, use_fft, in_type):
    return mk(radio.FIRFilterBlock, (np.hanning(taps + 2)[1:-1].astype(np.float32) / (taps / 2), use_fft), in_type)


def _cbp(taps, rate=1e6):
    return mk(radio.ComplexBandpassFilterBlock, (taps, (5e4, 2e5)), C, rate)


def _down(d, in_type, rate=1e6):
    return mk(radio.DownsamplerBlock, (d,), in_type, rate)


def _audio_tail(rate, taps=128):
    return [_lp(taps, R, rate, 15e3), mk(radio.FMDeemphasisFilterBlock, (75e-6,), R, rate), _down(5, R, rate)]


# name: (blocks, input is real)
CASES = {
    "tuner+discrim": (lambda: [_rot(), _lp(128, C), _down(5, C), mk(radio.FrequencyDiscriminatorBlock, (1.25,), C)], False),
    "tuner": (lambda: [_rot(), _lp(128, C), _down(5, C)], False),
    "tuner-unsupported-shape": (lambda: [_rot(), _lp(200, C), _down(5, C)], False),
    "tuner-unsupported-shape+discrim": (lambda: [_rot(), _lp(200, C), _down(5, C),
                                                 mk(radio.FrequencyDiscriminatorBlock, (1.25,), C)], False),
    "rot+fir": (lambda: [_rot(), _lp(128, C)], False),
    "rot+fir-513": (lambda: [_rot(), _lp(513, C)], False),
    "rot+fir-514": (lambda: [_rot(), _lp(514, C)], False),
    "rot+fir_cccf": (lambda: [_rot(), _cbp(64)], False),
    "rot+fir_cccf+down": (lambda: [_rot(), _cbp(64), _down(5, C)], False),
    "rot+down": (lambda: [_rot(), _down(5, C)], False),
    "interp-real-const": (lambda: [mk(radio.MultiplyConstantBlock, (2.0,), R), mk(radio.UpsamplerBlock, (3,), R),
                                   _lp(64, R, 3e6)], True),
    "interp-real-const+down": (lambda: [mk(radio.MultiplyConstantBlock, (2.0,), C), mk(radio.UpsamplerBlock, (3,), C),
                                        _lp(64, C, 3e6), _down(2, C, 3e6)], False),
    "interp-complex-const": (lambda: [mk(radio.MultiplyConstantBlock, (2.0 + 1.0j,), C), mk(radio.UpsamplerBlock, (3,), C),
                                      _lp(64, C, 3e6)], False),
    "interp-complex-taps": (lambda: [mk(radio.UpsamplerBlock, (3,), C), _cbp(64, 3e6)], False),
    "noble-low-rate": (lambda: _audio_tail(1e5), True),
    "noble-high-rate": (lambda: _audio_tail(1e6), True),
    "noble-no-polyphase-shape": (lambda: _audio_tail(1e5, 100), True),
    "fir+down-direct": (lambda: [_fir(64, False, C), _down(4, C)], False),
    "fir+down-fft": (lambda: [_fir(64, True, C), _down(4, C)], False),
    "hilbert+down": (lambda: [mk(radio.HilbertTransformBlock, (65,), R), _down(4, C)], True),
    "iir1+down-real": (lambda: [mk(radio.SinglepoleLowpassFilterBlock, (1e4,), R), _down(4, R)], True),
    "iir1+down-complex": (lambda: [mk(radio.SinglepoleLowpassFilterBlock, (1e4,), C), _down(4, C)], False),
    "iir-general+down": (lambda: [mk(radio.IIRFilterBlock, ([0.2, 0.3, 0.2], [1.0, -0.5, 0.2]), R), _down(4, R)], True),
}

# name: {fuse: (lrb200_graph_describe, lrb200_graph_num_stages, kernel launches of one execute of N samples)}
EXPECTED = {
    "tuner+discrim": {1: ("tuner+discrim(128,/5)[fused x4]", 1, 3),
                      0: ("rotator | fir_crcf | downsample | discrim", 4, 7)},
    "tuner": {1: ("tuner(128,/5)[fused x3]", 1, 3),
              0: ("rotator | fir_crcf | downsample", 3, 5)},
    "tuner-unsupported-shape": {1: ("rot+fir_crcf[fused x3]", 1, 3),
                                0: ("rotator | fir_crcf | downsample", 3, 5)},
    "tuner-unsupported-shape+discrim": {1: ("rot+fir_crcf[fused x3] | discrim", 2, 5),
                                        0: ("rotator | fir_crcf | downsample | discrim", 4, 7)},
    "rot+fir": {1: ("rot+fir_crcf[fused x2]", 1, 3),
                0: ("rotator | fir_crcf", 2, 4)},
    "rot+fir-513": {1: ("rot+fir_crcf[fused x2]", 1, 3),
                    0: ("rotator | fir_crcf", 2, 4)},
    "rot+fir-514": {1: ("rotator | fir_crcf", 2, 4),
                    0: ("rotator | fir_crcf", 2, 4)},
    "rot+fir_cccf": {1: ("rot+fir_cccf[fused x2]", 1, 3),
                     0: ("rotator | fir_cccf", 2, 4)},
    "rot+fir_cccf+down": {1: ("rot+fir_cccf[fused x3]", 1, 3),
                          0: ("rotator | fir_cccf | downsample", 3, 5)},
    "rot+down": {1: ("rotator | downsample", 2, 2),
                 0: ("rotator | downsample", 2, 2)},
    "interp-real-const": {1: ("mulconst+upsample+fir(64,x3)[fused x3]", 1, 2),
                          0: ("mulconst | upsample | fir_rrrf", 3, 5)},
    "interp-real-const+down": {1: ("mulconst+upsample+fir+down(64,x3/2)[fused x4]", 1, 2),
                               0: ("mulconst | upsample | fir_crcf | downsample", 4, 6)},
    "interp-complex-const": {1: ("mulconst | upsample+fir(64,x3)[fused x2]", 2, 3),
                             0: ("mulconst | upsample | fir_crcf", 3, 5)},
    "interp-complex-taps": {1: ("upsample | fir_cccf", 2, 4),
                            0: ("upsample | fir_cccf", 2, 4)},
    "noble-low-rate": {1: ("fir*iir1_rrrf(133,/5)+pole[fused x3]", 1, 3),
                       0: ("fir_rrrf | iir_rrrf | downsample", 3, 5)},
    "noble-high-rate": {1: ("fir*iir1_rrrf(133,/5)[fused x3] | pole_rrrf", 2, 4),
                        0: ("fir_rrrf | iir_rrrf | downsample", 3, 5)},
    "noble-no-polyphase-shape": {1: ("fir_rrrf | iir_rrrf[fused x2]", 2, 4),
                                 0: ("fir_rrrf | iir_rrrf | downsample", 3, 5)},
    "fir+down-direct": {1: ("fir_crcf[fused x2]", 1, 2),
                        0: ("fir_crcf | downsample", 2, 3)},
    "fir+down-fft": {1: ("fir_crcf[fused x2]", 1, 3),
                     0: ("fir_crcf | downsample", 2, 4)},
    "hilbert+down": {1: ("hilbert | downsample", 2, 4),
                     0: ("hilbert | downsample", 2, 4)},
    "iir1+down-real": {1: ("iir_rrrf[fused x2]", 1, 1),
                       0: ("iir_rrrf | downsample", 2, 2)},
    "iir1+down-complex": {1: ("iir_crcf[fused x2]", 1, 1),
                          0: ("iir_crcf | downsample", 2, 2)},
    "iir-general+down": {1: ("iir_rrrf(general) | downsample", 2, 4),
                         0: ("iir_rrrf(general) | downsample", 2, 4)},
}


def observe(case, fuse):
    lib = _lib.require_device()
    make_blocks, real = CASES[case]
    g = _lib.check_handle(lib.lrb200_graph_create(), "graph")
    try:
        for b in make_blocks():
            _lib.check(lib.lrb200_graph_append(g, b.make_device_handle()), "append")
            b.cleanup()
        _lib.check(lib.lrb200_graph_commit(g, fuse), "commit")
        rng = np.random.default_rng(7)
        x = rng.uniform(-1, 1, N).astype(np.float32)
        if not real:
            x = (x + 1j * rng.uniform(-1, 1, N)).astype(np.complex64)
        y = np.zeros(lib.lrb200_graph_max_output(g, N) * 8, np.uint8)
        no = ctypes.c_size_t()
        c0 = lib.lrb200_launch_count()
        _lib.check(lib.lrb200_graph_execute(g, x.ctypes.data, N, y.ctypes.data, ctypes.byref(no)), "execute")
        launches = lib.lrb200_launch_count() - c0
        return lib.lrb200_graph_describe(g).decode(), lib.lrb200_graph_num_stages(g), launches
    finally:
        lib.lrb200_graph_destroy(g)


@pytest.mark.parametrize("fuse", [1, 0])
@pytest.mark.parametrize("case", list(CASES))
def test_graph_rewrite(case, fuse):
    assert observe(case, fuse) == EXPECTED[case][fuse]


def observe_dag():
    from luaradio_b200.composite import GPUDagBlock
    rate = 220500.0
    top = radio.CompositeBlock()
    demod = radio.WBFMStereoDemodulator()
    top.connect(radio.ArraySource(np.zeros(1024, np.complex64), rate, 1024), demod)
    top.connect(demod, "left", radio.ArraySink(), "in")
    top.connect(demod, "right", radio.ArraySink(), "in")
    top._prepare_to_run()
    top._collapse_gpu_runs(True, 0, True)
    try:
        dags = [c for c in top._chains if isinstance(c, GPUDagBlock)]
        assert len(dags) == 1
        return _lib.load().lrb200_dag_describe(dags[0].dag).decode()
    finally:
        for c in top._chains:
            c.cleanup()


EXPECTED_DAG = ("discrim | hilbert ; fir_cccf ; pll ; delay ; multiplyconjugate_cc ; fir_crcf | c2r ; fir_crcf | c2r ; "
                "add_rr ; subtract_rr ; iir_rrrf ; iir_rrrf")


def test_wbfm_stereo_dag_rewrites():
    assert observe_dag() == EXPECTED_DAG
