"""Time-chunk sharding of device DAGs (lrb200_dag_halo / _seek / _shard_*): one device stands in for N ranks and runs
them in turn, each rank with its own DAG, as luaradio_b200.sharding.dag_shard_step runs them.

  * the concatenated shard outputs of every port equal the single stream within the comparison tests/
    test_gpu_dag_boundary.py uses for that graph (WBFM stereo, AM synchronous, RDS, and the PLL-free fan-out within the
    chain's 2e-6), worlds 2, 3 and 4, PLL modes 0 and 1;
  * rank 0 is lrb200_dag_execute_device bit for bit; locked pilots re-run nothing;
  * a zero stretch across a handoff point, and one starting exactly at it, re-run the shards the CPU model
    (tests/dag_shard_ref.py) predicts, with the PLL's outputs within its tolerances;
  * refusals, and a shard into guard-banded outputs at unaligned offsets."""
import ctypes
import math

import numpy as np
import pytest

from luaradio_b200 import _lib
from tests import dag_shard_ref as S
from tests import pll_ref as P
from tests.test_gpu_bounds import GUARD, SENTINELS, Guarded
from tests.test_gpu_dag_boundary import CASES, cmp_rel, planned_dag, release

pytestmark = pytest.mark.gpu

N = 1 << 22


def make_dag(name, x, mode):
    make = CASES[name][0]
    if name in ("stereo", "rds") and mode == 1:
        if name == "stereo":
            from tests.test_gpu_dag_boundary import stereo_top
            return planned_dag(lambda y: stereo_top(y, parallel_pll=True), x)
        from tests.test_gpu_rds import rds_top
        from tests.test_gpu_dag_boundary import RATE, VECTOR
        return planned_dag(lambda y: rds_top(y, RATE, VECTOR, tuner=True, parallel_pll=True), x)
    return planned_dag(make, x)


class Ranks:
    """`world` DAGs of one topology and the device buffers of their shards."""

    def __init__(self, lib, name, x, world, mode):
        self.lib, self.x, self.world = lib, x, world
        self.tops, self.dags = zip(*[make_dag(name, x, mode) for _ in range(world)])
        d = self.dags[0]
        self.halo = lib.lrb200_dag_halo(d.dag)
        assert self.halo > 0, _lib.last_error()
        self.nb = lib.lrb200_dag_shard_record_bytes(d.dag)
        self.sizes = [p.data_type.dtype.itemsize for p in d.ext_out]
        self.dtypes = [p.data_type.dtype for p in d.ext_out]
        per = (len(x) // world) // self.halo * self.halo
        self.starts = [r * per for r in range(world)]
        self.counts = [per] * (world - 1) + [len(x) - per * (world - 1)]
        self.bufs = []

    def dev(self, nbytes):
        p = self.lib.lrb200_malloc(max(16, nbytes))
        self.bufs.append(p)
        return p

    def run(self, dys=None):
        """All ranks: (outputs per port concatenated, per-rank outputs, re-run flags, records)."""
        lib, x = self.lib, self.x
        recs, pend = [], []
        for r in range(self.world):
            d = self.dags[r].dag
            start, n = self.starts[r], self.counts[r]
            lead = self.halo if start else 0
            seg = np.ascontiguousarray(x[start - lead:start + n]) if start else np.concatenate([np.zeros(self.halo, np.complex64), x[:n]])
            lead = self.halo
            dx = self.dev(seg.nbytes)
            _lib.check(lib.lrb200_memcpy_h2d(dx, seg.ctypes.data, seg.nbytes), "h2d")
            if dys is None or dys[r] is None:
                ys = [self.dev(max(1, lib.lrb200_dag_max_output(d, k, lead + n)) * s) for k, s in enumerate(self.sizes)]
            else:
                ys = dys[r]
            yp = (ctypes.c_void_p * len(ys))(*ys)
            n_out = (ctypes.c_size_t * len(ys))()
            rec = (ctypes.c_double * max(1, self.nb // 8))()
            _lib.check(lib.lrb200_dag_shard_begin(d, dx, lead, n, start, yp, n_out, ctypes.cast(rec, ctypes.c_void_p), self.nb), "shard_begin")
            recs.append(list(rec)[:self.nb // 8])
            pend.append((ys, yp, n_out))
        final, reruns, outs = [], [], [[] for _ in self.sizes]
        for r in range(self.world):
            d = self.dags[r].dag
            ys, yp, n_out = pend[r]
            left = [v for rr in final for v in rr]
            la = (ctypes.c_double * max(1, len(left)))(*left)
            out = (ctypes.c_double * max(1, self.nb // 8))()
            if r and self.nb:
                acc = lib.lrb200_dag_shard_accepts(d, ctypes.cast((ctypes.c_double * len(final[-1]))(*final[-1]), ctypes.c_void_p),
                                                   ctypes.cast((ctypes.c_double * len(recs[r]))(*recs[r]), ctypes.c_void_p), self.nb)
                assert acc in (0, 1)
            rc = lib.lrb200_dag_shard_end(d, ctypes.cast(la, ctypes.c_void_p), r, yp, n_out, ctypes.cast(out, ctypes.c_void_p), self.nb)
            assert rc in (0, 1), _lib.last_error()
            if r and self.nb:
                assert rc == (1 - acc)
            reruns.append(rc)
            final.append(list(out)[:self.nb // 8])
            _lib.check(lib.lrb200_sync(), "sync")
            for k, (y, s) in enumerate(zip(ys, self.sizes)):
                h = np.zeros(n_out[k], self.dtypes[k])
                if n_out[k]:
                    _lib.check(lib.lrb200_memcpy_d2h(h.ctypes.data, y, n_out[k] * s), "d2h")
                outs[k].append(h)
        return [np.concatenate(o) for o in outs], outs, reruns, final

    def close(self):
        for p in self.bufs:
            self.lib.lrb200_free(p)
        for t in self.tops:
            release(t)


def single(lib, name, x, mode, n=None):
    """lrb200_dag_execute_device of x[:n] on a fresh DAG: the single stream."""
    top, dag = make_dag(name, x, mode)
    n = len(x) if n is None else n
    sizes = [p.data_type.dtype.itemsize for p in dag.ext_out]
    dx = lib.lrb200_malloc(n * 8)
    _lib.check(lib.lrb200_memcpy_h2d(dx, np.ascontiguousarray(x[:n]).ctypes.data, n * 8), "h2d")
    ys = [lib.lrb200_malloc(max(1, lib.lrb200_dag_max_output(dag.dag, k, n)) * s) for k, s in enumerate(sizes)]
    n_out = (ctypes.c_size_t * len(ys))()
    _lib.check(lib.lrb200_dag_execute_device(dag.dag, dx, n, (ctypes.c_void_p * len(ys))(*ys), n_out), "execute_device")
    _lib.check(lib.lrb200_sync(), "sync")
    res = []
    for k, (y, s) in enumerate(zip(ys, sizes)):
        h = np.zeros(n_out[k], dag.ext_out[k].data_type.dtype)
        if n_out[k]:
            _lib.check(lib.lrb200_memcpy_d2h(h.ctypes.data, y, n_out[k] * s), "d2h")
        res.append(h)
    lib.lrb200_free(dx)
    for y in ys:
        lib.lrb200_free(y)
    release(top)
    return res


TOPOLOGIES = [("stereo", 0), ("stereo", 1), ("am_synchronous", 0), ("rds", 0), ("rds", 1), ("fanout", 0)]


@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("name,mode", TOPOLOGIES)
def test_shards_equal_the_single_stream(name, mode, world):
    lib = _lib.require_device()
    if name == "rds":
        # the phase corrector's window makes the RDS halo 1.29 Mi samples: 3 x 2^22 leaves 4 shards of 2 halos each
        from tests.test_gpu_dag_boundary import RATE
        from tests.test_gpu_rds import rds_input
        x = rds_input(3 * N, RATE, 33)
    else:
        x = CASES[name][1]()[:N]
    cmp = cmp_rel(2e-6) if name == "fanout" else CASES[name][3]
    ref = single(lib, name, x, mode)
    ranks = Ranks(lib, name, x, world, mode)
    try:
        got, per_rank, reruns, _ = ranks.run()
        print(name, mode, world, "halo", ranks.halo, "record bytes", ranks.nb, "re-runs", reruns)
        assert (ranks.nb == 0) == (name == "fanout")
        for k in range(len(ref)):
            assert got[k].shape == ref[k].shape, "port %d: %d outputs, the stream %d" % (k, len(got[k]), len(ref[k]))
            cmp(got[k], ref[k], "%s world %d mode %d port %d" % (name, world, mode, k))
        # rank 0 is the plain execute, bit for bit
        r0 = single(lib, name, x, mode, ranks.counts[0])
        for k in range(len(ref)):
            assert np.array_equal(per_rank[k][0].view(np.uint8), r0[k].view(np.uint8)), "rank 0 port %d" % k
        # a re-run is allowed here: behind the 18-20 kHz band-pass of a real multiplex a lead-in can land at the edge of
        # the acceptance box (the stereo loop's lead-in margin on pll_ref's pilots does not hold for it); the outputs
        # agree either way.  Locked pilots re-run nothing: test_misses_are_the_models.
        assert reruns[0] == 0
    finally:
        ranks.close()


# ---- misses, against the CPU model ------------------------------------------------------------------------------------
def pll_dag(lib, mode, loop="stereo"):
    """x -> PLL -> MultiplyConjugate(x, pll.out): the PLL reads the DAG input, its consumer needs 1 sample."""
    bw, fmin, fmax, mult, rate = P.LOOPS[loop]
    d = _lib.check_handle(lib.lrb200_dag_create(), "dag")
    pll = _lib.check_handle(lib.lrb200_pll_create(bw, fmin, fmax, mult, rate, _lib.LRB200_DEVICE), "pll")
    _lib.check(lib.lrb200_pll_set_mode(pll, mode), "set_mode")
    assert lib.lrb200_dag_add_block(d, pll, (ctypes.c_int * 1)(-1), 1) == 0
    mix = _lib.check_handle(lib.lrb200_binary_create(b"multiplyconjugate", 1, _lib.LRB200_DEVICE), "mulconj")
    assert lib.lrb200_dag_add_block(d, mix, (ctypes.c_int * 2)(-1, 0), 2) == 1
    _lib.check(lib.lrb200_dag_set_outputs(d, (ctypes.c_int * 3)(4, 0, 1), 3), "set_outputs")
    return d


class PllRanks(Ranks):
    def __init__(self, lib, x, starts, mode):
        self.lib, self.x, self.world = lib, x, len(starts)
        self.tops = []
        self.dags = [type("D", (), {"dag": pll_dag(lib, mode)})() for _ in starts]
        self.halo = lib.lrb200_dag_halo(self.dags[0].dag)
        self.nb = lib.lrb200_dag_shard_record_bytes(self.dags[0].dag)
        self.sizes, self.dtypes = [8, 8, 4], [np.complex64, np.complex64, np.float32]
        self.starts = list(starts)
        self.counts = [b - a for a, b in zip(starts, list(starts[1:]) + [len(x)])]
        self.bufs = []

    def close(self):
        for p in self.bufs:
            self.lib.lrb200_free(p)
        for d in self.dags:
            self.lib.lrb200_dag_destroy(d.dag)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("where", ["locked_clean", "locked_noisy", "across", "at_handoff"])
def test_misses_are_the_models(mode, where):
    lib = _lib.require_device()
    lp = P.loop("stereo")
    x, starts = S.long_shards(lp, "clean" if where == "locked_clean" else "noisy")
    n = len(x)
    need = 1                                             # MultiplyConjugate: no memory, one sample
    h = starts[1] - need
    # every handoff range and every shard's call is 2 L or longer: in mode 1 they run the chunk-parallel form
    assert all(b - a >= 2 * lp.L for a, b in zip(starts, starts[1:] + [n]))
    y = S.zero_stretch(x, h - lp.W - 100, h + 5000) if where == "across" else S.zero_stretch(x, h, h + 3 * lp.W) if where == "at_handoff" else x
    ranks = PllRanks(lib, y, starts, mode)
    assert ranks.halo == S.round_halo(S.halo_need(lp, need), 1) and ranks.nb == 8 * S.REC
    try:
        got, _, reruns, _ = ranks.run()
    finally:
        ranks.close()
    ref_out, ref_err = S.reference(lp, y)
    _, _, _, model_reruns = S.run_sharded(lp, mode, y, starts, need)
    print(where, mode, "gpu re-runs", reruns, "model", model_reruns)
    assert [bool(r) for r in reruns] == model_reruns
    if where == "across":
        assert any(reruns)
    if where.startswith("locked"):
        assert not any(reruns)
    tol = P.out_tol(S.lead_ins(lp, mode, starts, n, need))
    de = float(np.max(np.abs(got[2].astype(np.float64) - ref_err)))
    do = float(np.max(np.abs(got[1].astype(np.complex128) - ref_out)))
    print("  err %.3g (tol %.3g), out %.3g (tol %.3g)" % (de, P.ERR_TOL, do, tol))
    assert de <= P.ERR_TOL and do <= tol


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_refusals():
    lib = _lib.require_device()
    d = _lib.check_handle(lib.lrb200_dag_create(), "dag")
    agc = _lib.check_handle(lib.lrb200_agc_create(-20.0, -70.0, 0.01, 0.001, 48000.0, 1, _lib.LRB200_DEVICE), "agc")
    assert lib.lrb200_dag_add_block(d, agc, (ctypes.c_int * 1)(-1), 1) == 0
    _lib.check(lib.lrb200_dag_set_outputs(d, (ctypes.c_int * 1)(0), 1), "set_outputs")
    assert lib.lrb200_dag_halo(d) < 0 and "agc" in _lib.last_error(), _lib.last_error()
    lib.lrb200_dag_destroy(d)

    d = pll_dag(lib, 1)
    halo, nb = lib.lrb200_dag_halo(d), lib.lrb200_dag_shard_record_bytes(d)
    n = 4 * halo
    dx = lib.lrb200_malloc((halo + n) * 8)
    lib.lrb200_memset(dx, 0, (halo + n) * 8)
    ys = [lib.lrb200_malloc((halo + n) * 8) for _ in range(3)]
    yp = (ctypes.c_void_p * 3)(*ys)
    n_out = (ctypes.c_size_t * 3)()
    rec = (ctypes.c_double * (nb // 8))()
    rp = ctypes.cast(rec, ctypes.c_void_p)

    def fails(rc, words):
        assert rc < 0 and words in _lib.last_error(), _lib.last_error()
    try:
        fails(lib.lrb200_dag_shard_end(d, rp, 0, yp, n_out, rp, nb), "without shard_begin")
        fails(lib.lrb200_dag_shard_begin(d, dx, halo, n, halo - 4, yp, n_out, rp, nb), "inside the halo")
        fails(lib.lrb200_dag_shard_begin(d, dx, halo, n, 2 * halo, yp, n_out, rp, nb + 8), "bytes")
        fails(lib.lrb200_dag_shard_accepts(d, rp, rp, nb - 8), "bytes")
        _lib.check(lib.lrb200_dag_set_superchunk(d, 1 << 16), "superchunk")
        fails(lib.lrb200_dag_shard_begin(d, dx, halo, n, 2 * halo, yp, n_out, rp, nb), "super-chunk")
        _lib.check(lib.lrb200_dag_set_superchunk(d, 0), "superchunk 0")
        _lib.check(lib.lrb200_dag_shard_begin(d, dx, halo, n, 2 * halo, yp, n_out, rp, nb), "begin")
    finally:
        lib.lrb200_free(dx)
        for y in ys:
            lib.lrb200_free(y)
        lib.lrb200_dag_destroy(d)
    # a period of 5 (the stereo DAG's tuner): misaligned start and halo
    x = CASES["stereo"][1]()[:1 << 20]
    top, dag = planned_dag(CASES["stereo"][0], x)
    try:
        h = lib.lrb200_dag_halo(dag.dag)
        assert h > 0 and h % 20 == 0
        nb = lib.lrb200_dag_shard_record_bytes(dag.dag)
        rec = (ctypes.c_double * (nb // 8))()
        dx = lib.lrb200_malloc((h + 1000) * 8)
        ys = [lib.lrb200_malloc((h + 1000) * 4) for _ in range(2)]
        yp = (ctypes.c_void_p * 2)(*ys)
        n_out = (ctypes.c_size_t * 2)()
        fails(lib.lrb200_dag_shard_begin(dag.dag, dx, h, 1000, 2 * h + 1, yp, n_out, ctypes.cast(rec, ctypes.c_void_p), nb), "multiples")
        fails(lib.lrb200_dag_shard_begin(dag.dag, dx, h - 1, 1000, 2 * h, yp, n_out, ctypes.cast(rec, ctypes.c_void_p), nb), "multiples")
        lib.lrb200_free(dx)
        for y in ys:
            lib.lrb200_free(y)
    finally:
        release(top)


def iir_memory(block, rate):
    """IirBlock::memory_in of a single-pole block: its float32 pole's decay to 1e-12, plus its feed-forward taps."""
    b, a = block._design(rate)
    c = float(np.float32(-float(np.float32(a[1])) / float(np.float32(a[0]))))
    return int(math.ceil(math.log(1e-12) / math.log(abs(c)))) + 1 + len(b)


def need(need_out, mem, down=1):
    """The need at a node's input: ceil(need at its output * down) + its memory + 1."""
    return math.ceil(need_out * down) + mem + 1


def rounded(h, period):
    q = 4 * period
    return -(-h // q) * q


def halo_stereo():
    """tuner+discrim (128 taps, /5: 127 + 5) and Hilbert (129) in one graph node -> [bandpass (129) -> PLL | delay (129)]
    -> mixer -> [lowpass (128) -> c2r] x 2 -> add / subtract -> de-emphasis: the ports."""
    import luaradio_b200 as radio
    W = P.loop("stereo").W
    deemph = need(0, iir_memory(radio.FMDeemphasisFilterBlock(75e-6), 220500.0))
    addsub = need(deemph, 0)
    lowpass_c2r = need(need(addsub, 0), 127)
    mixer = need(lowpass_c2r, 0)
    pll = mixer + W + 1
    bandpass, delay = need(pll, 128), need(max(mixer, lowpass_c2r), 129)
    graph0 = need(need(max(bandpass, delay), 128), 127 + 5, 5)
    return rounded(graph0, 5)


def halo_am_synchronous():
    """bandpass (129) -> [PLL | mixer] -> [c2r -> single-pole high-pass (100 Hz) -> lowpass (128)]: the port."""
    import luaradio_b200 as radio
    W = P.loop("am_sync").W
    tail = need(need(need(0, 127), iir_memory(radio.SinglepoleHighpassFilterBlock(100.0), 48000.0)), 0)
    mixer = need(tail, 0)
    pll = mixer + W + 1
    return rounded(need(max(pll, mixer), 128), 1)


def halo_rds():
    """As the stereo front end, then mixer -> [lowpass (128) -> RRC (101)] (a port) -> phase corrector (8000 x 32, a
    port) -> c2r (a port)."""
    W = P.loop("rds").W
    c2r = need(0, 0)
    corr = need(c2r, 8000 * 32)
    graph = need(need(corr, 100), 127)
    mixer = need(graph, 0)
    pll = mixer + W + 1
    bandpass, delay = need(pll, 128), need(mixer, 129)
    graph0 = need(need(max(bandpass, delay), 128), 127 + 5, 5)
    return rounded(graph0, 5)


@pytest.mark.parametrize("name,count", [("stereo", halo_stereo), ("am_synchronous", halo_am_synchronous), ("rds", halo_rds)])
def test_halo_by_hand(name, count):
    """lrb200_dag_halo of the receivers' DAGs equals a count by hand from their blocks' memories, rates and the PLL's
    lead-in (Dag::plan walks the same rule back from the ports)."""
    lib = _lib.require_device()
    x = CASES[name][1]()[:1 << 16]
    top, dag = planned_dag(CASES[name][0], x)
    try:
        print(name, lib.lrb200_dag_describe(dag.dag).decode())
        assert lib.lrb200_dag_halo(dag.dag) == count()
    finally:
        release(top)


def test_guarded_outputs_at_unaligned_offsets():
    lib = _lib.require_device()
    name = "stereo"
    x = CASES[name][1]()[:1 << 21]
    ranks = Ranks(lib, name, x, 2, 1)
    try:
        n = ranks.counts[1]
        maxo = [lib.lrb200_dag_max_output(ranks.dags[1].dag, k, ranks.halo + n) for k in range(2)]
        obs = [Guarded(lib, m * 4 + 32) for m in maxo]
        sentinel = np.array([SENTINELS[0]], "<u4").view(np.uint8)
        imgs = []
        for b in obs:
            imgs.append(np.resize(sentinel, b.size))
            b.load(imgs[-1])
        offs = [4, 12]
        plain = Ranks(lib, name, x, 2, 1)
        try:
            ref, _, _, _ = plain.run()
        finally:
            plain.close()
        got, per_rank, _, _ = ranks.run(dys=[None, [b.ptr + GUARD + o for b, o in zip(obs, offs)]])
        for k, (b, o) in enumerate(zip(obs, offs)):
            host = b.read()
            nk = len(per_rank[k][1])
            assert np.array_equal(host[:GUARD + o], imgs[k][:GUARD + o]), "port %d: written before y" % k
            assert np.array_equal(host[GUARD + o + 4 * nk:], imgs[k][GUARD + o + 4 * nk:]), "port %d: written past y + n_out" % k
            assert np.array_equal(got[k], ref[k])
        for b in obs:
            b.free()
    finally:
        ranks.close()
