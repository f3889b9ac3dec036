"""luaradio_b200.sharding.dag_shard_step under gloo at world 3, with a fake library driven by the handoff model
(tests/dag_shard_ref.py) in place of lrb200_dag_shard_*: the step's all-gather, accept scan and record forwarding
reproduce the model's run, including a re-run on rank 1 whose corrected record rank 2 receives and is tested against.
Then the re-test step on its own, with scripted records: a miss on rank 1 flips rank 2's accept both ways (rank 2
accepts rank 1's begin record but not the corrected one, and the reverse)."""
import ctypes
import os
import socket

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

from luaradio_b200 import sharding
from tests import dag_shard_ref as S
from tests import pll_ref as P

NEED = 300


def scenario():
    """Shards of 3 L (chunk-parallel handoff ranges) with a zero stretch across rank 1's handoff point: rank 1 re-runs."""
    lp = P.loop("stereo")
    x, starts = S.long_shards(lp)
    h = starts[1] - NEED
    return lp, S.zero_stretch(x, h - lp.W - 100, h + 5000), starts


class FakeLib:
    """lrb200_dag_shard_* over one model shard; records are the C layout (S.REC doubles)."""

    def __init__(self, shard):
        self.sh = shard
        self.nb = 8 * S.REC

    @staticmethod
    def _get(p, k=1):
        return list(np.frombuffer(ctypes.string_at(p, 8 * S.REC * k), np.float64))

    def lrb200_dag_shard_record_bytes(self, dag):
        return self.nb

    def lrb200_dag_shard_begin(self, dag, dx, halo, n, start, dy, n_out, rec, nb):
        r = np.array(self.sh.begin(), np.float64)
        ctypes.memmove(rec, r.ctypes.data, nb)
        return 0

    def lrb200_dag_shard_accepts(self, dag, left, own, nb):
        return int(self.sh.accepts(self._get(left), self._get(own)))

    def lrb200_dag_shard_end(self, dag, lefts, num_left, dy, n_out, out, nb):
        flat = self._get(lefts, num_left) if num_left else []
        rr, o, e = self.sh.end([flat[i * S.REC:(i + 1) * S.REC] for i in range(num_left)])
        self.result = (o, e)
        r = np.array(self.sh.rec, np.float64)
        ctypes.memmove(out, r.ctypes.data, nb)
        return int(rr)


def _worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    lp, y, starts = scenario()
    ends = starts[1:] + [len(y)]
    lib = FakeLib(S.Shard(lp, 1, y, starts[rank], ends[rank], NEED))
    rc = sharding.dag_shard_step(dist, lib, None, None, 0, 0, starts[rank], None, None, rank, world)
    o, e = lib.result
    h = lib.sh.h
    np.save(os.path.join(out_dir, "o%d.npy" % rank), o[starts[rank] - h:])
    np.save(os.path.join(out_dir, "rc%d.npy" % rank), np.array([rc]))
    dist.barrier()
    dist.destroy_process_group()


def test_world3_step_reproduces_the_model(tmp_path):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_worker, args=(3, port, str(tmp_path)), nprocs=3, join=True)
    lp, y, starts = scenario()
    out, _, _, reruns = S.run_sharded(lp, 1, y, starts, NEED)
    got = np.concatenate([np.load(tmp_path / ("o%d.npy" % r)) for r in range(3)])
    rcs = [int(np.load(tmp_path / ("rc%d.npy" % r))[0]) for r in range(3)]
    assert [bool(r) for r in rcs] == reruns and reruns[1]
    assert np.array_equal(got, out)


# ---- the re-test step on its own: scripted records ---------------------------------------------------------------------
class ScriptedLib:
    """Records {spec phi, spec freq, end phi, sum, end freq, first}; a start is accepted when its spec phi equals the left
    record's end phi.  A shard that misses ends at `corrected` instead of its begin end state."""

    def __init__(self, spec, end, corrected, first=False):
        self.rec = [spec, 0.0, end, 0.0, 0.0, 1.0 if first else 0.0]
        self.corrected, self.seen = corrected, None

    def lrb200_dag_shard_record_bytes(self, dag):
        return 8 * S.REC

    def lrb200_dag_shard_begin(self, dag, dx, halo, n, start, dy, n_out, rec, nb):
        ctypes.memmove(rec, np.array(self.rec, np.float64).ctypes.data, nb)
        return 0

    def lrb200_dag_shard_accepts(self, dag, left, own, nb):
        l, o = FakeLib._get(left), FakeLib._get(own)
        return int(o[5] != 0 or o[0] == l[2])

    def lrb200_dag_shard_end(self, dag, lefts, num_left, dy, n_out, out, nb):
        rr = 0
        if num_left:
            left = FakeLib._get(lefts, num_left)[-S.REC:]
            self.seen = left[2]
            if left[2] != self.rec[0]:
                self.rec[2], rr = self.corrected, 1
        ctypes.memmove(out, np.array(self.rec, np.float64).ctypes.data, nb)
        return rr


def _scripted(rank, world, port, out_dir, spec2):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    # rank 0 ends at 1; rank 1 speculates 9 (a miss), ends at 2 from it and at 3 once run again from 1
    lib = [ScriptedLib(0.0, 1.0, 1.0, first=True), ScriptedLib(9.0, 2.0, 3.0), ScriptedLib(spec2, 5.0, 6.0)][rank]
    rc = sharding.dag_shard_step(dist, lib, None, None, 0, 0, rank, None, None, rank, world)
    np.save(os.path.join(out_dir, "s%d.npy" % rank), np.array([rc, -1.0 if lib.seen is None else lib.seen]))
    dist.barrier()
    dist.destroy_process_group()


def _run_scripted(tmp_path, spec2):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_scripted, args=(3, port, str(tmp_path), spec2), nprocs=3, join=True)
    return [tuple(np.load(tmp_path / ("s%d.npy" % r))) for r in range(3)]


def test_rank2_accepts_the_begin_record_but_not_the_corrected_one(tmp_path):
    """Rank 2's start matches rank 1's begin record (2) and not its corrected one (3): it must run again."""
    res = _run_scripted(tmp_path, 2.0)
    assert res[1] == (1, 1.0) and res[2] == (1, 3.0), res


def test_rank2_rejects_the_begin_record_but_accepts_the_corrected_one(tmp_path):
    """Rank 2's start matches only rank 1's corrected record (3): it must not run again."""
    res = _run_scripted(tmp_path, 3.0)
    assert res[1] == (1, 1.0) and res[2] == (0, 3.0), res
