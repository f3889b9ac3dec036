"""The PLL handoff model of a sharded device DAG (tests/dag_shard_ref.py) against the sequential PLL over the whole
stream: the shards' err / out within pll_ref's tolerances of the chunk-parallel form, no re-run on locked pilots, at
least one where a zero stretch straddles a handoff point, and each mutant caught.  (The DAG halo of
the receivers' topologies is checked against a count by hand in tests/test_gpu_dag_shard.py, where lrb200_dag_halo
runs.)"""
import numpy as np
import pytest

from tests import dag_shard_ref as S
from tests import pll_ref as P

NEED = 300          # samples of left context behind the PLL (a mixer and a FIR, say)


@pytest.mark.parametrize("kind", ["clean", "noisy", "offset", "drift"])
@pytest.mark.parametrize("world", [2, 3, 5])
def test_locked_pilots_hand_over_without_a_rerun(kind, world):
    lp = P.loop("stereo")
    x, starts = S.long_shards(lp, kind, world=world)
    ok, nums = S.check(lp, 1, x, starts, NEED)
    print(kind, world, nums)
    assert all(ok.values()), nums
    assert not any(nums["reruns"])


@pytest.mark.parametrize("gap", ["zeros"])        # a noise gap is no miss: the same noise drives both loops together
@pytest.mark.parametrize("mode", [0, 1])
def test_a_gap_across_a_handoff_point_reruns_and_stays_within_tolerance(gap, mode):
    lp = P.loop("stereo")
    x, starts = S.long_shards(lp)                    # handoff ranges of 3 L: mode 1 runs them chunk-parallel
    h = starts[1] - NEED
    y = np.array(x)
    a, b = h - lp.W - 100, h + 5000
    y[a:b] = 0 if gap == "zeros" else P.pilot(lp, b - a, "noise", seed=5)
    ok, nums = S.check(lp, mode, y, starts, NEED)
    print(gap, mode, nums)
    assert all(ok.values()), nums
    assert nums["reruns"] == [False, True, False]


@pytest.mark.parametrize("mutant", S.MUTANTS)
def test_each_mutant_breaks_it(mutant):
    lp = P.loop("stereo")
    x, starts = S.long_shards(lp)
    broken = []
    for y in (x, S.zero_stretch(x, starts[1] - NEED - lp.W - 100, starts[1] - NEED + 5000)):
        ok, nums = S.check(lp, 1, y, starts, NEED, mutant)
        locked = y is x
        broken.append(not all(ok.values()) or (locked and any(nums["reruns"])))
    assert any(broken), mutant
