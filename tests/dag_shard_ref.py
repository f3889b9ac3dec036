"""Model of the PLL handoff of a sharded device DAG (graph.cu, Dag::shard_begin / shard_accepts / shard_end; pll.cu,
PllBlock::shard_*), on one PLL whose consumers need `need` samples of left context, built on tests/pll_ref.py's Model.

A stream x (the PLL's input) is cut at starts s_0 = 0 < s_1 < ... ; shard r >= 1 holds x[s_r - halo, s_r + n_r) with
halo >= need + W.  Its handoff point is h_r = s_r - need: from h_r on, the PLL's outputs reach the shard's kept outputs.

  * begin, shard 0: the call over [0, s_1), and the loop state at h_1 (the record's end state; its sum of dP is the
    multiplied phase there, from the reset phase 0).  The GPU runs it as one call and replays the state at h_1 from the
    start of the chunk that holds it (pll_probe_kernel); the model runs two calls split at h_1.  In mode 1 their chunk
    layouts differ, so shard 0's err and out agree with the GPU's within the chunk-parallel tolerances, not bit for bit.
  * begin, shard r >= 1: the speculated start (phi, freq) at h_r after the chunk-parallel form's lead-in over
    x[h_r - W, h_r) (atan2f of the first sample, the centre frequency); the loop from it over [h_r, h_{r+1}) -- a call of
    that length, sequential or chunk-parallel -- gives the end state at h_{r+1} and the wrapped sum of dP; it continues
    over [h_{r+1}, end).
  * accept: |wrap(left end phi - spec phi)| <= DPHI and |left end freq - spec freq| <= DFREQ, pll_ref's thresholds.
  * end: a shard whose start is not accepted runs the loop again from the left shard's end state; the record is then the
    new end state and sum.  The VCO output starts at h_r from the base, the left shards' sums of dP folded and wrapped
    once per shard, over the same two calls [h_r, h_{r+1}) and [h_{r+1}, end).  (The GPU's re-run verifies the already
    simulated chunks again against the new start state; the model simulates the range again from it.  Every chunk after
    the first keeps its lead-in either way, and the first starts from the new state in both, so the errors agree.)  A shard that ran again changes its end state, so the next one is tested against the new record.

MUTANTS break one piece each: the base not folded (only the left neighbour's sum), h_r one sample late for the
speculation, the accept test against the first shard's record instead of the left neighbour's, and the corrected record
not forwarded (the shards after a re-run see its begin record)."""
import math

import numpy as np

from tests import pll_ref as P

MUTANTS = ("base_not_folded", "h_off_by_one", "accept_wrong_rank", "no_forward")
REC = 6          # spec phi, spec freq, end phi, end sum dP, end freq, first (the C record of one PLL)


def lead_in(lp, x, h):
    """The speculated (phi, freq) at h: pll_sim_kernel's lead-in over x[h - W, h)."""
    m = P.Model(lp, 0)
    x0 = np.complex64(x[h - lp.W])
    m.phi = float(np.arctan2(np.float32(x0.imag), np.float32(x0.real), dtype=np.float32))
    m.freq = lp.centre
    m._sequential(x[h - lp.W:h])
    return m.phi, m.freq


def run_from(lp, mode, x, phi, phim, freq):
    """(out, err, model) of one call over x from the state (phi, phim, freq)."""
    m = P.Model(lp, mode)
    m.phi, m.phim, m.freq = phi, phim, freq
    out, err = m.process(x)
    return out, err, m


def fold(sums):
    ph = 0.0
    for s in sums:
        ph = ph + s
        ph = ph - P.TWO_PI if ph > P.TWO_PI else ph
        ph = ph + P.TWO_PI if ph < -P.TWO_PI else ph
    return ph


class Shard:
    """One shard's PLL: begin() -> record; accepts(left, own); end(lefts) -> (rerun, out, err) over [h, end)."""

    def __init__(self, lp, mode, x, start, end, need, mutant=None):
        self.lp, self.mode, self.x, self.start, self.stop, self.need, self.mutant = lp, mode, x, start, end, need, mutant
        self.first = start == 0
        self.h = start - need if not self.first else 0
        self.h_next = end - need

    def begin(self):
        lp, x = self.lp, self.x
        if self.first:
            m = P.Model(lp, self.mode)
            o1, e1 = m.process(x[:self.h_next])
            rec = [0.0, 0.0, m.phi, m.phim, m.freq, 1.0]
            o2, e2 = m.process(x[self.h_next:self.stop])
            self.out, self.err = np.concatenate([o1, o2]), np.concatenate([e1, e2])
            self.rec = rec
            return list(rec)
        hs = self.h + 1 if self.mutant == "h_off_by_one" else self.h
        self.spec = lead_in(lp, x, hs)
        self.rec = [self.spec[0], self.spec[1]] + self._loop(*self.spec) + [0.0]
        return list(self.rec)

    def _loop(self, phi, freq):
        _, _, m = run_from(self.lp, self.mode, self.x[self.h:self.h_next], phi, 0.0, freq)
        return [m.phi, m.phim, m.freq]

    def accepts(self, left, own=None):
        own = self.rec if own is None else own
        if own[5]:
            return True
        m = P.Model(self.lp)
        d = abs(float(P.wrap_diff(left[2] - own[0])))
        return d <= m.dphi and abs(left[4] - own[1]) <= m.dfreq

    def end(self, lefts):
        """lefts: the final records of the shards to the left.  (rerun, out, err) over [h, end), and self.rec final."""
        if self.first:
            return False, self.out, self.err
        left = lefts[0] if self.mutant == "accept_wrong_rank" else lefts[-1]
        rerun = not self.accepts(left)
        start = self.spec
        if rerun:
            start = (lefts[-1][2], lefts[-1][4])
            self.rec = self.rec[:2] + self._loop(*start) + [0.0]
        sums = [r[3] for r in lefts]
        base = fold(sums[-1:] if self.mutant == "base_not_folded" else sums)
        # two calls, as the GPU runs [h_r, h_{r+1}) and [h_{r+1}, end): the chunk boundary at h_{r+1} is forced
        o1, e1, m = run_from(self.lp, self.mode, self.x[self.h:self.h_next], start[0], base, start[1])
        o2, e2 = m.process(self.x[self.h_next:self.stop])
        return rerun, np.concatenate([o1, o2]), np.concatenate([e1, e2])


def run_sharded(lp, mode, x, starts, need, mutant=None):
    """The protocol of luaradio_b200.sharding.dag_shard_step over shards starting at `starts` (starts[0] == 0):
    (out, err) over the whole stream from each shard's [start, end), the slices [h_r, end) per shard, and the re-run
    flags."""
    ends = list(starts[1:]) + [len(x)]
    shards = [Shard(lp, mode, x, s, e, need, mutant) for s, e in zip(starts, ends)]
    begun = [sh.begin() for sh in shards]
    final, reruns, pieces = [], [], []
    for r, sh in enumerate(shards):
        lefts = begun[:r] if mutant == "no_forward" else final
        rr, out, err = sh.end(lefts)
        final.append(list(sh.rec))
        reruns.append(rr)
        pieces.append((sh.h, out, err))
    out = np.concatenate([o[s - h:] for (h, o, e), s in zip(pieces, starts)])
    err = np.concatenate([e[s - h:] for (h, o, e), s in zip(pieces, starts)])
    return out, err, pieces, reruns


def reference(lp, x):
    """mode 0 over the whole stream: (out, err)."""
    return P.Model(lp, 0).process(x)


def lead_ins(lp, mode, starts, n, need):
    """The lead-ins of a sharded run (an upper count): one per handoff, and in mode 1 those of each shard's calls."""
    ends = list(starts[1:]) + [n]
    c = len(starts) - 1
    if mode == 1:
        c += sum(P.lead_ins([e - s + need], lp) for s, e in zip(starts, ends))
    return c


def check(lp, mode, x, starts, need, mutant=None):
    """(ok dict, numbers): the sharded run against mode 0 over the whole stream, every kept slice [h_r, end) included."""
    ref_out, ref_err = reference(lp, x)
    out, err, pieces, reruns = run_sharded(lp, mode, x, starts, need, mutant)
    tol = P.out_tol(lead_ins(lp, mode, starts, len(x), need))
    de = do = 0.0
    for h, o, e in pieces:
        de = max(de, float(np.max(np.abs(e.astype(np.float64) - ref_err[h:h + len(e)]))))
        do = max(do, float(np.max(np.abs(o.astype(np.complex128) - ref_out[h:h + len(o)]))))
    assert len(out) == len(x)
    ok = {"err": de <= P.ERR_TOL, "out": do <= tol}
    return ok, {"de": de, "do": do, "tol": tol, "reruns": reruns}


def long_shards(lp, kind="noisy", seed=21, world=3):
    """(x, starts): a pilot cut into `world` shards of 3 L samples (and a tail), so that every handoff range [h_r,
    h_{r+1}) is a call of three chunks in mode 1 -- the chunk-parallel form runs, and a miss re-verifies its chunks."""
    per = 3 * lp.L
    x = P.pilot(lp, world * per + 5000, kind, seed=seed)
    return x, [r * per for r in range(world)]


def zero_stretch(x, a, b):
    y = np.array(x, np.complex64)
    y[a:b] = 0
    return y


def halo_need(lp, need):
    """The PLL's share of a DAG halo: what its consumers need, its lead-in and the one sample of every node."""
    return need + lp.W + 1


# ---- DAG halo arithmetic by hand --------------------------------------------------------------------------------------
def round_halo(need, period):
    q = 4 * period
    return int(math.ceil(math.ceil(need) / q) * q)
