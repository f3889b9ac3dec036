"""Time-chunk sharding of a sample stream across GPUs (SURVEY.md 8e).

The hot path has no cross-sample coupling beyond a finite memory: FIR histories, one discriminator
sample and an exponentially decaying IIR state.  So the stream is cut into contiguous chunks on
multiples of `align` input samples (the product of the decimation factors, so every decimator keeps
its phase), rank r > 0 additionally receives the last `halo` input samples of rank r-1's chunk from its
left neighbour (one point-to-point message per step: NCCL send/recv over NVLink on GPUs, gloo in the
CPU tests), runs from a cold state `halo` samples early and drops the outputs that belong to the halo.
There is no other exchange on this path; outputs are disjoint slices.

This module is transport-agnostic host logic (torch.distributed tensors, any backend); the kernels never
see it.  bench.py uses it for the N > 1 runs.
"""
import math


def plan_chunks(total, world, align=25):
    """Contiguous [start, start+count) per rank; every boundary is a multiple of `align`."""
    per = (total // world) // align * align
    if per <= 0:
        raise ValueError("stream too short to shard: total=%d world=%d align=%d" % (total, world, align))
    plan = []
    for r in range(world):
        start = r * per
        count = per if r < world - 1 else total - start
        plan.append((start, count))
    return plan


def chain_halo(fir_taps_by_rate, iir_pole=None, iir_rate_div=1, tol=1e-12, align=25):
    """Input samples of lead-in needed so a cold start is indistinguishable (to `tol`) from the stream.

    fir_taps_by_rate: [(ntaps, rate_divisor)]: a FIR with ntaps at input_rate / rate_divisor needs
    (ntaps - 1) * rate_divisor input samples; a discriminator needs 1 sample at its rate (pass ntaps=2).
    iir_pole: |c| of a single-pole recurrence running at input_rate / iir_rate_div.
    """
    need = 0
    for ntaps, div in fir_taps_by_rate:
        need += (ntaps - 1) * div
    if iir_pole:
        warm = int(math.ceil(math.log(tol) / math.log(abs(iir_pole)))) if abs(iir_pole) < 1 else 0
        need += warm * iir_rate_div
    return int(math.ceil(need / align) * align)


def exchange_halo(dist, chunk, halo_buf, rank, world, halo):
    """Rank r sends the last `halo` samples of `chunk` to r+1 and receives its own halo from r-1 into
    `halo_buf` (both 1-D tensors on the backend's device).  One batched P2P op per neighbour."""
    ops = []
    if rank + 1 < world:
        ops.append(dist.P2POp(dist.isend, chunk[chunk.shape[0] - halo:], rank + 1))
    if rank > 0:
        ops.append(dist.P2POp(dist.irecv, halo_buf, rank - 1))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()


def trim_outputs(n_out_total, lead, total_decimation):
    """Outputs produced from `lead` halo inputs (lead is a multiple of the total decimation) to drop."""
    assert lead % total_decimation == 0
    skip = lead // total_decimation
    return skip, n_out_total - skip


def dag_shard_step(dist, lib, dag, dx, halo, n, start, dy, n_out, rank, world, device="cpu", times=None):
    """One step of a sharded device DAG (lrb200_dag_shard_*, include/lrb200.h) on every rank: dx -> [halo | n] input
    samples on this rank's device, chunk starting at `start`; dy / n_out as lrb200_dag_shard_end takes them (ctypes
    arrays).  Returns 1 when this rank's PLL ran again, else 0.

    1. every rank begins: the nodes that are not behind a PLL run, and each PLL's loop from its speculated start;
    2. the records (a few dozen bytes each) are all-gathered;
    3. k = the first rank whose start its left neighbour's record does not accept;
    4. ranks below k end with the gathered records;
    5. from k on, each rank ends with the final records of the ranks to its left, received from its left neighbour, and
       passes them on with its own: a rank that ran again moves its end state, so its right neighbour is tested again.
    A step with no miss costs the one all-gather.  Records travel as float64 tensors on `device` (the backend's).  A dict
    `times` receives the seconds of begin, of the exchange (begin's return to end's call) and of end."""
    import ctypes
    import time
    import torch
    t0 = time.perf_counter()
    nb = lib.lrb200_dag_shard_record_bytes(dag)
    rec = (ctypes.c_double * max(1, nb // 8))()
    ptr = lambda a: ctypes.cast(a, ctypes.c_void_p)
    rc = lib.lrb200_dag_shard_begin(dag, dx, halo, n, start, dy, n_out, ptr(rec), nb)
    if rc != 0:
        raise RuntimeError("dag_shard_begin: rc %d" % rc)
    t1 = time.perf_counter()
    if times is not None:
        times.update(begin=t1 - t0, exchange=0.0, end=0.0)
    if nb == 0:
        return 0
    m = nb // 8
    mine = torch.tensor(list(rec)[:m], dtype=torch.float64, device=device)
    gathered = [torch.empty(m, dtype=torch.float64, device=device) for _ in range(world)]
    dist.all_gather(gathered, mine)
    recs = [g.cpu().numpy() for g in gathered]

    def carr(rows):
        flat = [float(v) for r in rows for v in r]
        return (ctypes.c_double * max(1, len(flat)))(*flat)

    k = world
    for j in range(1, world):
        a = lib.lrb200_dag_shard_accepts(dag, ptr(carr([recs[j - 1]])), ptr(carr([recs[j]])), nb)
        if a < 0:
            raise RuntimeError("dag_shard_accepts failed")
        if a == 0:
            k = j
            break
    lefts = recs[:rank]
    if rank > k:
        buf = torch.empty(rank * m, dtype=torch.float64, device=device)
        dist.recv(buf, rank - 1)
        flat = buf.cpu().numpy()
        lefts = [flat[i * m:(i + 1) * m] for i in range(rank)]
    out = (ctypes.c_double * m)()
    t2 = time.perf_counter()
    rc = lib.lrb200_dag_shard_end(dag, ptr(carr(lefts)), rank, dy, n_out, ptr(out), nb)
    if times is not None:
        times.update(exchange=t2 - t1, end=time.perf_counter() - t2)
    if rc < 0:
        raise RuntimeError("dag_shard_end: rc %d" % rc)
    if rank >= k and rank + 1 < world:
        final = [list(r) for r in lefts] + [list(out)]
        dist.send(torch.tensor([v for r in final for v in r], dtype=torch.float64, device=device), rank + 1)
    return rc
