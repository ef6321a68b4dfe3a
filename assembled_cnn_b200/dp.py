"""Data-parallel plumbing of the training step (the reference's MirroredStrategy,
official/utils/misc/distribution_utils.py:24-76), shared by the CUDA Trainer and
by the CPU (gloo) tests so that both exercise the same code:

  * gradients: SUM over replicas of the flat fp32 gradient buffer, bucketed in reverse layer order
    so that a bucket is all-reduced (NCCL, asynchronously) while the backward of the earlier layers
    still runs; the 1/N of the average is folded into the SGD kernel's grad_scale;
  * BN moving statistics: mirrored variables whose per-replica updates are MEAN-aggregated.

Everything here works on flat tensors + a Plan; no CUDA-specific calls.
"""
from __future__ import annotations

import torch
import torch.distributed as dist



# bucket boundaries as fractions of the flat buffer, from its end: the early layers hold few parameters
# but most of the backward's time, so the LAST bucket (the only one whose all-reduce cannot overlap
# any compute) is kept small
DEFAULT_CUTS = (0.75, 0.5, 0.25, 0.08, 0.02)


def grad_buckets(plan, cuts=DEFAULT_CUTS):
    """[(lo, hi, ready)]: contiguous element ranges of the flat gradient buffer, LAST layers first,
    and the index of the backward op after which every gradient of the range (and of all later
    ranges) is final.  Parameters are laid out in creation (= forward) order, the backward produces
    their gradients roughly from the end of the buffer to its beginning."""
    done_at = plan.grad_done_at()
    total = plan.param_elems
    offsets = sorted(p.offset for p in plan.params.values())
    bounds = [total]
    for frac in cuts:
        off = next((o for o in offsets if o >= int(total * frac)), 0)   # snap to a parameter boundary
        if 0 < off < bounds[-1]:
            bounds.append(off)
    bounds.append(0)
    out, run_max = [], -1
    for hi, lo in zip(bounds[:-1], bounds[1:]):
        ready = max([done_at.get(n, -1) for n, p in plan.params.items() if lo <= p.offset < hi]
                    or [-1])
        run_max = max(run_max, ready)       # ops are issued in order
        out.append((lo, hi, run_max))
    return out


def backward_segments(plan, buckets):
    """One (start, stop) slice of plan.backward per bucket: after segment k has run, bucket k may be
    reduced.  The last segment extends to the end of the backward."""
    segs, start = [], 0
    for k, (_, _, ready) in enumerate(buckets):
        stop = len(plan.backward) if k == len(buckets) - 1 else ready + 1
        segs.append((start, max(stop, start)))
        start = max(stop, start)
    return segs


def schedule(buckets, segments):
    """The order of work of one data-parallel forward + backward: ('run', a, b) = backward ops
    [a, b) (the forward precedes the first one), ('reduce', lo, hi) = all-reduce that bucket."""
    for (lo, hi, _), (a, b) in zip(buckets, segments):
        yield ("run", a, b)
        yield ("reduce", lo, hi)


def all_reduce_bucket(flat: torch.Tensor, lo: int, hi: int, async_op: bool = False):
    """SUM of flat[lo:hi] over the replicas, in place."""
    return dist.all_reduce(flat[lo:hi], async_op=async_op)


def average_moving_statistics(state: torch.Tensor, world: int):
    """Mean aggregation of the mirrored BN moving statistics."""
    if world > 1:
        dist.all_reduce(state)
        state.mul_(1.0 / world)
