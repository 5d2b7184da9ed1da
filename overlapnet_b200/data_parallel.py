"""The ranks of a data-parallel training run (overlapnet_b200.training, DESIGN.md section 6).

One process per GPU, torch.distributed's default group: NCCL between GPUs, gloo in the CPU tests and for two
processes sharing one GPU.  A batch of n pairs is cut into contiguous shares in rank order
(``search.shard_range``); rank r computes the gradients of its n_r pairs, the ranks all-gather them, and every
rank applies g = sum_r (n_r / n) g_r (``Engine.adagrad_step_sum``).  The losses are means over a batch's pairs,
so that sum is the gradient of the whole batch up to the order of the float32 sums, and every rank ends a step
with the same weights and accumulators bit for bit.
"""
import collections

import numpy as np
import torch
import torch.distributed as dist

from .search import shard_range


def default_group():
  """A DataParallel over the initialised default process group when it has more than one rank, else None."""
  if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
    return DataParallel()
  return None


def shares(n, world):
  """The contiguous [lo, hi) share of each rank of n pairs, and each rank's weight n_r / n (0 for an empty
  share)."""
  bounds = [shard_range(n, r, world) for r in range(world)]
  return bounds, [(hi - lo) / float(n) for lo, hi in bounds]


def chunk_plan(n, n_chunks, world, rank):
  """A batch of n pairs cut into n_chunks contiguous chunks (``shares(n, n_chunks)``), of which each rank trains a
  contiguous range of chunks (``shares(n_chunks, world)``; n_chunks >= world).  Returns the chunk bounds, the chunk
  weights n_k / n, ``rank``'s chunk range (c0, c1) and the pairs [a, b) of the batch it covers."""
  bounds, weights = shares(n, n_chunks)
  c0, c1 = shard_range(n_chunks, rank, world)
  return bounds, weights, (c0, c1), (bounds[c0][0], bounds[c1 - 1][1])


StepPlan = collections.namedtuple('StepPlan', 'lo hi offsets weights counts')


def step_plan(n, world, rank, gradient_chunks=None):
  """What ``rank`` of ``world`` trains in a step on a batch of n pairs: its pairs [lo, hi) of the batch; with
  gradient_chunks K the offsets of its chunks within them, relative to lo (None without chunks); the weights of the
  parts the Adagrad step sums, the chunks' n_k / n or the ranks' n_r / n; and how many of those parts each rank
  computes, in rank order (its chunk count, or 1)."""
  if gradient_chunks is None:
    bounds, weights = shares(n, world)
    return StepPlan(bounds[rank][0], bounds[rank][1], None, weights, [1] * world)
  bounds, weights, (c0, c1), (lo, hi) = chunk_plan(n, gradient_chunks, world, rank)
  offsets = [bounds[c][0] - lo for c in range(c0, c1)] + [hi - lo]
  return StepPlan(lo, hi, offsets, weights, [d1 - d0 for d0, d1 in shares(gradient_chunks, world)[0]])


def chunk_rows(n_chunks, world):
  """The most chunks one rank trains, ceil(n_chunks / world): the rows each rank adds to the all-gathered parts."""
  return -(-n_chunks // world)


class DataParallel:
  """Rank, world size and the collectives of the training loop.  NCCL moves device tensors; on gloo they are
  staged through host memory."""

  def __init__(self):
    self.rank = dist.get_rank()
    self.world = dist.get_world_size()
    self.nccl = dist.get_backend() == 'nccl'
    self.device = torch.device('cuda', torch.cuda.current_device()) if self.nccl else torch.device('cpu')

  def broadcast(self, obj):
    """Rank 0's ``obj`` on every rank (other ranks pass anything, e.g. None)."""
    box = [obj if self.rank == 0 else None]
    dist.broadcast_object_list(box, src=0, device=self.device if self.nccl else None)
    return box[0]

  def gather_flat(self, flat, out):
    """out[r] = rank r's ``flat`` ([n] float32 on the training device; out [world, n] there)."""
    if self.nccl:
      dist.all_gather_into_tensor(out, flat)
      return out
    host = flat.cpu()
    parts = [torch.empty_like(host) for _ in range(self.world)]
    dist.all_gather(parts, host)
    for r, p in enumerate(parts):
      out[r].copy_(p)
    return out

  def gather_rows(self, rows, counts):
    """Every rank's ``rows`` (float64 [counts[rank], m] NumPy) stacked in rank order."""
    k = max(counts)
    pad = torch.zeros((k,) + rows.shape[1:], dtype=torch.float64)
    pad[:rows.shape[0]] = torch.from_numpy(np.ascontiguousarray(rows, np.float64))
    pad = pad.to(self.device)
    parts = [torch.empty_like(pad) for _ in range(self.world)]
    dist.all_gather(parts, pad)
    return np.concatenate([p[:c].cpu().numpy() for p, c in zip(parts, counts)])
