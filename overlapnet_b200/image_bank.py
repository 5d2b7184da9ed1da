"""Where a training flow keeps its image bank -- the packed input [n, H, W, C] float32 of every distinct scan it
trains on -- and how a step's images reach the device when that bank does not live whole on the device (DESIGN.md
sections 1 and 6).

The flow compares the bank's bytes with the device's free memory minus the working set of its largest step
(``working_set_bytes``).  A bank that fits goes on the device, as it always did.  Under data-parallel training on
one node, a bank that does not fit one GPU but whose 1/world share does is sharded over the ranks' GPUs
(``ShardedImageBank``): each rank holds a contiguous block of rows and maps its peers' blocks.  Otherwise the bank
goes into one page-locked host block (``HostBank``).  With either of these, every step copies only its own distinct
rows into one of two device slots (``StagingRing``) on a copy stream while the previous step computes: from the
host one copy per row, from the shards one gather launch.  The kernels a step runs are those of the device bank,
on the same image values, so every placement trains bit-identical weights.
"""
import collections
import logging
import socket

import numpy as np
import torch
import torch.distributed as dist

from . import data_parallel
from ._cabi import OvnError
from .engine import FEAT_C
from .search import shard_range

logger = logging.getLogger('overlapnet_b200.training')

PLACEMENTS = ('device', 'host', 'sharded')
STAGED = ('host', 'sharded')     # the placements whose steps read their images from a StagingRing's slot
MARGIN_BYTES = 1 << 30   # the CUDA context's own growth, allocator rounding and the small per-step tensors


def image_bytes(eng):
  return eng.H * eng.W * eng.C * 4


def share_pairs(n_pairs, world, gradient_chunks=None):
  """The most pairs of an n_pairs batch that one of ``world`` data-parallel ranks trains in a step
  (data_parallel.step_plan), with or without gradient_chunks K.  A full batch has the largest shares: a shorter one
  only makes some of them smaller."""
  plans = (data_parallel.step_plan(n_pairs, world, r, gradient_chunks) for r in range(world))
  return max(p.hi - p.lo for p in plans)


def parts_bytes(eng, whole_network, world, gradient_chunks=None):
  """Device bytes of the per-chunk gradients of a step with gradient_chunks K: world ceil(K / world) all-gathered
  parts, and with more than one rank ceil(K / world) local ones; 0 without chunks."""
  if gradient_chunks is None:
    return 0
  m = data_parallel.chunk_rows(gradient_chunks, world)
  return (world * m + (m if world > 1 else 0)) * eng.gradient_size(whole_network) * 4


def working_set_bytes(eng, b_share, whole_network, gathered, features, parts=0):
  """Device bytes a training run needs besides its image bank, from the shapes of its largest step of
  ``b_share`` pairs: the handle's training buffers (Engine.train_workspace_bytes: for the whole network the leg
  activations of 2 b_share images, the split-K partials, the head buffers), the staging ring (two slots of
  2 b_share images), ``gathered`` images of a step's gathered batch (yaw augmentation), ``features`` feature volumes
  (the validation feature bank, the frozen leg's bank), ``parts`` bytes of per-chunk gradients (parts_bytes) and
  MARGIN_BYTES."""
  return (eng.train_workspace_bytes(b_share, whole_network) + 2 * 2 * b_share * image_bytes(eng)
          + gathered * image_bytes(eng) + features * eng.Wf * FEAT_C * 4 + int(parts) + MARGIN_BYTES)


def choose_placement(bank_bytes, free_bytes, working_set):
  """'device' when the bank fits into the free device memory left after the working set, else 'host'; and that
  budget (free_bytes - working_set)."""
  budget = int(free_bytes) - int(working_set)
  return ('device' if int(bank_bytes) <= budget else 'host'), budget


def choose_rank_placement(bank_bytes, shard_bytes, budgets, hosts):
  """The placement of the data-parallel ranks with device budgets ``budgets`` (free memory minus working set, one
  per rank) on hosts ``hosts``, and the smallest budget, which decides for every rank: 'device' when the bank fits
  it; else 'sharded' when the largest shard (``shard_bytes``, ceil(n / world) images) fits it and every rank is on
  one host; else 'host'.  One rank is never sharded."""
  budget = min(int(b) for b in budgets)
  if int(bank_bytes) <= budget:
    return 'device', budget
  if len(budgets) > 1 and len(set(hosts)) == 1 and int(shard_bytes) <= budget:
    return 'sharded', budget
  return 'host', budget


def free_device_bytes(eng):
  return int(torch.cuda.mem_get_info(eng.device)[0])


def shard_plan(n, world):
  """The first bank row of each rank's shard, and n: rank r holds rows [first[r], first[r + 1]) (search.shard_range:
  contiguous blocks in rank order that differ by at most one row)."""
  return [shard_range(n, r, world)[0] for r in range(world)] + [int(n)]


def shard_of(first, row):
  """(rank, local row) of bank row ``row`` under the shard plan ``first``."""
  r = int(np.searchsorted(first, row, side='right')) - 1
  return r, int(row) - first[r]


def plan_rows(*row_lists):
  """The distinct rows of a step's row lists, in order of first appearance (the lists in the order given), and the
  local index of every entry of every list among them: rows[local[k][i]] == row_lists[k][i].  Returns (rows int64,
  [local int32 per list])."""
  parts = [np.asarray(r, np.int64).reshape(-1) for r in row_lists]
  cat = np.concatenate(parts) if parts else np.zeros(0, np.int64)
  uniq, first, inverse = np.unique(cat, return_index=True, return_inverse=True)
  order = np.argsort(first, kind='stable')
  rank = np.empty(order.size, np.int64)
  rank[order] = np.arange(order.size)
  local = rank[inverse.reshape(-1)].astype(np.int32)
  out, o = [], 0
  for p in parts:
    out.append(local[o:o + p.size])
    o += p.size
  return uniq[order], out


def bank_rows(keys):
  """{key: row} of the distinct (dir, scan) keys: by directory, then by scan name."""
  rows = {}
  for d in sorted({k[0] for k in keys}):
    for name in sorted(k[1] for k in keys if k[0] == d):
      rows[(d, name)] = len(rows)
  return rows


def fill_image_bank(infer, rows, bank, chunk=256):
  """bank[rows[key]] = the packed network input of each key, through Infer's cue loader (one sequence directory
  at a time, ``chunk`` scans per load).  ``bank``: a device tensor or a host NumPy array [n, H, W, C]."""
  keys = list(rows)
  for d in sorted({k[0] for k in keys}):
    names = sorted(k[1] for k in keys if k[0] == d)
    infer.seq = d
    for s in range(0, len(names), chunk):
      x = infer._prepare_inputs(names[s:s + chunk])
      r0 = rows[(d, names[s])]
      if isinstance(bank, np.ndarray):
        bank[r0:r0 + len(x)] = x
      else:
        bank[r0:r0 + len(x)] = torch.from_numpy(x).to(bank.device)


def load_image_bank(infer, keys, chunk=256):
  """Packed network inputs of the distinct (dir, scan) keys, through Infer's cue loader (one sequence
  directory at a time), in one device tensor [n, H, W, C].  Returns it and {key: row}."""
  eng = infer._engine
  rows = bank_rows(keys)
  bank = torch.empty((len(rows), eng.H, eng.W, eng.C), dtype=torch.float32, device=eng.device)
  fill_image_bank(infer, rows, bank, chunk)
  return bank, rows


class HostBank:
  """The images [n, H, W, C] float32 in one page-locked host block, pinned through the handle
  (Engine.host_register), which releases it on close() or when the handle closes."""

  def __init__(self, eng, n):
    self.eng = eng
    shape = (int(n), eng.H, eng.W, eng.C)
    nbytes = int(np.prod(shape)) * 4
    try:
      self.images = np.empty(shape, np.float32)
      eng.host_register(self.images)
    except Exception as e:
      raise Exception('image bank in host memory: could not pin %d bytes (%.2f GB) for %d images of %d x %d x %d '
                      'float32: %s' % (nbytes, nbytes / 1e9, shape[0], shape[1], shape[2], shape[3], e)) from e

  @property
  def nbytes(self):
    return self.images.nbytes

  def stage(self, rows, out):
    """out[i] = images[rows[i]], one asynchronous copy per row on the current stream (Engine.stage_rows)."""
    self.eng.stage_rows(self.images, rows, out)

  def close(self):
    if self.images is not None:
      self.eng.host_unregister(self.images)
      self.images = None


class ShardOpenError(Exception):
  """A sharded image bank could not be set up on some rank (every rank raises it, with every rank's reason)."""


class ShardedImageBank:
  """The images [n, H, W, C] float32 of a bank sharded over the data-parallel ranks of one node: rank r holds rows
  [first[r], first[r + 1]) (shard_plan) in a shard of its own device memory (Engine.shard_create), filled through
  the cue loader with only its own scans, and maps every other rank's shard through the CUDA IPC handles the
  ranks exchange over the default process group (Engine.shard_open).  A process cannot map its own allocation, so
  a rank reads its own shard through its own pointer.  With one process (``dp`` None) the bank is one own shard.

  Construction is collective: every rank builds its shard, and if any rank cannot allocate its shard or open a
  peer's, every rank closes what it made and raises ShardOpenError with the reasons.  So is ``close``."""

  def __init__(self, infer, rows, dp):
    self.eng = eng = infer._engine
    self.dp = dp
    world, rank = (1, 0) if dp is None else (dp.world, dp.rank)
    n = len(rows)
    self.first = shard_plan(n, world)
    lo, hi = self.first[rank], self.first[rank + 1]
    self.rank_rows = hi - lo
    self.images, self.own, self.ptrs, self.closed = None, None, [], False
    ipc, err = None, None
    try:
      self.images, self.own, ipc = eng.shard_create(hi - lo)
    except OvnError as e:
      err = 'rank %d could not allocate its shard of %d images (%.1f MB): %s' % (rank, hi - lo,
                                                                                 (hi - lo) * image_bytes(eng) / 1e6, e)
    if err is None:
      fill_image_bank(infer, {k: r - lo for k, r in rows.items() if lo <= r < hi}, self.images)
      torch.cuda.synchronize(eng.device)               # the shard is complete before any peer can read it
    handles = self._all(dict(ipc=ipc, err=err))
    errors = [h['err'] for h in handles if h['err']]
    if not errors:
      for r, h in enumerate(handles):
        if r == rank:
          self.ptrs.append(self.own)
          continue
        try:
          self.ptrs.append(eng.shard_open(h['ipc']))
        except OvnError as e:
          err = 'rank %d could not open the shard of rank %d: %s' % (rank, r, e)
          break
      errors = [e for e in self._all(err) if e]
    if errors:
      self.close()
      raise ShardOpenError('; '.join(errors))

  def _all(self, obj):
    """Every rank's ``obj``, in rank order (one all_gather_object over the default group)."""
    if self.dp is None:
      return [obj]
    out = [None] * self.dp.world
    dist.all_gather_object(out, obj)
    return out

  @property
  def nbytes(self):
    """The device bytes of this rank's shard."""
    return self.rank_rows * image_bytes(self.eng)

  def stage(self, rows, out):
    """out[i] = bank row rows[i], one gather launch on the current stream (Engine.gather_rows)."""
    self.eng.gather_rows(self.ptrs, self.first, rows, out)

  def close(self):
    """Collective: synchronise the device (the ring's copy stream included), unmap every peer's shard, wait for
    every rank to have done so, then free the own shard.  So no shard is freed while a rank may still read it."""
    if self.closed:
      return
    self.closed = True
    torch.cuda.synchronize(self.eng.device)
    for p in self.ptrs:
      if p != self.own:
        self.eng.shard_close(p)
    self.ptrs = []
    if self.dp is not None:
      dist.barrier()
    self.images = None                                 # the view goes before the memory it shows
    if self.own is not None:
      self.eng.shard_close(self.own)
      self.own = None


class StagingRing:
  """Two device slots of ``slot_rows`` images, filled from a HostBank or a ShardedImageBank (``source``) on a copy
  stream of their own.

  ``plan`` takes the row lists of the steps to come, in the order they will run; each step's distinct rows
  (plan_rows) are copied into the next slot (``source.stage``).  ``take`` hands the compute stream the
  oldest filled slot after making it wait for that slot's copy-done event, with the step's local indices;
  ``release`` records the compute-done event of the step that read the slot, and issues the next planned copy into
  it, which waits for that event.  So step k + 1's copies run while step k computes, and a slot is never written
  while a step still reads it."""

  def __init__(self, eng, source, slot_rows, timing=False):
    self.eng, self.source, self.slot_rows = eng, source, int(slot_rows)
    dev = eng.device
    self.slots = [torch.empty((self.slot_rows, eng.H, eng.W, eng.C), dtype=torch.float32, device=dev)
                  for _ in range(2)]
    self.copy_stream = torch.cuda.Stream(device=dev)
    self._copied = [torch.cuda.Event(), torch.cuda.Event()]
    self._computed = [None, None]
    self._queue = collections.deque()                 # planned, not yet issued: (rows, locals)
    self._ready = collections.deque()                 # issued, not yet taken: (slot, locals)
    self._next = 0                                    # the slot the next issue fills
    self._taken = None
    self.step_rows = 0                                # the distinct rows staged for the step taken last
    self.timing = timing
    self.waits = []                                   # with timing: (before, after) events around each wait

  def plan(self, steps):
    """``steps``: for each step to come, a tuple of row lists (plan_rows)."""
    assert not self._queue and not self._ready and self._taken is None, 'the previous plan is not consumed'
    for lists in steps:
      rows, local = plan_rows(*lists)
      assert rows.size <= self.slot_rows, (rows.size, self.slot_rows)
      self._queue.append((rows, local))
    while self._queue and len(self._ready) < 2:
      self._issue()

  def _issue(self):
    rows, local = self._queue.popleft()
    s = self._next
    self._next ^= 1
    with torch.cuda.stream(self.copy_stream):
      if self._computed[s] is not None:
        self.copy_stream.wait_event(self._computed[s])
      self.source.stage(rows, self.slots[s])
      self._copied[s].record(self.copy_stream)
    self._ready.append((s, local, int(rows.size)))

  def take(self):
    """The next step's slot (a device tensor [slot_rows, H, W, C]) and its local indices (int32 device tensors,
    one per row list), ordered after its copies on the current stream."""
    assert self._taken is None and self._ready, 'take without a planned step'
    s, local, self.step_rows = self._ready.popleft()
    idx = [torch.from_numpy(l).to(self.eng.device) for l in local]
    cur = torch.cuda.current_stream(self.eng.device)
    if self.timing:
      before, after = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      before.record(cur)
    cur.wait_event(self._copied[s])
    if self.timing:
      after.record(cur)
      self.waits.append((before, after))
    self._taken = s
    return self.slots[s], idx

  def release(self):
    """The step that took the slot has queued its last read of it."""
    s, self._taken = self._taken, None
    if self._computed[s] is None:
      self._computed[s] = torch.cuda.Event()
    self._computed[s].record(torch.cuda.current_stream(self.eng.device))
    if self._queue:
      self._issue()

  def wait_ms(self):
    """With timing: for each take since the last call, the milliseconds the compute stream waited on the slot's
    copy-done event.  Waits for those events only, not for the device, so copies still in flight on the copy
    stream keep running."""
    out = []
    for before, after in self.waits:
      after.synchronize()
      out.append(before.elapsed_time(after))
    self.waits = []
    return out


def open_bank(infer, keys, image_bank, b_share, whole_network, gathered, features, what, parts=0):
  """The image bank of the distinct (dir, scan) ``keys``: ``image_bank`` None chooses its placement from the free
  device memory and the working set (working_set_bytes; with several data-parallel ranks the smallest budget of any
  rank, choose_rank_placement), 'device', 'host' or 'sharded' forces it.  Returns (placement, the device tensor,
  HostBank or ShardedImageBank, {key: row}).  ``what`` names the bank in the log.  A chosen sharded bank that some
  rank cannot set up falls back to the host bank on every rank; a forced one raises."""
  eng = infer._engine
  if image_bank not in (None,) + PLACEMENTS:
    raise ValueError('image_bank %r: use None, %s' % (image_bank, ' or '.join(repr(p) for p in PLACEMENTS)))
  n = len(set(keys))
  bank_bytes = n * image_bytes(eng)
  dp = data_parallel.default_group()
  world = 1 if dp is None else dp.world
  shard_bytes = -(-n // world) * image_bytes(eng)
  placement = image_bank
  if placement is None:
    ws = working_set_bytes(eng, b_share, whole_network, gathered, features, parts)
    if dp is None:
      placement, budget = choose_placement(bank_bytes, free_device_bytes(eng), ws)
      logger.info('%s: %d scans, %.1f MB; device budget %.1f MB (free memory minus a working set of %.1f MB): '
                  'on the %s', what, n, bank_bytes / 1e6, budget / 1e6, ws / 1e6,
                  'GPU' if placement == 'device' else 'host, pinned')
    else:                      # one collective: every rank's budget and host, so that every rank decides alike
      ranks = [None] * world
      dist.all_gather_object(ranks, (free_device_bytes(eng) - ws, socket.gethostname()))
      placement, budget = choose_rank_placement(bank_bytes, shard_bytes, [b for b, _ in ranks], [h for _, h in ranks])
      logger.info('%s: %d scans, %.1f MB, %.1f MB per shard over %d ranks on %d host(s); device budget %.1f MB (the '
                  'smallest over the ranks of free memory minus a working set of %.1f MB): %s', what, n,
                  bank_bytes / 1e6, shard_bytes / 1e6, world, len(set(h for _, h in ranks)), budget / 1e6, ws / 1e6,
                  {'device': 'on every GPU', 'sharded': "sharded over the ranks' GPUs",
                   'host': 'on the host, pinned'}[placement])
  if placement == 'device':
    images, rows = load_image_bank(infer, keys)
    return placement, images, rows
  rows = bank_rows(keys)
  if placement == 'sharded':
    try:
      bank = ShardedImageBank(infer, rows, dp)
    except ShardOpenError as e:
      if image_bank == 'sharded':
        raise
      logger.info('%s: the sharded bank could not be set up, so it goes into pinned host memory: %s', what, e)
      placement = 'host'
    else:
      logger.info('%s: %d scans sharded over the GPUs of %d ranks, up to %.1f MB per rank, %.1f MB on the node; '
                  'each step gathers its rows from the shards into a ring of 2 x %d images on the GPU', what,
                  len(rows), world, shard_bytes / 1e6, bank_bytes / 1e6, 2 * b_share)
      return placement, bank, rows
  host = HostBank(eng, len(rows))
  fill_image_bank(infer, rows, host.images)
  logger.info('%s: %d scans in pinned host memory, %.1f MB per rank, %.1f MB on the node over %d ranks; each step '
              'copies its rows into a ring of 2 x %d images on the GPU', what, len(rows), host.nbytes / 1e6,
              world * host.nbytes / 1e6, world, 2 * b_share)
  return placement, host, rows
