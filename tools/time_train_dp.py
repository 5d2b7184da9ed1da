"""Step times of data-parallel training (overlapnet_b200.data_parallel) for both flows, fp32 handle, C = 4 with
s_conv3a, synthetic banks, CUDA events around each step.  One command, rounds alternated three times:

  plain   today's one-GPU step of 16 pairs: ovn_head_gradients / ovn_net_gradients + the Adagrad step
  sum1    the same 16 pairs through the data-parallel path at world size 1: the gradients, ovn_copy_gradients and
          ovn_adagrad_step_sum with one part (the world-1 overhead of the new step)
  share8  one rank's compute of a 16-pair global batch at world size 2: the gradients of 8 pairs, the copy and a
          two-part ovn_adagrad_step_sum (the all-gather is not in it)

With two or more visible GPUs it also times the whole data-parallel step of a 16-pair global batch at world sizes
2 .. G (spawned ranks, NCCL all_gather_into_tensor), on rank 0.  The card name and power limit are read in the
same run, because they are part of the number."""
import json
import os
import socket
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from overlapnet_b200 import data_parallel, synth
from overlapnet_b200 import weights as W
from overlapnet_b200.engine import Engine
from time_train import card

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
PAIRS, BANK, WARMUP, STEPS, ROUNDS = 16, 64, 3, 20, 3


class Bench:
  """A handle, a bank and 16-pair batches for one flow ('frozen': head gradients on leg volumes; 'whole': the
  whole network on images)."""

  def __init__(self, kind, device=0, world=1):
    self.kind, self.whole = kind, kind == 'whole'
    self.eng = Engine(model=MODEL, precision='fp32', device=device, max_batch_scans=16, max_batch_pairs=PAIRS)
    self.eng.load_weights(W.glorot_init(4, MODEL, seed=0))
    dev = self.eng.device
    images = torch.from_numpy(synth.range_like_images(0, BANK, 4)).to(dev)
    self.bank = images if self.whole else self.eng.leg(images)
    rng = np.random.default_rng(0)
    self.batches = []
    for _ in range(WARMUP + STEPS):
      li = torch.from_numpy(rng.integers(0, BANK, PAIRS).astype(np.int32)).to(dev)
      ri = torch.from_numpy(rng.integers(0, BANK, PAIRS).astype(np.int32)).to(dev)
      self.batches.append((li, ri, torch.from_numpy(rng.uniform(0, 1, PAIRS).astype(np.float32)).to(dev),
                           torch.from_numpy(rng.integers(0, 360, PAIRS).astype(np.int32)).to(dev)))
    n = self.eng.gradient_size(self.whole)
    self.parts = torch.from_numpy((rng.standard_normal((max(world, 2), n)) * 1e-6).astype(np.float32)).to(dev)
    self.grad = torch.empty((n,), dtype=torch.float32, device=dev)

  def gradients(self, batch, lo, hi):
    li, ri, ov, yaw = (t[lo:hi] for t in batch)
    if self.whole:
      self.eng.net_gradients(self.bank, li, ri, ov, yaw, 0.7)
    else:
      self.eng.head_gradients(self.bank, li, ri, ov, yaw, 0.7)

  def step(self, mode, batch):
    if mode == 'plain':
      self.gradients(batch, 0, PAIRS)
      if self.whole:
        self.eng.net_adagrad_step(1e-6)
      else:
        self.eng.adagrad_step(1e-6)
    elif mode == 'sum1':
      self.gradients(batch, 0, PAIRS)
      self.eng.copy_gradients(self.whole, out=self.parts[0])
      self.eng.adagrad_step_sum(self.parts[:1], [1.0], 1e-6, self.whole)
    else:                                                          # share8
      self.gradients(batch, 0, PAIRS // 2)
      self.eng.copy_gradients(self.whole, out=self.parts[0])
      self.eng.adagrad_step_sum(self.parts[:2], [0.5, 0.5], 1e-6, self.whole)

  def time(self, fn):
    ms = []
    for i, batch in enumerate(self.batches):
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      fn(batch)
      e1.record()
      torch.cuda.synchronize()
      if i >= WARMUP:
        ms.append(e0.elapsed_time(e1))
    return round(float(np.median(ms)), 3)


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _rank(rank, world, port, kind, out):
  import torch.distributed as dist
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(rank)
  dist.init_process_group('nccl', rank=rank, world_size=world)
  try:
    b = Bench(kind, rank, world)
    dp = data_parallel.DataParallel()
    bounds, weights = data_parallel.shares(PAIRS, world)
    lo, hi = bounds[rank]
    parts = b.parts[:world]

    def dp_step(batch):
      b.gradients(batch, lo, hi)
      b.eng.copy_gradients(b.whole, out=b.grad)
      dp.gather_flat(b.grad, parts)
      b.eng.adagrad_step_sum(parts, weights, 1e-6, b.whole)

    ms = b.time(dp_step)
    if rank == 0:
      with open(out, 'w') as f:
        json.dump(ms, f)
  finally:
    dist.destroy_process_group()


def main():
  res = {'card': card(), 'global_batch_pairs': PAIRS, 'steps': STEPS, 'rounds': ROUNDS,
         'ms_per_step_median': {}}
  benches = {kind: Bench(kind) for kind in ('frozen', 'whole')}
  for _ in range(ROUNDS):
    for kind, b in benches.items():
      for mode in ('plain', 'sum1', 'share8'):
        res['ms_per_step_median'].setdefault('%s/%s' % (kind, mode), []).append(b.time(lambda x: b.step(mode, x)))
  for b in benches.values():
    b.eng.close()
  gpus = torch.cuda.device_count()
  if gpus >= 2:
    import tempfile
    import torch.multiprocessing as mp
    res['nccl_ms_per_step_median'] = {}
    with tempfile.TemporaryDirectory() as tmp:
      for kind in ('frozen', 'whole'):
        for world in range(2, gpus + 1):
          out = os.path.join(tmp, '%s_%d.json' % (kind, world))
          mp.spawn(_rank, args=(world, _free_port(), kind, out), nprocs=world, join=True)
          with open(out) as f:
            res['nccl_ms_per_step_median']['%s/world%d' % (kind, world)] = json.load(f)
  else:
    res['nccl_ms_per_step_median'] = 'not measured: %d visible GPU' % gpus
  print(json.dumps(res))


if __name__ == '__main__':
  main()
