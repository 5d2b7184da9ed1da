"""Step time of training the whole network with the image bank on the GPU, sharded over the GPUs of two
data-parallel ranks, and in pinned host memory (overlapnet_b200.image_bank): 16-pair steps, 8 pairs per rank, at
C = 4 and C = 25, the three placements alternated three times in one command, each the median of 20 steps after 3
warm-up steps.  Two
ranks: NCCL on two GPUs when the machine has them, otherwise gloo with both ranks on one GPU.  The flow is
training_leg.WholeNetwork itself, built on a synthetic bank of 256 scans (random cues, Glorot weights, fp32); each
rank runs its own steps (the flow's step, without the gradient all-gather), so the numbers are those of the staging.

Reported per run and rank 0: ms per step (events on the compute stream at the step boundaries), and with a staged
bank the milliseconds per step the compute stream waited on copy-done events (StagingRing.wait_ms) and the distinct
images staged per step; per C the realised rate of k_gather_rows over one step's rows (2 x 8 distinct random rows
of the sharded bank, half of them in the peer's shard on average), from its CUDA events (ovn_profile_read) and the
bytes it moved.  The card name and power limit are read in the same run, because they are part of the numbers.

  python tools/time_train_sharded_bank.py [--out results.json]
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from overlapnet_b200 import training_leg
from overlapnet_b200 import weights as W
from overlapnet_b200.engine import Engine
from time_train import card
from time_train_image_bank import MODEL, PAIRS, ROUNDS, SCANS, STEPS, USE, WARMUP, SyntheticInfer

RANKS = 2
SHARE = PAIRS // RANKS         # the pairs of a 16-pair step each rank trains


def run(eng, images, placement):
  infer = SyntheticInfer(eng, images)
  keys = {('00', '%06d' % i) for i in range(SCANS)}
  flow = training_leg.WholeNetwork(infer, keys, image_bank=placement)
  rng = np.random.default_rng(dist.get_rank())
  n = (WARMUP + STEPS) * SHARE
  left_h, right_h = rng.integers(0, SCANS, n), rng.integers(0, SCANS, n)
  dev = eng.device
  left, right = torch.from_numpy(left_h.astype(np.int32)).to(dev), torch.from_numpy(right_h.astype(np.int32)).to(dev)
  ov = torch.from_numpy(rng.uniform(0, 1, n).astype(np.float32)).to(dev)
  orient = torch.from_numpy(rng.integers(0, 360, n).astype(np.int32)).to(dev)
  if flow.ring is not None:
    flow.ring.timing = True
    flow.begin_epoch([(s, s + SHARE) for s in range(0, n, SHARE)], left_h, right_h)
  marks, rows = [], []
  for s in range(0, n, SHARE):
    marks.append(torch.cuda.Event(enable_timing=True))
    marks[-1].record()
    flow.step(left[s:s + SHARE], right[s:s + SHARE], ov[s:s + SHARE], orient[s:s + SHARE], 0.7, 1e-3)
    if flow.ring is not None:
      rows.append(flow.ring.step_rows)
  marks.append(torch.cuda.Event(enable_timing=True))
  marks[-1].record()
  torch.cuda.current_stream().synchronize()
  ms = [marks[i].elapsed_time(marks[i + 1]) for i in range(WARMUP, WARMUP + STEPS)]
  eng.check()
  out = {'image_bank': flow.image_bank, 'ms_per_step_median': round(float(np.median(ms)), 3),
         'ms_per_step_min': round(float(np.min(ms)), 3), 'ms_per_step_max': round(float(np.max(ms)), 3)}
  if flow.ring is not None:
    waits = flow.ring.wait_ms()[WARMUP:]
    out['copy_wait_ms_per_step_median'] = round(float(np.median(waits)), 3)
    out['copy_wait_ms_per_step_max'] = round(float(np.max(waits)), 3)
    out['images_staged_per_step_mean'] = round(float(np.mean(rows[WARMUP:])), 2)
  if flow.image_bank == 'sharded':
    out['gather'] = gather_rate(eng, flow.images)
  if flow.image_bank != 'device':
    flow.images.close()                              # collective for the sharded bank
  return out


def gather_rate(eng, bank):
  """k_gather_rows' bytes/s over one step's rows (2 x SHARE distinct random rows) into a device slot."""
  slot = torch.empty((2 * SHARE, eng.H, eng.W, eng.C), dtype=torch.float32, device=eng.device)
  rng = np.random.default_rng(1)
  eng.profile_enable(True)
  eng.profile_read('gather_rows')
  ms = []
  for i in range(WARMUP + STEPS):
    bank.stage(rng.choice(SCANS, 2 * SHARE, replace=False), slot)
    t, launches = eng.profile_read('gather_rows')                  # synchronises
    assert launches == 1, launches
    if i >= WARMUP:
      ms.append(t)
  eng.profile_enable(False)
  med = float(np.median(ms))
  nbytes = 2 * SHARE * eng.H * eng.W * eng.C * 4
  return {'bytes_per_step': int(nbytes), 'ms_median': round(med, 4), 'gb_per_s': round(nbytes / med / 1e6, 2)}


def worker(rank, world, port, backend, out):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(rank if backend == 'nccl' else 0)
  dist.init_process_group(backend, rank=rank, world_size=world)
  try:
    results = {'card': card(), 'backend': backend, 'ranks': world, 'pairs_per_step': PAIRS, 'pairs_per_rank': SHARE,
               'scans': SCANS, 'steps': STEPS, 'warmup': WARMUP, 'runs': []}
    for C in (4, 25):
      eng = Engine(use=USE[C], model=MODEL, precision='fp32', max_batch_scans=16, max_batch_pairs=PAIRS)
      assert eng.C == C, eng.C
      eng.load_weights(W.glorot_init(C, MODEL, seed=0))
      images = np.random.default_rng(C).random((SCANS, eng.H, eng.W, C), dtype=np.float32)
      for r in range(ROUNDS):
        for placement in ('device', 'sharded', 'host'):
          res = dict(run(eng, images, placement), C=C, round=r)
          results['runs'].append(res)
          if rank == 0:
            print(json.dumps(res), flush=True)
      eng.close()
    if rank == 0:
      print(json.dumps(results))
      if out:
        with open(out, 'w') as f:
          json.dump(results, f, indent=1)
  finally:
    dist.destroy_process_group()


def main():
  import socket
  argv = sys.argv[1:]
  out = argv[argv.index('--out') + 1] if '--out' in argv else None
  backend = 'nccl' if torch.cuda.device_count() >= 2 else 'gloo'
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  port = s.getsockname()[1]
  s.close()
  mp.spawn(worker, args=(RANKS, port, backend, out), nprocs=RANKS, join=True)


if __name__ == '__main__':
  main()
