"""Step time of ``gradient_chunks`` (overlapnet_b200.training, DESIGN.md section 5) on one GPU: 16-pair steps of
both training flows at training precision fp32 and tf32x3 (C = 4 with s_conv3a, synthetic banks), CUDA events
around each step, the median of STEPS steps after WARMUP warm-up steps.  For each flow and precision:

  plain      today's step: ovn_head_gradients / ovn_net_gradients + ovn_head_adagrad_step / ovn_net_adagrad_step
  chunks K   ovn_*_gradients_chunks over the 16 pairs in K chunks + ovn_adagrad_step_sum of the K parts
  separate K K one-chunk calls, each followed by ovn_copy_gradients, + ovn_adagrad_step_sum: what the chunked call
             replaces

``--rounds`` rounds (default 3) alternate every configuration in one command.  One JSON line per timing; the card
name and power limit are in every line."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from overlapnet_b200 import data_parallel, synth
from overlapnet_b200 import weights as W
from overlapnet_b200.engine import Engine
from time_train import card

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
PAIRS, BANK, WARMUP, STEPS = 16, 64, 3, 20
CHUNKS = (1, 2, 4, 8, 16)
PRECISIONS = ('fp32', 'tf32x3')


def _timings(flow, precision, card_info, rnd):
  whole = flow == 'whole_network'
  eng = Engine(model=MODEL, precision='fp32', max_batch_scans=16, max_batch_pairs=PAIRS)
  eng.load_weights(W.glorot_init(4, MODEL, seed=0))
  eng.set_train_precision(precision)
  if whole:
    rows = torch.from_numpy(synth.range_like_images(0, BANK, 4)).cuda()
    grads, step = eng.net_gradients, eng.net_adagrad_step
    chunked = eng.net_gradients_chunks
  else:
    g = torch.Generator(device='cuda').manual_seed(0)
    rows = torch.rand((BANK, 360, 128), device='cuda', generator=g)
    grads, step = eng.head_gradients, eng.adagrad_step
    chunked = eng.head_gradients_chunks
  rng = np.random.default_rng(0)
  batches = []
  for _ in range(WARMUP + STEPS):
    li = torch.from_numpy(rng.integers(0, BANK, PAIRS).astype(np.int32)).cuda()
    ri = torch.from_numpy(rng.integers(0, BANK, PAIRS).astype(np.int32)).cuda()
    ov = torch.from_numpy(rng.uniform(0, 1, PAIRS).astype(np.float32)).cuda()
    yaw = torch.from_numpy(rng.integers(0, 360, PAIRS).astype(np.int32)).cuda()
    batches.append((li, ri, ov, yaw))
  parts = torch.empty((max(CHUNKS), eng.gradient_size(whole)), dtype=torch.float32, device='cuda')

  def plain(li, ri, ov, yaw):
    grads(rows, li, ri, ov, yaw, 0.7)
    step(1e-6)

  def chunks(k):
    bounds, weights = data_parallel.shares(PAIRS, k)
    offsets = [a for a, _ in bounds] + [PAIRS]

    def run(li, ri, ov, yaw):
      chunked(rows, li, ri, offsets, ov, yaw, 0.7, out=parts[:k])
      eng.adagrad_step_sum(parts[:k], weights, 1e-6, whole)
    return run

  def separate(k):
    bounds, weights = data_parallel.shares(PAIRS, k)

    def run(li, ri, ov, yaw):
      for c, (a, b) in enumerate(bounds):
        grads(rows, li[a:b], ri[a:b], ov[a:b], yaw[a:b], 0.7)
        eng.copy_gradients(whole, out=parts[c])
      eng.adagrad_step_sum(parts[:k], weights, 1e-6, whole)
    return run

  modes = [('plain', 1, plain)] + [('chunks', k, chunks(k)) for k in CHUNKS] + \
          [('separate', k, separate(k)) for k in CHUNKS if k > 1]
  out = []
  for mode, k, fn in modes:
    ms = []
    for i, batch in enumerate(batches):
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      fn(*batch)
      e1.record()
      torch.cuda.synchronize()
      if i >= WARMUP:
        ms.append(e0.elapsed_time(e1))
    med = float(np.median(ms))
    out.append({'card': card_info, 'round': rnd, 'flow': flow, 'training_precision': precision, 'mode': mode,
                'chunks': k, 'pairs_per_step': PAIRS, 'steps': STEPS, 'ms_per_step_median': round(med, 3),
                'ms_per_step_min': round(float(np.min(ms)), 3), 'ms_per_step_max': round(float(np.max(ms)), 3)})
  eng.check()
  eng.close()
  return out


def main():
  argv = sys.argv[1:]
  rounds = int(argv[argv.index('--rounds') + 1]) if '--rounds' in argv else 3
  info = card()
  for r in range(rounds):
    for flow in ('frozen_leg', 'whole_network'):
      for p in PRECISIONS:
        for line in _timings(flow, p, info, r):
          print(json.dumps(line), flush=True)


if __name__ == '__main__':
  main()
