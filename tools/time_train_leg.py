"""Step time of whole-network training (legsType 360OutputkLegs): CUDA events around ovn_net_gradients +
ovn_net_adagrad_step for 16-pair batches (fp32 handle, C = 4 with s_conv3a, a synthetic image bank), reported as
ms per step, pairs/s and achieved TFLOP/s against 17.9 GFLOP per training pair (8.94 G MAC, DESIGN.md section 4).
The card name and power limit are read in the same run, because they are part of the number.

--yaw-augmentation times the step of ``yaw_augmentation: True`` (overlapnet_b200.training_leg.WholeNetwork): the
16 LEFT images and the 16 rolled and rotated RIGHT images are gathered into a 32-image batch (ovn_gather_images)
that ovn_net_gradients then trains on.

--training-precision tf32x3 times the 3xTF32 tensor-core step (Engine.set_train_precision); tflops_issued counts
its three MMAs per product."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from overlapnet_b200 import augment, synth
from overlapnet_b200 import weights as W
from overlapnet_b200.engine import Engine
from time_train import card

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
GFLOP_PER_PAIR = 17.9
PAIRS, BANK, WARMUP, STEPS = 16, 64, 3, 20


def run(yaw_aug=False, precision='fp32'):
  """The timing of one configuration, as the dict main prints."""
  eng = Engine(model=MODEL, precision='fp32', max_batch_scans=16, max_batch_pairs=PAIRS)
  eng.load_weights(W.glorot_init(4, MODEL, seed=0))
  eng.set_train_precision(precision)
  images = torch.from_numpy(synth.range_like_images(0, BANK, 4)).cuda()
  rng = np.random.default_rng(0)
  batches = []
  for _ in range(WARMUP + STEPS):
    li = torch.from_numpy(rng.integers(0, BANK, PAIRS).astype(np.int32)).cuda()
    ri = torch.from_numpy(rng.integers(0, BANK, PAIRS).astype(np.int32)).cuda()
    batches.append((li, ri, rng.uniform(0, 1, PAIRS).astype(np.float32), rng.integers(0, 360, PAIRS).astype(np.int32)))
  np.random.seed(0)
  shifts = augment.sample_shifts(PAIRS, 900, 360)
  sh, rot = torch.from_numpy(shifts).cuda(), torch.from_numpy(augment.rotation(shifts, 900)).cuda()
  batch = torch.empty((2 * PAIRS,) + tuple(images.shape[1:]), dtype=torch.float32, device='cuda')
  pairs = torch.arange(2 * PAIRS, dtype=torch.int32, device='cuda')
  ms = []
  for i, (li, ri, ov, yaw) in enumerate(batches):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    if yaw_aug:
      eng.gather_images(images, li, out=batch[:PAIRS])
      eng.gather_images(images, ri, sh, rot, out=batch[PAIRS:])
      eng.net_gradients(batch, pairs[:PAIRS], pairs[PAIRS:], ov, yaw, 0.7)
    else:
      eng.net_gradients(images, li, ri, ov, yaw, 0.7)
    eng.net_adagrad_step(1e-6)
    e1.record()
    torch.cuda.synchronize()
    if i >= WARMUP:
      ms.append(e0.elapsed_time(e1))
  med = float(np.median(ms))
  eng.close()
  res = {'card': card(), 'training_precision': precision, 'yaw_augmentation': yaw_aug, 'pairs_per_step': PAIRS, 'steps': STEPS, 'ms_per_step_median': round(med, 3),
         'ms_per_step_min': round(float(np.min(ms)), 3), 'ms_per_step_max': round(float(np.max(ms)), 3),
         'pairs_per_s': round(PAIRS / med * 1e3, 1),
         'tflops': round(PAIRS * GFLOP_PER_PAIR / med, 3)}
  if precision == 'tf32x3':             # three MMAs per product
    res['tflops_issued'] = round(3 * res['tflops'], 3)
  return res


def main():
  argv = sys.argv[1:]
  precision = argv[argv.index('--training-precision') + 1] if '--training-precision' in argv else 'fp32'
  print(json.dumps(run('--yaw-augmentation' in argv, precision)))


if __name__ == '__main__':
  main()
