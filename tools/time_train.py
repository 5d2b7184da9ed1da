"""Step time of overlap-head training: CUDA events around ovn_head_gradients + ovn_head_adagrad_step for
16-pair batches (fp32 handle, synthetic bank), reported as ms per step, pairs/s and achieved TFLOP/s
against 5.53 GFLOP per training pair (forward 1.275 G MAC + backward 1.489 G MAC, DESIGN.md section 4).
The card name and power limit are read in the same run, because they are part of the number.

--yaw-augmentation times the step of ``yaw_augmentation: True`` (overlapnet_b200.training.FrozenLeg): the 16
RIGHT images are gathered from a synthetic image bank, rolled and rotated (ovn_gather_images), encoded by the
frozen fp32 leg into scratch rows after the volume bank, and the heads train on those rows.  The TFLOP/s figure
counts the heads only.

--training-precision tf32x3 times the 3xTF32 tensor-core step (Engine.set_train_precision); tflops_issued counts
its three MMAs per product."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from overlapnet_b200 import augment, synth
from overlapnet_b200.engine import Engine
from overlapnet_b200 import weights as W

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
GFLOP_PER_PAIR = 5.53
PAIRS, BANK, WARMUP, STEPS = 16, 64, 3, 20


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                          str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
    return out.strip()
  except Exception as e:                      # nvidia-smi missing: report what torch knows
    return '%s (power limit unknown: %s)' % (torch.cuda.get_device_name(), e)


def run(yaw_aug=False, precision='fp32'):
  """The timing of one configuration, as the dict main prints."""
  eng = Engine(model=MODEL, precision='fp32', max_batch_scans=16, max_batch_pairs=PAIRS)
  eng.load_weights(W.glorot_init(4, MODEL, seed=0))
  eng.set_train_precision(precision)
  g = torch.Generator(device='cuda').manual_seed(0)
  bank = torch.rand((BANK + (PAIRS if yaw_aug else 0), 360, 128), device='cuda', generator=g)
  if yaw_aug:
    images = torch.from_numpy(synth.range_like_images(0, BANK, 4)).cuda()
    scratch = torch.arange(BANK, BANK + PAIRS, dtype=torch.int32, device='cuda')
  rng = np.random.default_rng(0)
  batches = []
  for _ in range(WARMUP + STEPS):
    li = torch.from_numpy(rng.integers(0, BANK, PAIRS).astype(np.int32)).cuda()
    ri = torch.from_numpy(rng.integers(0, BANK, PAIRS).astype(np.int32)).cuda()
    batches.append((li, ri, rng.uniform(0, 1, PAIRS).astype(np.float32), rng.integers(0, 360, PAIRS).astype(np.int32)))
  np.random.seed(0)
  shifts = augment.sample_shifts(PAIRS, 900, 360)
  sh, rot = torch.from_numpy(shifts).cuda(), torch.from_numpy(augment.rotation(shifts, 900)).cuda()
  ms = []
  for i, (li, ri, ov, yaw) in enumerate(batches):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    if yaw_aug:
      eng.leg(eng.gather_images(images, ri, sh, rot), out=bank[BANK:])
      ri = scratch
    eng.head_gradients(bank, li, ri, ov, yaw, 0.7)
    eng.adagrad_step(1e-3)
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
