"""Step time of training with the image bank on the GPU against the image bank in pinned host memory
(overlapnet_b200.image_bank): 16-pair steps of both flows -- the whole network, and the frozen leg with yaw
augmentation -- at C = 4 and C = 25, the two placements alternated three times in one command, each the median of
20 steps after 3 warm-up steps.  The flows are the training flows themselves, built on a synthetic bank of 256
scans (random cues, Glorot weights, fp32).

The steps run back to back with one synchronise of the compute stream at the end, so the ring's copies overlap
the following steps as they do in training.  Reported per run: ms per step (between events on the compute stream
at the step boundaries); with the host bank also the milliseconds per step the compute stream waited on copy-done
events and the distinct images staged per step; per C the realised host-to-device rate of one step's row copies
(ovn_stage_rows from the pinned bank into a slot, CUDA events on the copy stream).  The card name and power limit
are read in the same run, because they are part of the numbers.

  python tools/time_train_image_bank.py [--out results.json]
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from overlapnet_b200 import augment, image_bank, training, training_leg
from overlapnet_b200 import weights as W
from overlapnet_b200.engine import Engine
from time_train import card

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
USE = {4: {}, 25: {'use_class_probabilities': True, 'use_intensity': True}}
PAIRS, SCANS, WARMUP, STEPS, ROUNDS = 16, 256, 3, 20, 3


class SyntheticInfer:
  """What the flows read of overlapnet_b200.infer.Infer, over an in-memory bank: the handle, the cue loader
  (``_prepare_inputs``) and the frozen leg's encoder."""

  def __init__(self, eng, images):
    self._engine, self.images, self.seq = eng, images, None

  def _prepare_inputs(self, names):
    return self.images[[int(n) for n in names]]

  def _create_feature_volumes_device(self, names):
    dev = self._engine.device
    return torch.cat([self._engine.leg(torch.from_numpy(self._prepare_inputs(names[s:s + 16])).to(dev))
                      for s in range(0, len(names), 16)])


def run(eng, images, legs, placement):
  infer = SyntheticInfer(eng, images)
  keys = {('00', '%06d' % i) for i in range(SCANS)}
  yaw = legs == 'frozen'
  if yaw:
    flow = training.FrozenLeg(infer, keys, keys, image_bank=placement)
  else:
    flow = training_leg.WholeNetwork(infer, keys, image_bank=placement)
  rng = np.random.default_rng(0)
  n = (WARMUP + STEPS) * PAIRS
  left_h, right_h = rng.integers(0, SCANS, n), rng.integers(0, SCANS, n)
  dev = eng.device
  left, right = torch.from_numpy(left_h.astype(np.int32)).to(dev), torch.from_numpy(right_h.astype(np.int32)).to(dev)
  ov = torch.from_numpy(rng.uniform(0, 1, n).astype(np.float32)).to(dev)
  orient = torch.from_numpy(rng.integers(0, 360, n).astype(np.int32)).to(dev)
  rotate = None
  if yaw:
    shifts = augment.sample_shifts(n, eng.W, eng.Wf)
    rotate = (right, torch.from_numpy(shifts).to(dev), torch.from_numpy(augment.rotation(shifts, eng.W)).to(dev))
  if flow.ring is not None:
    flow.ring.timing = True
    flow.begin_epoch([(s, s + PAIRS) for s in range(0, n, PAIRS)], left_h, right_h, right_h if yaw else None)
  # The steps run back to back as in the training loop: one event on the compute stream at each step boundary and
  # one synchronise of the compute stream after the last step.  Nothing synchronises the device in between, so
  # the copies the ring issues after a step overlap the next step as they do in training.
  marks, rows = [], []
  for s in range(0, n, PAIRS):
    marks.append(torch.cuda.Event(enable_timing=True))
    marks[-1].record()
    flow.step(left[s:s + PAIRS], right[s:s + PAIRS], ov[s:s + PAIRS], orient[s:s + PAIRS], 0.7, 1e-3,
              None if rotate is None else tuple(t[s:s + PAIRS] for t in rotate))
    if flow.ring is not None:
      rows.append(flow.ring.step_rows)
  marks.append(torch.cuda.Event(enable_timing=True))
  marks[-1].record()
  torch.cuda.current_stream().synchronize()
  ms = [marks[i].elapsed_time(marks[i + 1]) for i in range(WARMUP, WARMUP + STEPS)]
  eng.check()
  out = {'flow': legs, 'image_bank': flow.image_bank, 'ms_per_step_median': round(float(np.median(ms)), 3),
         'ms_per_step_min': round(float(np.min(ms)), 3), 'ms_per_step_max': round(float(np.max(ms)), 3),
         'ms_per_step_mean': round(marks[WARMUP].elapsed_time(marks[-1]) / STEPS, 3)}
  if flow.ring is not None:
    waits = flow.ring.wait_ms()[WARMUP:]
    out['copy_wait_ms_per_step_median'] = round(float(np.median(waits)), 3)
    out['copy_wait_ms_per_step_max'] = round(float(np.max(waits)), 3)
    out['images_copied_per_step_mean'] = round(float(np.mean(rows[WARMUP:])), 2)
    flow.images.close()
  return out


def h2d_rate(eng, images):
  """GB/s of one step's row copies (2 x PAIRS distinct random rows) from a pinned bank into a device slot."""
  host = image_bank.HostBank(eng, images.shape[0])
  host.images[:] = images
  slot = torch.empty((2 * PAIRS,) + images.shape[1:], dtype=torch.float32, device=eng.device)
  stream = torch.cuda.Stream(device=eng.device)
  rng = np.random.default_rng(1)
  ms = []
  for i in range(WARMUP + STEPS):
    rows = rng.choice(images.shape[0], 2 * PAIRS, replace=False)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
      e0.record(stream)
      eng.stage_rows(host.images, rows, slot)
      e1.record(stream)
    stream.synchronize()
    if i >= WARMUP:
      ms.append(e0.elapsed_time(e1))
  host.close()
  med = float(np.median(ms))
  nbytes = 2 * PAIRS * images[0].nbytes
  return {'bytes_per_step': int(nbytes), 'ms_median': round(med, 3), 'gb_per_s': round(nbytes / med / 1e6, 2)}


def main():
  argv = sys.argv[1:]
  results = {'card': card(), 'pairs_per_step': PAIRS, 'scans': SCANS, 'steps': STEPS, 'warmup': WARMUP, 'runs': []}
  for C in (4, 25):
    eng = Engine(use=USE[C], model=MODEL, precision='fp32', max_batch_scans=16, max_batch_pairs=PAIRS)
    assert eng.C == C, eng.C
    eng.load_weights(W.glorot_init(C, MODEL, seed=0))
    images = np.random.default_rng(C).random((SCANS, eng.H, eng.W, C), dtype=np.float32)
    results['h2d_C%d' % C] = h2d_rate(eng, images)
    print(json.dumps({'C': C, 'h2d': results['h2d_C%d' % C]}), flush=True)
    for legs in ('whole', 'frozen'):
      for r in range(ROUNDS):
        for placement in ('device', 'host'):
          res = dict(run(eng, images, legs, placement), C=C, round=r)
          results['runs'].append(res)
          print(json.dumps(res), flush=True)
    eng.close()
  print(json.dumps(results))
  if '--out' in argv:
    with open(argv[argv.index('--out') + 1], 'w') as f:
      json.dump(results, f, indent=1)


if __name__ == '__main__':
  main()
