"""Both training flows at training precision fp32 and tf32x3, alternated: `--rounds` rounds (default 3) of
tools/time_train.py (frozen leg) and tools/time_train_leg.py (whole network), each timing fp32 and then tf32x3 on a
fresh handle.  Then the deviation between the two precisions on the batch each flow's timing draws first after its
warm-up: the three losses, and per layer max |g_tf32x3 - g_fp32| / max |g_fp32|, both computed on one handle at
the initial weights (the timed runs reach that batch after their warm-up Adagrad steps, at other weights).
One JSON line per timing and per flow's deviation; the card name and power limit are in every timing line."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import time_train
import time_train_leg
from overlapnet_b200 import synth
from overlapnet_b200 import weights as W
from overlapnet_b200.engine import Engine

PRECISIONS = ('fp32', 'tf32x3')


def deviation(flow):
  """Losses and per-layer gradient deviation of tf32x3 from fp32 on the first timed batch of ``flow``."""
  mod = time_train if flow == 'frozen_leg' else time_train_leg
  eng = Engine(model=mod.MODEL, precision='fp32', max_batch_scans=16, max_batch_pairs=mod.PAIRS)
  eng.load_weights(W.glorot_init(4, mod.MODEL, seed=0))
  rng = np.random.default_rng(0)
  for _ in range(mod.WARMUP + 1):        # the batches the timing draws, up to its first timed one
    li = torch.from_numpy(rng.integers(0, mod.BANK, mod.PAIRS).astype(np.int32)).cuda()
    ri = torch.from_numpy(rng.integers(0, mod.BANK, mod.PAIRS).astype(np.int32)).cuda()
    ov, yaw = rng.uniform(0, 1, mod.PAIRS).astype(np.float32), rng.integers(0, 360, mod.PAIRS).astype(np.int32)
  if flow == 'frozen_leg':
    g = torch.Generator(device='cuda').manual_seed(0)
    data = torch.rand((mod.BANK, 360, 128), device='cuda', generator=g)
    names = ('c_conv1', 'c_conv2', 'c_conv3', 'overlap_output')
  else:
    data = torch.from_numpy(synth.range_like_images(0, mod.BANK, 4)).cuda()
    names = eng.layers
  out = {}
  for p in PRECISIONS:
    eng.set_train_precision(p)
    if flow == 'frozen_leg':
      loss = eng.head_gradients(data, li, ri, ov, yaw, 0.7)
    else:
      loss = eng.net_gradients(data, li, ri, ov, yaw, 0.7)
    out[p] = loss, eng.get_gradients(names)
  eng.close()
  (l32, g32), (l3, g3) = out['fp32'], out['tf32x3']
  res = {'flow': flow, 'loss_fp32': l32, 'loss_tf32x3': l3,
         'loss_rel_dev': [abs(a - b) / abs(a) if a else abs(b) for a, b in zip(l32, l3)], 'grad_rel_dev': {}}
  for name in names:
    res['grad_rel_dev'][name] = [float(np.abs(g3[name][i] - g32[name][i]).max() / np.abs(g32[name][i]).max())
                                 for i in range(2)]
  return res


def main():
  argv = sys.argv[1:]
  rounds = int(argv[argv.index('--rounds') + 1]) if '--rounds' in argv else 3
  for r in range(rounds):
    for flow, mod in (('frozen_leg', time_train), ('whole_network', time_train_leg)):
      for p in PRECISIONS:
        print(json.dumps(dict(mod.run(False, p), flow=flow, round=r)), flush=True)
  for flow in ('frozen_leg', 'whole_network'):
    print(json.dumps(deviation(flow)), flush=True)


if __name__ == '__main__':
  main()
