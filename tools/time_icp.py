"""Time point-to-plane ICP of loop-closure pairs on the GPU (ovn_icp_pairs): pairs/s at np = 1, 132, 1024 and 8192
street-scene pairs at 64 x 900, both at exactly 30 iterations (eps_rot = eps_trans = 0, so no pair stops early) and
with the default stopping rules (with the iterations those pairs actually run); the bytes one iteration reads per
pair, from shapes; and the time that --register adds to lcd_eval.evaluate_clouds on a two-lap street-scene sequence.

  python tools/time_icp.py [--distinct 16] [--repeats 5] [--out result.json]

The pairs cycle through ``--distinct`` street-scene pairs 0-3 m and up to 30 degrees apart, seeded from their true
yaw bin.  Times are CUDA events around one ovn_icp_pairs call each, after warm-up calls of the same shape; the
evaluate_clouds times are host clocks around whole calls that end in a device synchronise.  Prints one JSON line
with the card's name and power limit beside the numbers."""
import argparse
import copy
import json
import math
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import gpu_timing                                                 # noqa: E402
from oracle import network as N                                   # noqa: E402
from overlapnet_b200 import gt, lcd_eval, registration, synth, weights as W     # noqa: E402
from overlapnet_b200.engine import Engine                         # noqa: E402

MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
         'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
         'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
         'additional_unsymmetric_layer3a': True}
PAIRS = (1, 132, 1024, 8192)
SOURCE_BYTES = 16 + 12      # per source pixel and iteration: its float4 vertex and float3 normal
TARGET_BYTES = 16 + 12      # per gathered target pixel: the same of the pixel it projects to


def rz(yaw, t):
  T = np.eye(4)
  T[:2, :2] = [[math.cos(yaw), -math.sin(yaw)], [math.sin(yaw), math.cos(yaw)]]
  T[:3, 3] = t
  return T


def street_pairs(n, seed=3):
  """n (LEFT, RIGHT, T*) street-scene pairs: RIGHT 0-3 m and up to 30 degrees from LEFT."""
  rng = np.random.default_rng(seed)
  out = []
  for _ in range(n):
    x, y = rng.uniform(-10, 10), rng.choice([-1.0, 1.0]) * rng.uniform(0, 2)
    TL = rz(rng.uniform(-math.pi, math.pi), (x, y, 1.73))
    d, a = rng.uniform(0, 3), rng.uniform(-math.pi, math.pi)
    TR = rz(math.atan2(TL[1, 0], TL[0, 0]) + math.radians(rng.uniform(-30, 30)),
            (x + d * math.cos(a), y + d * math.sin(a), 1.73))
    out.append((synth.street_scene_cloud(TL, seed), synth.street_scene_cloud(TR, seed), np.linalg.solve(TL, TR)))
  return out


def time_pairs(eng, vertex, normal, init, distinct, n_pairs, repeats, params):
  k = np.arange(n_pairs) % distinct
  src, dst = torch.as_tensor(2 * k + 1, dtype=torch.int32).cuda(), torch.as_tensor(2 * k, dtype=torch.int32).cuda()
  ini = torch.as_tensor(init[k]).cuda()
  res = {}

  def call(_):
    res.update(eng.icp(vertex, normal, src, dst, ini, params))
  ms = gpu_timing.step_ms(call, range(repeats + 2), 2)
  eng.check()
  it = res['iterations'].double()
  valid = res['valid'].double()
  return dict(gpu_timing.summary(ms), pairs=n_pairs, pairs_per_s=round(n_pairs / (float(np.median(ms)) * 1e-3), 1),
              iterations_mean=round(float(it.mean()), 2), iterations_max=int(it.max()),
              status_counts=np.bincount(res['status'].cpu().numpy(), minlength=5).tolist(),
              bytes_per_iteration_per_pair=int(eng.H * eng.W * SOURCE_BYTES + float(valid.mean()) * TARGET_BYTES))


def loop_sequence():
  poses = []
  for lap, off in ((0, 0.0), (1, 1.5)):
    for k in range(32):
      s = k * 5.0
      side, u = int(s // 40), s % 40
      x, y, yaw = [(u, off, 0.0), (40 - off, u, 90.0), (40 - u, 40 - off, 180.0), (off, 40 - u, 270.0)][side]
      poses.append(rz(math.radians(yaw), (x, y, 1.73)))
  poses = np.array(poses)
  return [synth.street_scene_cloud(T, seed=11) for T in poses], poses


def time_register(repeats):
  """Seconds of evaluate_clouds without and with register on the 64-scan loop, alternating, median of each."""
  from overlapnet_b200.infer import Infer
  clouds, poses = loop_sequence()
  with tempfile.TemporaryDirectory() as tmp:
    wpath = os.path.join(tmp, 'weights.npz')
    W.save_npz(wpath, N.glorot_weights(4, MODEL, seed=5))
    cfg = {'pretrained_weightsfilename': wpath, 'use_depth': True, 'use_normals': True,
           'use_class_probabilities': False, 'use_class_probabilities_pca': False, 'use_intensity': False,
           'data_root_folder': tmp, 'infer_seqs': '07', 'batch_size': 16, 'model': copy.deepcopy(MODEL)}
    t = {False: [], True: []}
    for rep in range(repeats + 1):
      for reg in (False, True):
        infer = Infer(copy.deepcopy(cfg))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s, res = lcd_eval.evaluate_clouds(infer, clouds, poses, top_k=3, exclude_frames=10, exclude_distance=20.0,
                                          register=reg)
        torch.cuda.synchronize()
        if rep:                                                   # the first round warms up both
          t[reg].append(time.perf_counter() - t0)
    records = int((res['top_index'][:, 0] >= 0).sum())
  plain, reg = float(np.median(t[False])), float(np.median(t[True]))
  return {'scans': len(clouds), 'records_registered_twice': records, 'evaluate_s_median': round(plain, 3),
          'evaluate_register_s_median': round(reg, 3), 'register_overhead_s': round(reg - plain, 3),
          'registration': s['registration']}


def main():
  p = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  p.add_argument('--distinct', type=int, default=16)
  p.add_argument('--repeats', type=int, default=5)
  p.add_argument('--out', default=None)
  a = p.parse_args()
  gpu_timing.require_cuda('time_icp')
  card = gpu_timing.card()
  eng = Engine(precision='fp32', max_batch_scans=16, max_batch_pairs=1)
  pairs = street_pairs(a.distinct)
  vertex, normal = registration.images(eng, [c for L, R, _ in pairs for c in (L, R)], list(range(2 * a.distinct)))
  init = np.stack([registration.seed_pose(gt.yaw_bin(np.eye(4), T, 360), 360) for _, _, T in pairs])
  fixed = [time_pairs(eng, vertex, normal, init, a.distinct, n, a.repeats, {'eps_rot': 0.0, 'eps_trans': 0.0})
           for n in PAIRS]
  default = [time_pairs(eng, vertex, normal, init, a.distinct, n, a.repeats, None) for n in PAIRS]
  eng.close()
  out = {'tool': 'time_icp', 'card': card, 'geometry': '64x900', 'distinct_pairs': a.distinct,
         'thirty_iterations': fixed, 'default_stopping': default, 'lcd_eval_register': time_register(2)}
  line = json.dumps(out)
  print(line)
  if a.out:
    with open(a.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
