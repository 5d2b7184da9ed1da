"""Time one Monte Carlo localization step on the GPU: the filter's predict + update at N = 10^4, 10^5 and 10^6
particles, with the bytes its kernels move and the rate against the H100 SXM's 3.35 TB/s; the heads on 1, 16, 256
touched keyframes and on the whole map; and the encode of one query scan.

  python tools/time_mcl.py [--keyframes 2000] [--steps 50] [--out result.json]

The map is K keyframes every 2 m along a line, rasterised at 0.5 m within 5 m; the particles start in the disk of
2 m around random keyframes and the observations are synthetic.  Times are CUDA events around the calls (the predict
and the update each end with a host synchronisation, which is part of the step).  Prints one JSON line with the
card's name and power limit beside the numbers."""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import gpu_timing                                                 # noqa: E402
from overlapnet_b200 import mcl, synth                            # noqa: E402
from overlapnet_b200.engine import Engine                         # noqa: E402
from overlapnet_b200.infer import Infer                           # noqa: E402

MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
         'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
         'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
         'additional_unsymmetric_layer3a': True}
HBM_BYTES_PER_S = 3.35e12


def step_bytes(n, resampled):
  """DRAM bytes one predict + update moves for n particles (float64 x, y, theta, log-weight; int32 lookup), from the
  kernels' loads and stores; the map, touched list and partials are negligible.
    motion      reads x, y, theta (24), writes them (24) and the lookup (4)
    loglik      reads lookup, theta, log-weight (20), writes the log-likelihood (8)
    expsum      reads log-weight and log-likelihood (16)
    normalize   reads log-weight, log-likelihood, x, y, theta (40), writes log-weight and weight (16)
    resampling  tile sums read the weights (8); the prefix reads them again and writes C (16); the resampling reads
                each particle's ancestor (32) and C on its binary search (~8), writes the new set (32) and the
                ancestor (4)"""
  b = n * (24 + 24 + 4 + 20 + 8 + 16 + 40 + 16)
  if resampled:
    b += n * (8 + 16 + 32 + 8 + 32 + 4)
  return b


def timed(fn, reps):
  s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  s.record()
  for _ in range(reps):
    fn()
  e.record()
  torch.cuda.synchronize()
  return s.elapsed_time(e) / reps


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--keyframes', type=int, default=2000)
  p.add_argument('--steps', type=int, default=50)
  p.add_argument('--out')
  a = p.parse_args()
  gpu_timing.require_cuda('time_mcl.py')
  K = a.keyframes
  kf = np.stack([2.0 * np.arange(K), np.zeros(K), np.zeros(K)], 1)
  idx = mcl.MapIndex(kf[:, :2], 0.5, 5.0)
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=1101)
  eng.mcl_set_map(kf, idx.raster, idx.x0, idx.y0, idx.cell)
  rng = np.random.default_rng(0)
  ov_all = torch.as_tensor(rng.random(K).astype(np.float32)).cuda()
  yaw_all = torch.as_tensor(rng.integers(-180, 180, K).astype(np.int32)).cuda()
  result = {'card': gpu_timing.card(), 'keyframes': K, 'filter': []}
  for n in (10 ** 4, 10 ** 5, 10 ** 6):
    for rho, label in ((0.0, 'no_resampling'), (1.0, 'resampling')):
      eng.mcl_init('global', n, 1, init_radius=2.0)
      state = {}

      def step():
        touched, nt = eng.mcl_predict((2.0, 0.0, 0.0), (0.1, 0.1, 0.01))
        state['e'] = eng.mcl_update(ov_all[:nt], yaw_all[:nt], nt, 0.1, math.radians(10), rho)
      for _ in range(5):
        step()
      ms = timed(step, a.steps)
      resampled = state['e']['resampled']
      by = step_bytes(n, resampled)
      result['filter'].append({'particles': n, 'mode': label, 'resampled': bool(resampled), 'ms_per_step': ms,
                               'bytes_per_step': by, 'bytes_per_s': by / (ms * 1e-3),
                               'share_of_hbm_peak': by / (ms * 1e-3) / HBM_BYTES_PER_S,
                               'n_touched': state['e']['n_touched']})
  # the heads on the touched keyframes, and one query's encode
  cfg = {'pretrained_weightsfilename': '', 'use_depth': True, 'use_normals': True, 'use_class_probabilities': False,
         'use_class_probabilities_pca': False, 'use_intensity': False, 'data_root_folder': '', 'infer_seqs': '',
         'batch_size': 16, 'model': dict(MODEL)}
  infer = Infer(cfg)
  src = torch.cat([infer.encode_clouds([synth.kitti_like_cloud(s) for s in range(b, b + 16)]) for b in (0, 16)])
  bank = src[torch.arange(K, device=src.device) % src.shape[0]].contiguous()
  ieng = infer._engine
  ieng.calibrate(bank[0])
  infer._set_bank(bank)
  q = src[0]
  heads = []
  for nt in (1, 16, 256, K):
    ids = torch.arange(nt, dtype=torch.int32, device=bank.device)
    fn = (lambda ids=ids: ieng.heads_1vsN(infer._bank, q, cand_idx=ids))
    fn()
    heads.append({'n_touched': nt, 'ms': timed(fn, 20 if nt <= 256 else 3)})
  result['heads'] = heads
  cloud = synth.kitti_like_cloud(99)
  infer.encode_clouds([cloud])
  result['encode_ms'] = timed(lambda: infer.encode_clouds([cloud]), 20)
  line = json.dumps(result)
  print(line)
  if a.out:
    with open(a.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
