"""Time the loop-closure search over a whole sequence: ovn_heads_prefix_topk over every row of a 4 541-volume bank
with demo 3's 100-frame exclusion (9 859 020 pairs), against the same rows through ovn_heads_rows_vs_bank plus a
host argmax on a sample of rows, alternated in one process.

  python tools/time_lcd_eval.py [--precision f16_tc] [--k 5] [--repeats 3] [--sample-rows 64] [--out result.json]

The bank is bench.py's config 4: 32 seeded synthetic volumes yaw-rolled to 4 541 rows.  Prints one JSON line with
the card's name and power limit beside the numbers."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import gpu_timing                                                 # noqa: E402
from oracle import network as N                                   # noqa: E402
from overlapnet_b200 import synth                                 # noqa: E402
from overlapnet_b200.engine import Engine                         # noqa: E402

MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
         'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
         'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
         'additional_unsymmetric_layer3a': True}
N_BANK, N_SRC, EXCLUDE = 4541, 32, 100


def rolled_bank(fv_src, n, dev):
  """bench.py's rolled_bank: row i is source volume i % 32 rolled by 7 (i // 32) columns."""
  src = torch.arange(n, device=dev) % fv_src.shape[0]
  roll = (torch.arange(n, device=dev) // fv_src.shape[0]) * 7
  rows = (torch.arange(fv_src.shape[1], device=dev)[None, :] - roll[:, None]) % fv_src.shape[1]
  return fv_src[src[:, None], rows].contiguous()


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--precision', default='f16_tc', choices=('f16_tc', 'fp32'))
  p.add_argument('--k', type=int, default=5)
  p.add_argument('--repeats', type=int, default=3)
  p.add_argument('--sample-rows', type=int, default=64)
  p.add_argument('--out')
  a = p.parse_args()
  gpu_timing.require_cuda('time_lcd_eval.py')
  dev = torch.device('cuda', 0)
  eng = Engine(model=MODEL, precision=a.precision, max_batch_scans=N_SRC, max_batch_pairs=1101)
  eng.load_weights(N.glorot_weights(4, MODEL, seed=0))
  fv_src = torch.from_numpy(synth.feature_volumes(7, N_SRC)[:, 0]).to(dev)
  bank = rolled_bank(fv_src, N_BANK, dev)
  eng.calibrate(bank[0])
  eng.bank_prepare(bank)
  c = np.maximum(np.arange(N_BANK) - EXCLUDE, 0)
  pairs = int(c.sum())

  def events(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out

  full = lambda: eng.heads_prefix_topk(bank, 0, N_BANK, c, a.k)
  eng.heads_prefix_topk(bank, 1000, 1064, c[1000:1064], a.k)        # warm-up: modules, scratch, operand caches
  eng.check()
  full_ms = [events(full)[0] for _ in range(a.repeats)]
  eng.check()
  # the reduction's share, from the per-kernel events of a separate profiled run
  eng.profile_enable(True)
  eng.profile_read('rows_topk')
  prof_ms, _ = events(full)
  topk_ms, topk_launches = eng.profile_read('rows_topk')
  eng.profile_enable(False)
  # prefix top-k vs full rows + host argmax on a sample of late rows, alternated
  lo = N_BANK - a.sample_rows
  hi = N_BANK
  sample_pairs = int(c[lo:hi].sum())

  def rows_and_argmax():
    ov, yaw = eng.heads_rows_vs_bank(bank, lo, hi)
    ov, yaw = ov.cpu().numpy(), yaw.cpu().numpy()
    best = np.array([int(np.argmax(ov[r, :c[lo + r]])) for r in range(hi - lo)])
    return best, ov, yaw

  prefix_sample = lambda: eng.heads_prefix_topk(bank, lo, hi, c[lo:hi], 1)
  rows_and_argmax()
  t_prefix, t_rows = [], []
  for _ in range(a.repeats):
    ms, rec = events(prefix_sample)
    t_prefix.append(ms)
    ms, (best, ov, _) = events(rows_and_argmax)
    t_rows.append(ms)
  eng.check()
  agree = bool(np.array_equal(rec[1][:, 0].cpu().numpy(), best))
  res = {
      'card': gpu_timing.card(), 'precision': a.precision, 'k': a.k,
      'bank': N_BANK, 'exclude_frames': EXCLUDE, 'pairs': pairs,
      'prefix_topk_all_rows_ms': full_ms, 'prefix_topk_pairs_per_s': pairs / (min(full_ms) * 1e-3),
      'rows_topk_ms_profiled': topk_ms, 'rows_topk_launches': topk_launches, 'profiled_run_ms': prof_ms,
      'rows_topk_share': topk_ms / prof_ms,
      'sample': {'rows': [lo, hi], 'prefix_pairs': sample_pairs, 'full_row_pairs': (hi - lo) * N_BANK,
                 'prefix_topk_ms': t_prefix, 'rows_vs_bank_plus_host_argmax_ms': t_rows,
                 'top1_equals_host_argmax': agree},
  }
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, 'w') as f:
      f.write(line + '\n')
  eng.close()


if __name__ == '__main__':
  main()
