#!/usr/bin/env python3
"""Batched leg encode timing (BASELINE config 3 and the geo-only variant): scans/s and TFLOP/s."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from overlapnet_b200 import synth
from overlapnet_b200.engine import Engine
sys.path.insert(0, ROOT)
import bench

def run(channels, use, batch, total):
  eng = Engine(use=use, model=bench.MODEL, precision='f16_tc', max_batch_scans=batch, max_batch_pairs=1)
  eng.load_weights(bench.make_weights(channels))
  x = torch.from_numpy(synth.range_like_images(5, 8, channels)).to(eng.device).repeat(total // 8, 1, 1, 1)
  for _ in range(2): eng.leg(x)
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(5): eng.leg(x)
  b.record(); torch.cuda.synchronize()
  ms = a.elapsed_time(b) / 5
  flop = {4: bench.FLOP_LEG_C4, 25: bench.FLOP_LEG_C25}.get(channels, bench.FLOP_LEG_C4)
  print('C=%d batch=%d total=%d: %.3f ms  %.2f us/scan  %.1f TFLOP/s algorithmic (x3 issued)' %
        (channels, batch, total, ms, ms * 1e3 / total, total * flop / 1e12 / (ms * 1e-3)))
  eng.close()

if __name__ == '__main__':
  sem = {'use_intensity': True, 'use_class_probabilities': True}
  run(4, {}, 64, 256)
  run(4, {}, 256, 256)
  run(5, {'use_intensity': True}, 64, 256)
  run(25, sem, 64, 256)
  run(25, sem, 256, 256)
