#!/usr/bin/env python3
"""torch.profiler trace of the 1 x 1101 query step (the shape of bench.py's device-resident step: preprocess ->
leg -> heads_1vsN over a prepared bank).  Prints the mean device time of every kernel per step, the step's
wall time and the busy / idle split of the device.  `profile_step.py [TRACE.json]` also writes the Chrome
trace there.  Profile in a run of its own: tracing slows the host."""
import os, sys
from collections import defaultdict
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from torch.profiler import ProfilerActivity, profile
from overlapnet_b200 import synth
from overlapnet_b200.engine import Engine
from oracle import network as N

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
N_CAND, STEPS = 1101, 5


def main():
  out = sys.argv[1] if len(sys.argv) > 1 else None
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=N_CAND)
  eng.load_weights(N.glorot_weights(4, MODEL, seed=0))
  g = torch.Generator(device='cuda').manual_seed(0)
  bank = torch.rand((N_CAND, 360, 128), device='cuda', generator=g)
  eng.bank_prepare(bank)
  q = eng.upload_clouds([synth.kitti_like_cloud(50000)])
  qfv = torch.empty((360, 128), dtype=torch.float32, device='cuda')

  def step():
    qfv.copy_(eng.leg(eng.preprocess(q))[0])
    eng.heads_1vsN(bank, qfv, n_cand=N_CAND)

  for _ in range(3):
    step()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    for _ in range(STEPS):
      step()
    torch.cuda.synchronize()
  eng.check()
  kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
  per = defaultdict(lambda: [0.0, 0])
  for e in kern:
    per[e.name][0] += e.device_time
    per[e.name][1] += 1
  t0 = min(e.time_range.start for e in kern)
  t1 = max(e.time_range.end for e in kern)
  busy = sum(v[0] for v in per.values())
  print('%s, %d steps: device span %.3f ms per step, kernel time %.3f ms per step (%.1f %% busy)'
        % (torch.cuda.get_device_name(), STEPS, (t1 - t0) / 1e3 / STEPS, busy / 1e3 / STEPS, 100 * busy / (t1 - t0)))
  print('%-60s %8s %10s %10s' % ('kernel', 'calls', 'us/step', 'us/call'))
  for name, (us, c) in sorted(per.items(), key=lambda kv: -kv[1][0]):
    print('%-60s %8d %10.1f %10.1f' % (name[:60], c // STEPS, us / STEPS, us / c))
  if out:
    prof.export_chrome_trace(out)
  eng.close()


if __name__ == '__main__':
  main()
