"""Timings of a semantic config (C = 25: depth, normals, 20 class probabilities, intensity) from raw scans.

1. Preprocess per scan, at 1 and 32 scans per call: the fused ``Engine.preprocess_cues`` (ovn_preprocess_cues_batch:
   one scatter into two key images, one gather) against the five-call device route that gives the same bits
   (ovn_project_batch at max_range, ovn_normals_batch, ovn_project_batch at inf for the index, ovn_semantic_batch,
   ovn_pack_input).  CUDA events around each call on the current stream; medians.
2. One raw query (cloud + probabilities in host memory) against 1101 candidates, results back in host memory:
   ``query_cloud_vs_bank_host(probs=...)`` (ovn_query_cloud_probs_vs_bank_host, one host synchronisation) against
   upload + the five calls + leg + heads_1vsN + copies back.  Both end in a device synchronisation, so a host clock
   around each call is the call's time; medians.

KITTI-shaped clouds of 124 668 points, softmax class probabilities, seeded.  Prints one JSON line with the card's
name and power limit; ``--out`` also writes it to a file.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import gpu_timing
from oracle import network as N
from overlapnet_b200 import synth
from overlapnet_b200.engine import Engine

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
USE = {'use_class_probabilities': True, 'use_intensity': True}
N_POINTS = 124668
N_CAND = 1101


def event_median_ms(fn, reps, warm):
  return float(np.median(gpu_timing.step_ms(lambda _: fn(), range(warm + reps), warm)))


def host_median_ms(fn, reps, warm):
  for _ in range(warm):
    fn()
  torch.cuda.synchronize()
  times = []
  for _ in range(reps):
    t0 = time.perf_counter()
    fn()
    times.append((time.perf_counter() - t0) * 1e3)
  return float(np.median(times))


def five_calls(eng, batch, probs):
  out = eng.project(batch, want=('range', 'vertex', 'intensity'))
  nrm = eng.normals(out['range'], out['vertex'])
  idx = eng.project(batch, max_range=float('inf'), want=('idx',))['idx']
  sem = eng.semantic(idx, probs, batch.offsets)
  return eng.pack_input(out['range'], nrm, sem, out['intensity'])


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=30)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  gpu_timing.require_cuda('time_semantic_raw.py')
  eng = Engine(use=USE, model=MODEL, precision='f16_tc', max_batch_scans=32, max_batch_pairs=N_CAND)
  assert eng.C == 25
  eng.load_weights(N.glorot_weights(25, MODEL, seed=0))
  clouds = [synth.kitti_like_cloud(s, n_points=N_POINTS) for s in range(32)]
  probs = [synth.random_probs(1000 + s, N_POINTS) for s in range(32)]
  res = {'card': gpu_timing.card(), 'C': eng.C, 'n_points': N_POINTS, 'reps': args.reps}

  for n in (1, 32):
    batch = eng.upload_clouds(clouds[:n])
    p = torch.from_numpy(np.concatenate(probs[:n])).to(eng.device)
    fused, split = eng.preprocess_cues(batch, p), five_calls(eng, batch, p)
    assert torch.equal(fused.view(torch.int32), split.view(torch.int32))
    t_fused = event_median_ms(lambda: eng.preprocess_cues(batch, p), args.reps, args.warmup)
    t_split = event_median_ms(lambda: five_calls(eng, batch, p), args.reps, args.warmup)
    res['preprocess_%d_scans' % n] = {'fused_ms_per_scan': t_fused / n, 'five_calls_ms_per_scan': t_split / n,
                                      'speedup': t_split / t_fused}

  bank = torch.from_numpy(synth.feature_volumes(7, N_CAND)[:, 0]).to(eng.device)
  eng.bank_prepare(bank)
  q, qp = clouds[0], probs[0]
  ov_h, yaw_h = np.empty(N_CAND, np.float32), np.empty(N_CAND, np.int32)

  def host_query():
    eng.query_cloud_vs_bank_host(q, bank, n_cand=N_CAND, out_overlap=ov_h, out_yaw=yaw_h, probs=qp)

  def device_route():
    batch = eng.upload_clouds([q])
    p = torch.from_numpy(qp).to(eng.device)
    fv = eng.leg(five_calls(eng, batch, p))
    ov, yaw, _ = eng.heads_1vsN(bank, fv[0], n_cand=N_CAND)
    return ov.cpu().numpy(), yaw.cpu().numpy()

  host_query()
  ov_d, yaw_d = device_route()
  assert np.array_equal(ov_h.view(np.uint32), ov_d.view(np.uint32)) and np.array_equal(yaw_h, yaw_d)
  t_host = host_median_ms(host_query, args.reps, args.warmup)
  t_dev = host_median_ms(device_route, args.reps, args.warmup)
  res['query_1101'] = {'query_cloud_probs_vs_bank_host_ms': t_host, 'upload_five_calls_leg_heads_ms': t_dev,
                       'speedup': t_dev / t_host}
  eng.check()
  eng.close()
  line = json.dumps(res)
  print(line)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
