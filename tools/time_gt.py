"""Timing of the all-pairs ground truth (gt.overlap_yaw_all_pairs / ovn_gt_pairs_count) on a synthetic
KITTI-shaped sequence: ``--scans`` clouds of 124 668 points (synth.kitti_like_cloud) on a trajectory of
two laps around a circle, so that revisits overlap and pairs across the circle are pruned.

Prints, as one JSON line:
  * all_pairs: wall time of overlap_yaw_all_pairs for every frame (upload, frame images, counts, host yaw
    bins), pairs/s and pair-points/s (reference points projected per second, pruned pairs included);
  * device: CUDA-event time of ovn_gt_pairs_count alone on the resident sequence, its pairs/s and points/s;
  * host_yaw_bins_s: the scalar host loop of the yaw bins alone (part of all_pairs, overlapped with the device);
  * the pruned fraction;
  * per_frame: overlap_yaw_from_clouds (the com_overlap_yaw path) with in-memory clouds, per frame, over
    ``--per-frame`` frames, and the speed-up of all-pairs over running it for every frame;
  * whether those frames' rows are identical in both paths;
  * the card's name and power limit, and SM clocks sampled during the all-pairs run.

  python tools/time_gt.py [--scans 300] [--per-frame 3]
"""
import argparse
import json
import os
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import gpu_timing
from overlapnet_b200 import gt, synth


class ClockSampler:
  """SM clock (MHz) of the current device every 0.5 s inside the ``with`` block; the thread ends when the block
  does."""

  def __init__(self):
    self.samples, self._stop, self._device = [], threading.Event(), torch.cuda.current_device()
    self._t = threading.Thread(target=self._run, daemon=True)

  def _run(self):
    while not self._stop.is_set():
      v = gpu_timing.nvidia_smi(('clocks.sm',), self._device)[0].split()
      if v and v[0].isdigit():
        self.samples.append(int(v[0]))
      self._stop.wait(0.5)

  def __enter__(self):
    self._t.start()
    return self

  def __exit__(self, *exc):
    self._stop.set()
    self._t.join()


def trajectory(n, radius=80.0, laps=2, seed=0):
  rng = np.random.default_rng(seed)
  poses = np.tile(np.eye(4), (n, 1, 1))
  for i in range(n):
    th = 2 * np.pi * laps * i / n
    c, s = np.cos(th + np.pi / 2), np.sin(th + np.pi / 2)
    poses[i, :3, :3] = [[c, -s, 0], [s, c, 0], [0, 0, 1]]
    poses[i, :3, 3] = [radius * np.cos(th) + rng.normal(0, 1.0), radius * np.sin(th) + rng.normal(0, 1.0),
                       rng.normal(0, 0.2)]
  return poses


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--scans', type=int, default=300)
  ap.add_argument('--points', type=int, default=synth.KITTI_POINTS)
  ap.add_argument('--per-frame', type=int, default=3)
  args = ap.parse_args()
  gpu_timing.require_cuda('time_gt.py')
  torch.cuda.set_device(0)
  n = args.scans
  clouds = [synth.kitti_like_cloud(i, n_points=args.points) for i in range(n)]
  poses = trajectory(n)
  total_points = sum(c.shape[0] for c in clouds)
  gt.overlap_yaw_all_pairs(clouds[:4], poses[:4])                 # warm-up: modules, workspaces
  gt.overlap_yaw_from_clouds(clouds[:4], poses[:4], 0)

  torch.cuda.synchronize()
  with ClockSampler() as clk:
    t0 = time.perf_counter()
    res = gt.overlap_yaw_all_pairs(clouds, poses)
    torch.cuda.synchronize()
    t_all = time.perf_counter() - t0
  rows = gt.all_pairs_rows(res)

  # the counting alone, on the resident sequence (what ovn_gt_pairs_count costs per call)
  eng = gt._engine(3.0, -25.0, 64, 900, 50)
  batch = eng.upload_clouds(clouds)
  radius = eng.gt_scan_radius(batch)
  d_pose = torch.from_numpy(poses.reshape(n, 16).copy()).cuda()
  d_inv = torch.from_numpy(np.stack([np.linalg.inv(p) for p in poses]).reshape(n, 16)).cuda()
  cur = eng.gt_range(batch)
  counts = torch.empty((n, n), dtype=torch.int32, device='cuda')
  eng.gt_pairs_count(batch, d_pose, radius, cur, d_inv, counts=counts)
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  reps = 3
  e0.record()
  for _ in range(reps):
    eng.gt_pairs_count(batch, d_pose, radius, cur, d_inv, counts=counts)
  e1.record()
  torch.cuda.synchronize()
  t_dev = e0.elapsed_time(e1) / 1e3 / reps
  assert np.array_equal(counts.cpu().numpy(), res.counts)
  del batch, cur, counts

  # the host part: yaw bins of every pair, scalar pose arithmetic as com_overlap_yaw does it
  t0 = time.perf_counter()
  inv = [np.linalg.inv(p) for p in poses]
  for j in range(n):
    for r in range(n):
      gt.yaw_bin(inv[j], poses[r])
  t_yaw = time.perf_counter() - t0

  frames = np.linspace(0, n - 1, args.per_frame).astype(int)
  identical = True
  t_pf = []
  for f in frames:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m = gt.overlap_yaw_from_clouds(clouds, poses, int(f))
    torch.cuda.synchronize()
    t_pf.append(time.perf_counter() - t0)
    identical &= bool(np.array_equal(m, rows[f * n:(f + 1) * n]))
  pairs = n * n
  out = {
      'card': gpu_timing.card(), 'sm_clock_mhz_sampled': [min(clk.samples, default=0), max(clk.samples, default=0)],
      'scans': n, 'points_per_scan': args.points, 'pairs': pairs,
      'pruned_fraction': round(res.n_pruned / pairs, 4), 'pairs_with_overlap': int(np.count_nonzero(res.counts)),
      'all_pairs_s': round(t_all, 3), 'all_pairs_pairs_per_s': round(pairs / t_all),
      'all_pairs_points_per_s': float('%.4g' % (n * total_points / t_all)),
      'device_count_s': round(t_dev, 4), 'device_pairs_per_s': round(pairs / t_dev),
      'device_points_per_s': float('%.4g' % (n * total_points / t_dev)),
      'host_yaw_bins_s': round(t_yaw, 3),
      'per_frame_s': round(float(np.median(t_pf)), 3),
      'per_frame_points_per_s': float('%.4g' % (total_points / np.median(t_pf))),
      'speedup_vs_per_frame': round(float(np.median(t_pf)) * n / t_all, 1),
      'per_frame_rows_identical': identical,
  }
  print(json.dumps(out))


if __name__ == '__main__':
  main()
