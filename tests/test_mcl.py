"""Host logic of Monte Carlo localization (overlapnet_b200.mcl): the map raster against brute force, the map / query
split, the odometry from poses, the convergence metric and the command line."""
import math

import numpy as np
import pytest

from overlapnet_b200 import mcl


def brute_raster(xy, cell, max_distance):
  idx = mcl.MapIndex(xy, cell, max_distance)
  cx = idx.x0 + (np.arange(idx.cols) + 0.5) * cell
  cy = idx.y0 + (np.arange(idx.rows) + 0.5) * cell
  out = np.full((idx.rows, idx.cols), -1, np.int32)
  for r in range(idx.rows):
    for c in range(idx.cols):
      d2 = (xy[:, 0] - cx[c]) ** 2 + (xy[:, 1] - cy[r]) ** 2
      k = int(np.argmin(d2))                                    # the first minimum: ties to the lowest index
      if d2[k] <= max_distance ** 2:
        out[r, c] = k
  return idx, out


@pytest.mark.parametrize('seed,K,cell,md', [(0, 1, 0.5, 2.0), (1, 7, 0.5, 3.0), (2, 40, 1.0, 2.5), (3, 12, 0.3, 0.0)])
def test_raster_equals_brute_force(seed, K, cell, md):
  rng = np.random.default_rng(seed)
  xy = rng.uniform(-10, 10, (K, 2))
  idx, want = brute_raster(xy, cell, md)
  assert np.array_equal(idx.raster, want)
  assert idx.x0 == xy[:, 0].min() - md and idx.y0 == xy[:, 1].min() - md
  assert idx.cols * cell >= np.ptp(xy[:, 0]) + 2 * md and idx.rows * cell >= np.ptp(xy[:, 1]) + 2 * md


def test_raster_ties_go_to_the_lowest_index():
  # cell centres on the grid 0.5 + j: keyframes mirrored about the centre (2.5, 2.5) are equally far from it
  xy = np.array([[3.5, 2.5], [1.5, 2.5], [2.5, 3.5], [2.5, 1.5], [1.5, 2.5]])
  idx, want = brute_raster(xy, 1.0, 5.0)
  assert np.array_equal(idx.raster, want)
  r, c = int((2.5 - idx.y0) // 1.0), int((2.5 - idx.x0) // 1.0)
  assert idx.raster[r, c] == 0                                # four keyframes at distance 1: the lowest wins
  assert not (idx.raster == 4).any()                          # the duplicate of keyframe 1 never wins


def test_lookup_outside_the_raster_is_minus_one():
  from oracle.mcl import lookup
  idx = mcl.MapIndex(np.array([[0.0, 0.0], [10.0, 0.0]]), 0.5, 1.0)
  k = lookup([0.0, 10.0, 5.0, -1.01, 11.01, float('nan')], [0.0] * 6, idx.raster, idx.x0, idx.y0, idx.cell)
  assert list(k) == [0, 1, -1, -1, -1, -1]


def test_split_sequence():
  kf, q = mcl.split_sequence(23, 5)
  assert list(kf) == [0, 5, 10, 15, 20] and list(q) == [2, 7, 12, 17, 22]
  kf, q = mcl.split_sequence(7, 2)
  assert list(kf) == [0, 2, 4, 6] and list(q) == [1, 3, 5]
  assert not set(kf) & set(q)
  for s in (1, 0, -3):
    with pytest.raises(ValueError, match='at least 2'):
      mcl.split_sequence(10, s)


def _pose(x, y, t):
  T = np.eye(4)
  T[:2, :2] = [[math.cos(t), -math.sin(t)], [math.sin(t), math.cos(t)]]
  T[0, 3], T[1, 3] = x, y
  return T


def test_odometry_recomposes_the_poses():
  rng = np.random.default_rng(4)
  poses = np.array([_pose(*rng.uniform(-50, 50, 2), rng.uniform(-math.pi, math.pi)) for _ in range(30)])
  p = mcl.planar(poses)
  odom = mcl.odometry(p)
  assert np.all(odom[0] == 0)
  for i in range(1, len(p)):
    rel = np.linalg.inv(poses[i - 1]) @ poses[i]                # the relative pose in the previous frame
    assert np.allclose(odom[i], [rel[0, 3], rel[1, 3], math.atan2(rel[1, 0], rel[0, 0])], atol=1e-9)
  assert np.allclose(p[:, 2], [math.atan2(T[1, 0], T[0, 0]) for T in poses])


@pytest.mark.parametrize('err,want', [
    ([5, 3, 1, 0.5, 0.2], 2), ([1, 1, 1], 0), ([1, 3, 1, 1], 2), ([1, 1, 3], -1), ([], 0),
    ([0.1, 2.0, 0.1], 2),                                       # below, strictly
    ([0.1, float('nan'), 0.1], 2),
])
def test_convergence_step(err, want):
  assert mcl.convergence_step(err, 2.0) == want


def test_summary_over_runs():
  pos = np.array([[5.0, 1.0, 1.0], [5.0, 5.0, 5.0], [0.5, 0.5, 1.5]])
  yaw = np.radians(np.array([[9.0, 1.0, 1.0], [9.0, 9.0, 9.0], [2.0, 2.0, 2.0]]))
  conv = [mcl.convergence_step(p, 2.0) for p in pos]
  s = mcl.summarize(pos, yaw, conv, 2.0)
  assert conv == [1, -1, 0] and abs(s['success_rate'] - 2 / 3) < 1e-12
  after = np.array([1.0, 1.0, 0.5, 0.5, 1.5])
  assert abs(s['position_error_mean'] - after.mean()) < 1e-12
  assert abs(s['position_error_rms'] - math.sqrt((after ** 2).mean())) < 1e-12
  assert abs(s['yaw_error_mean_deg'] - np.mean([1, 1, 2, 2, 2])) < 1e-9


def test_cli_parsing_and_refusals():
  a = mcl.parse_args([])
  assert a.config == 'config/demo.yml' and a.keyframe_stride == 5 and a.particles == 100000 and a.runs == 5
  assert a.cell == 0.5 and a.max_distance == 5.0 and a.converged_m == 2.0
  a = mcl.parse_args(['x.yml', '--keyframe-stride', '2', '--particles', '1000', '--runs', '3', '--sigma-overlap',
                      '0.2', '--sigma-yaw-deg', '5', '--cell', '1', '--max-distance', '4', '--converged-m', '3'])
  assert (a.config, a.keyframe_stride, a.particles, a.runs, a.sigma_overlap, a.sigma_yaw_deg, a.cell,
          a.max_distance, a.converged_m) == ('x.yml', 2, 1000, 3, 0.2, 5.0, 1.0, 4.0, 3.0)
  for bad in (['--keyframe-stride', '1'], ['--particles', '0'], ['--particles', str((1 << 24) + 1)], ['--runs', '0'],
              ['--sigma-overlap', '0'], ['--cell', '-1'], ['--max-distance', '-1']):
    with pytest.raises(SystemExit):
      mcl.parse_args(bad)


def test_semantic_configs_are_refused(tmp_path):
  net = tmp_path / 'net.yml'
  net.write_text('use_class_probabilities: True\n')
  with pytest.raises(Exception, match='class probabilities'):
    mcl.network_config({'Demo3': {'network_config': str(net)}})
  net.write_text('use_class_probabilities: False\n')
  assert mcl.network_config({'Demo3': {'network_config': str(net)}})['use_class_probabilities'] is False
