"""Host logic of loop-closure registration: the yaw seed, the pose error, the registration summary and the
command line."""
import math

import numpy as np
import pytest

from conftest import load_golden
from overlapnet_b200 import gt, lcd_eval
from overlapnet_b200.registration import pose_error, seed_pose, seed_yaw

TILT_ALLOWANCE = 2.5e-4     # rad: the Euler yaw of the golden poses (tilts up to 1.3 deg), DESIGN section 7


def yaw_bin_expression(yaw, Wf):
  return int(- (yaw / np.pi) * Wf // 2 + Wf // 2)          # gt.yaw_bin's own expression


@pytest.mark.parametrize('Wf', [360, 225, 405])
def test_seed_round_trips_every_bin(Wf):
  for b in range(Wf):
    assert yaw_bin_expression(float(seed_yaw(b, Wf)), Wf) == b
    T = seed_pose(b, Wf)
    assert gt.yaw_bin(np.eye(4), T, Wf) == b


@pytest.mark.parametrize('Wf', [360, 225, 405])
def test_seed_lies_within_half_a_bin_of_the_golden_yaws(Wf):
  poses = load_golden('gt_overlap_yaw')['poses']
  for i in range(len(poses)):
    cur_inv = np.linalg.inv(poses[i])
    for j in range(len(poses)):
      rel = cur_inv @ poses[j]
      yaw = math.atan2(rel[1, 0], rel[0, 0])
      b = gt.yaw_bin(cur_inv, poses[j], Wf)
      d = (float(seed_yaw(b, Wf)) - yaw + math.pi) % (2 * math.pi) - math.pi
      assert abs(d) <= math.pi / Wf + TILT_ALLOWANCE, (i, j, d)


def test_pose_error():
  T = np.eye(4)
  T[:3, 3] = (3.0, 4.0, 0.0)
  te, re = pose_error(T, np.eye(4))
  assert te == pytest.approx(5.0) and re == 0.0
  c, s = math.cos(0.3), math.sin(0.3)
  R = np.eye(4)
  R[1:3, 1:3] = [[c, -s], [s, c]]
  G = np.eye(4)
  G[:3, 3] = (1.0, 2.0, 3.0)
  te, re = pose_error(G @ R, G)
  assert te == pytest.approx(0.0, abs=1e-12) and re == pytest.approx(0.3, abs=1e-12)
  te, re = pose_error(np.stack([G @ R, G]), np.stack([G, G]))
  assert te.shape == (2,) and re[0] == pytest.approx(0.3) and re[1] == pytest.approx(0.0, abs=1e-12)
  assert pose_error(seed_pose(0, 360), np.eye(4))[1] == pytest.approx(math.radians(179.5), abs=1e-12)


def test_registration_summary_on_crafted_arrays():
  # five rows: 0-2 true positives, 3 a false positive, 4 without a record
  top_ov = np.array([[0.9], [0.8], [0.7], [0.6], [-1.0]], np.float32)
  top_idx = np.array([[1], [2], [3], [4], [-1]], np.int32)
  gt_top = np.array([[0.8], [0.7], [0.5], [0.1], [-1.0]])
  gt_best = np.array([0.8, 0.7, 0.5, 0.5, -1.0])
  err = np.full((5, 2, 2), np.nan)
  err[0] = [[0.1, 0.5], [0.2, 1.0]]            # both seeds succeed
  err[1] = [[0.4, 1.9], [3.0, 40.0]]           # the yaw seed succeeds
  err[2] = [[0.6, 0.1], [0.1, 0.1]]            # the identity succeeds
  err[3] = [[0.1, 0.1], [0.1, 0.1]]
  frac = np.array([[0.5, 0.5], [0.2, 0.1], [0.4, 0.4], [0.9, 0.9], [np.nan, np.nan]])
  s = lcd_eval.registration_summary(top_ov, top_idx, gt_top, gt_best, np.array([0, 1, 2]), err, frac, 0.3, 0.3)
  assert s['true_positives'] == 3
  assert s['success_rate_yaw'] == pytest.approx(2 / 3) and s['success_rate_identity'] == pytest.approx(2 / 3)
  assert s['median_error_translation_m_yaw'] == pytest.approx(0.4)
  assert s['max_error_translation_m_yaw'] == pytest.approx(0.6)
  assert s['median_error_rotation_deg_yaw'] == pytest.approx(0.5)
  assert s['max_error_rotation_deg_yaw'] == pytest.approx(1.9)
  assert (s['success_translation_m'], s['success_rotation_deg'], s['min_inlier_fraction']) == (0.5, 2.0, 0.3)
  # declared at > 0.3 with a fraction >= 0.3: rows 0, 2 (correct) and 3 (wrong); positives: rows 0-3
  assert s['precision_at_operating_point_verified'] == pytest.approx(2 / 3)
  assert s['recall_at_operating_point_verified'] == pytest.approx(2 / 4)
  empty = lcd_eval.registration_summary(top_ov, top_idx, gt_top, gt_best, np.zeros(0, np.int64), err, frac)
  assert math.isnan(empty['success_rate_yaw']) and math.isnan(empty['median_error_translation_m_yaw'])


def test_register_arguments():
  a = lcd_eval.parse_args([])
  assert a.register is False and a.min_inlier_fraction == 0.3
  a = lcd_eval.parse_args(['cfg.yml', '--register', '--min-inlier-fraction', '0.5'])
  assert a.register is True and a.min_inlier_fraction == 0.5 and a.config == 'cfg.yml'
  with pytest.raises(SystemExit):
    lcd_eval.parse_args(['--register', '--min-inlier-fraction', '1.5'])


def test_street_scene_is_seeded_and_level_ground_is_flat():
  from overlapnet_b200.synth import street_scene_cloud
  T = np.eye(4)
  T[:3, 3] = (2.0, 3.0, 1.73)
  a = street_scene_cloud(T, seed=4)
  assert a.dtype == np.float32 and a.shape[1] == 4
  np.testing.assert_array_equal(a, street_scene_cloud(T, seed=4))
  assert not np.array_equal(a, street_scene_cloud(T, seed=5))
  r = np.linalg.norm(a[:, :3].astype(np.float64), axis=1)
  assert r.max() < 80.0 + 1e-3
  g = street_scene_cloud(T, seed=4, ground_only=True)
  assert np.all(g[:, 2] == np.float32(-1.73))
  noisy = street_scene_cloud(T, seed=4, noise=0.02)
  assert noisy.shape[0] > 0.9 * a.shape[0]
