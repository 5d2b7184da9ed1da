"""The float64 ICP model (oracle/icp.py) recovers known transforms, and ends degenerate or short of inliers
instead of producing NaN."""
import math

import numpy as np
import pytest

from icp_cases import (GATE_ROTATION_DEG, GATE_TRANSLATION, KITTI_TRANSFORMS, STREET_LEFT, STREET_RIGHT, kitti_pair,
                       street_pair, street_pose)
from oracle import icp
from oracle import projection as P
from overlapnet_b200 import gt
from overlapnet_b200.registration import pose_error, seed_pose


def images(points):
  r, v, _, _ = P.range_projection(np.asarray(points, np.float32))
  return v.astype(np.float32), P.gen_normal_map(r, v).astype(np.float32)


def run(left, right, init):
  vt, nt = images(left)
  vs, ns = images(right)
  return icp.register(vs, ns, vt, nt, init, icp.geometry())


def yaw_seed_of(T, Wf=360):
  return seed_pose(gt.yaw_bin(np.eye(4), T, Wf), Wf)


@pytest.mark.parametrize('yaw_deg,t', KITTI_TRANSFORMS)
def test_recovers_kitti_transforms_from_the_yaw_seed(yaw_deg, t):
  left, right, T = kitti_pair(yaw_deg, t)
  res = run(left, right, yaw_seed_of(T))
  te, re = pose_error(res['pose'], T)
  assert res['status'] in (icp.CONVERGED, icp.MAX_ITERATIONS)
  assert te < GATE_TRANSLATION and math.degrees(re) < GATE_ROTATION_DEG, (te, math.degrees(re))


def test_near_half_turn_needs_the_yaw_seed():
  """The paper's comparison in miniature: at 179 degrees ICP from the identity does not find the loop."""
  left, right, T = kitti_pair(179.0, (1.0, 1.0, 0.0))
  te, re = pose_error(run(left, right, np.eye(4))['pose'], T)
  assert math.degrees(re) > 10.0
  te, re = pose_error(run(left, right, yaw_seed_of(T))['pose'], T)
  assert te < GATE_TRANSLATION and math.degrees(re) < GATE_ROTATION_DEG


@pytest.mark.parametrize('k', range(len(STREET_RIGHT)))
def test_recovers_street_scene_pairs(k):
  left, right, T = street_pair(k)
  assert np.linalg.norm(T[:2, 3]) <= 3.0
  res = run(left, right, yaw_seed_of(T))
  te, re = pose_error(res['pose'], T)
  assert te < GATE_TRANSLATION and math.degrees(re) < GATE_ROTATION_DEG, (te, math.degrees(re))


def test_ground_plane_only_is_degenerate():
  from overlapnet_b200.synth import street_scene_cloud
  left = street_scene_cloud(street_pose(*STREET_LEFT), 7, ground_only=True)
  right = street_scene_cloud(street_pose(*STREET_RIGHT[0]), 7, ground_only=True)
  res = run(left, right, np.eye(4))
  assert res['status'] == icp.DEGENERATE and res['iterations'] == 1
  assert np.all(np.isfinite(res['pose']))


def test_empty_target_has_too_few_inliers():
  left, right, T = kitti_pair(0.0, (0.5, 0.3, 0.0))
  vs, ns = images(right)
  empty_v, empty_n = np.full_like(vs, -1.0), np.full_like(ns, -1.0)
  res = icp.register(vs, ns, empty_v, empty_n, np.eye(4), icp.geometry())
  assert res['status'] == icp.TOO_FEW_INLIERS and res['inliers'] == 0 and res['valid'] > 0
  assert np.all(np.isfinite(res['pose']))


def test_distance_schedule():
  d = icp.distances(dict(icp.DEFAULTS))
  assert len(d) == 30 and d[0] == 2.0 and d[-1] == 0.3
  assert all(a >= b for a, b in zip(d, d[1:]))
  k = next(i for i, x in enumerate(d) if x == 0.3)
  assert 2.0 * 0.8 ** (k - 1) > 0.3 >= 2.0 * 0.8 ** k * (1 + 1e-12)
