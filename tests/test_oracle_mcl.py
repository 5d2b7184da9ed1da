"""The NumPy model of the Monte Carlo localization filter (oracle/mcl.py) on its own: Philox against published
answers, resampling on hand-made weights, the circular estimate across +-180 degrees and the expected yaw bin
against gt.yaw_bin."""
import math

import numpy as np
import pytest

from oracle import mcl as om
from overlapnet_b200 import gt


def test_philox_known_answers():
  """Random123's known-answer vectors for Philox4x32-10."""
  assert [hex(v) for v in om.philox(0, [[0, 0, 0, 0]])[0]] == ['0x6627e8d5', '0xe169c58d', '0xbc57ac4c', '0x9b00dbd8']
  assert [hex(v) for v in om.philox(2 ** 64 - 1, [[2 ** 32 - 1] * 4])[0]] == \
      ['0x408f276d', '0x41c83b0e', '0xa20bc7c6', '0x6d5451fd']
  key = 0xa4093822 | (0x299f31d0 << 32)
  assert [hex(v) for v in om.philox(key, [[0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344]])[0]] == \
      ['0xd16cfe09', '0x94fdcceb', '0x5001e420', '0x24126ea1']


def test_uniforms_lie_in_the_open_interval():
  top = np.uint32(2 ** 32 - 1)
  assert om.u53([0], [0])[0] == 2.0 ** -54
  assert om.u53([top], [top])[0] == 1.0 - 2.0 ** -53
  w = om.philox(5, om.counters(np.arange(100000), 3, om.STREAM_MOTION, 0))
  u = om.u53(w[:, 0], w[:, 1])
  assert u.min() > 0 and u.max() < 1 and abs(u.mean() - 0.5) < 0.01
  n0, n1 = om.box_muller(w)
  assert abs(n0.std() - 1) < 0.02 and abs(n1.mean()) < 0.02


@pytest.mark.parametrize('w,u0,want', [
    ([0.25, 0.25, 0.25, 0.25], 0.5, [0, 1, 2, 3]),
    ([1.0, 0.0, 0.0, 0.0], 0.3, [0, 0, 0, 0]),
    ([0.0, 0.0, 0.0, 1.0], 0.3, [3, 3, 3, 3]),
    ([0.5, 0.0, 0.5, 0.0], 0.9, [0, 0, 2, 2]),
    ([0.5, 0.5, 0.0], 0.999999, [0, 1, 1]),
    ([0.1, 0.6, 0.3], 0.5, [1, 1, 2]),
    ([0.25, 0.25, 0.25, 0.25], 0.0, [0, 1, 2, 3]),       # thresholds exactly on the steps: C_i > t
])
def test_systematic_resampling_on_hand_made_weights(w, u0, want):
  assert list(om.systematic(np.cumsum(w), u0)) == want


def test_systematic_resampling_keeps_expected_counts():
  rng = np.random.default_rng(0)
  w = rng.random(1000)
  w /= w.sum()
  a = om.systematic(np.cumsum(w), 0.37)
  counts = np.bincount(a, minlength=w.size)
  assert np.all(np.abs(counts - w * w.size) < 1 + 1e-9)


def test_circular_estimate_across_180_degrees():
  th = np.radians([179.0, -179.0, 178.0, -178.0])
  w = np.full(4, 0.25)
  e = om.estimate(w, np.zeros(4), np.zeros(4), th)
  assert abs(abs(e['theta']) - math.pi) < 1e-12                  # not 0, as a plain mean would give
  e = om.estimate(np.array([0.7, 0.3]), np.array([0.0, 10.0]), np.array([1.0, 1.0]), np.radians([179.0, -179.0]))
  assert abs(e['x'] - 3.0) < 1e-12 and abs(math.degrees(e['theta']) - 179.6) < 1e-2
  assert abs(om.estimate(np.full(4, 0.25), *np.zeros((3, 4)))['ess'] - 4.0) < 1e-12


def test_expected_bin_equals_gt_yaw_bin_on_planar_poses():
  rng = np.random.default_rng(1)
  for width in (360, 180, 90):
    for _ in range(500):
      a, b = rng.uniform(-math.pi, math.pi, 2)

      def pose(t):
        T = np.eye(4)
        T[:2, :2] = [[math.cos(t), -math.sin(t)], [math.sin(t), math.cos(t)]]
        T[:2, 3] = rng.uniform(-50, 50, 2)
        return T
      cur, ref = pose(a), pose(b)                               # LEFT = the keyframe (current), RIGHT = the query
      want = gt.yaw_bin(np.linalg.inv(cur), ref, width) % width
      got = om.expected_bin(om.wrap_pi(b - a), width)
      psi = om.wrap_pi(b - a)
      edge = abs((-(psi / math.pi) * width * 0.5) - round(-(psi / math.pi) * width * 0.5)) < 1e-9
      assert got == want or edge, (width, a, b, got, want)


def test_loglik_outside_and_inside():
  kf_th = np.array([0.0, 1.0])
  ll = om.loglik(np.array([-1, 0, 1]), np.array([0.0, 0.0, 1.0]), kf_th, np.array([0, 1]),
                 np.array([1.0, 0.5], np.float32), np.array([180 - 180, 180 - 180], np.int32), 360, 0.1, 0.2)
  assert ll[0] == -0.5 * (1 / 0.1) ** 2 - 0.5 * (math.pi / 0.2) ** 2      # O = 0, D = pi
  assert ll[1] == 0.0                                                     # O = 1, bins agree
  assert abs(ll[2] - (-0.5 * (0.5 / 0.1) ** 2)) < 1e-12


def test_normalize_is_shift_invariant():
  lw = np.array([-1000.0, -1001.0, -1002.0])
  a, w = om.normalize(lw)
  b, v = om.normalize(lw + 700)
  assert abs(w.sum() - 1) < 1e-12 and np.allclose(a, b, atol=1e-12) and np.allclose(w, v, atol=1e-12)


def test_cpu_filter_converges_on_the_scenario():
  """The oracle filter on the GPU convergence test's scenario, at 10^4 particles and 80 steps."""
  from overlapnet_b200 import mcl
  poses = om.scenario()
  kfi, qi = mcl.split_sequence(len(poses), 2)
  kf, truth = poses[kfi], poses[qi]
  idx = mcl.MapIndex(kf[:, :2], 0.5, 3.0)
  f = om.Filter(kf, idx.raster, idx.x0, idx.y0, idx.cell)
  f.init_global(10000, 0, 1.0)
  odom = mcl.odometry(truth)
  err = []
  for t in range(80):
    e = f.step(odom[t], (0.1, 0.1, math.radians(1.0)), om.fake_sensor(truth[t], kf), 0.05, math.radians(10.0))
    err.append(math.hypot(e['x'] - truth[t, 0], e['y'] - truth[t, 1]))
  assert 0 <= mcl.convergence_step(err, 2.0) <= 50
