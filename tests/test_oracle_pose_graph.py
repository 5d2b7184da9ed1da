"""The float64 pose-graph model (oracle/pose_graph.py): Log / Exp, J_l^-1 and the edge Jacobians against central
differences, the gradient against the cost, a known answer and the robust kernel against false loops."""
import numpy as np
import pytest

from oracle import pose_graph as P
from overlapnet_b200 import synth
from overlapnet_b200.pose_graph import trajectory_error


def random_pose(rng, scale=5.0):
  T = np.eye(4)
  T[:3, :3] = P.rodrigues(rng.normal(0, 1, 3))
  T[:3, 3] = rng.normal(0, scale, 3)
  return T


@pytest.mark.parametrize('angle', [0.0, 1e-9, 1.0, np.pi - 1e-6, np.pi])
def test_log_exp_round_trip(angle):
  rng = np.random.default_rng(0)
  for _ in range(5):
    k = rng.normal(0, 1, 3)
    phi = angle * k / np.linalg.norm(k)
    got = P.log_so3(P.exp_so3(phi))
    if angle == np.pi and np.allclose(got, -phi, atol=1e-7):
      continue                  # at pi, phi and -phi are the same rotation
    np.testing.assert_allclose(got, phi, atol=1e-9, rtol=0)
    np.testing.assert_allclose(P.exp_so3(got), P.exp_so3(phi), atol=1e-12)


@pytest.mark.parametrize('angle', [1e-4, 0.5, 2.0, 3.0])
def test_jl_inv_matches_central_differences(angle):
  # Log(R(dw) R(phi)) = phi + J_l^-1(phi) dw + O(dw^2)
  rng = np.random.default_rng(1)
  k = rng.normal(0, 1, 3)
  phi = angle * k / np.linalg.norm(k)
  h = 1e-6
  J = np.stack([(P.log_so3(P.exp_so3(h * np.eye(3)[c]) @ P.exp_so3(phi)) -
                 P.log_so3(P.exp_so3(-h * np.eye(3)[c]) @ P.exp_so3(phi))) / (2 * h) for c in range(3)], 1)
  np.testing.assert_allclose(P.jl_inv(phi), J, rtol=1e-6, atol=1e-7)


def test_edge_jacobians_match_central_differences():
  rng = np.random.default_rng(2)
  h = 1e-6
  for _ in range(10):
    Ta, Tb, Z = random_pose(rng), random_pose(rng), random_pose(rng)
    _, A = P.jacobian(Ta, Tb, Z)
    for which, want in (('a', -A), ('b', A)):
      num = np.empty((6, 6))
      for c in range(6):
        d = h * np.eye(6)[c]
        if which == 'a':
          ep, _ = P.residual(P.update(Ta, d), Tb, Z)
          em, _ = P.residual(P.update(Ta, -d), Tb, Z)
        else:
          ep, _ = P.residual(Ta, P.update(Tb, d), Z)
          em, _ = P.residual(Ta, P.update(Tb, -d), Z)
        num[:, c] = (ep - em) / (2 * h)
      np.testing.assert_allclose(want, num, rtol=1e-6, atol=1e-6 * np.abs(want).max())


def test_gradient_matches_central_differences_of_the_cost():
  g, _ = synth.pose_graph_scene(30, 4, seed=3, n_false=2, init_noise=(1.0, 0.1))
  phi = 25.0
  F, _, s, grad, _ = P.linearize(g, g['poses'], phi)
  assert np.any(s[29:] < 0.9)                      # the Geman-McClure loops are away from their quadratic zone
  h = 1e-6
  for i in (1, 7, 29):
    for c in range(6):
      d = h * np.eye(6)[c]
      Tp, Tm = g['poses'].copy(), g['poses'].copy()
      Tp[i], Tm[i] = P.update(Tp[i], d), P.update(Tm[i], -d)
      num = (P.evaluate(g, Tp, phi)[0] - P.evaluate(g, Tm, phi)[0]) / (2 * h)
      assert abs(num - grad[i, c]) <= 1e-6 * max(1.0, abs(grad).max()), (i, c, num, grad[i, c])


def test_known_answer():
  g, gt = synth.pose_graph_scene(300, 20, seed=1)
  r = P.optimize(g)
  assert r['status'] == 'converged'
  assert r['final_cost'] < 1e-16
  err = trajectory_error(r['poses'], gt)
  assert err['translation_max_m'] < 1e-8
  assert np.deg2rad(err['rotation_max_deg']) < 1e-9


def test_false_loops_are_switched_off():
  clean, gt = synth.pose_graph_scene(300, 20, seed=1)
  dirty, _ = synth.pose_graph_scene(300, 20, seed=1, n_false=5)
  base = trajectory_error(P.optimize(clean)['poses'], gt)
  r = P.optimize(dirty)
  s = r['scale'][299:]
  assert np.all(s[:20] > 0.9) and np.all(s[20:] < 0.1), s
  err = trajectory_error(r['poses'], gt)
  assert err['translation_max_m'] - base['translation_max_m'] < 1e-3
  ls = trajectory_error(P.optimize(dirty, {'phi': np.inf})['poses'], gt)
  assert ls['translation_max_m'] > 10 * max(err['translation_max_m'], 1e-3)
