"""Graph builders, the Python-side refusals that mirror the library's, parameter overrides and the trajectory error
of overlapnet_b200.pose_graph (no GPU)."""
import numpy as np
import pytest

from oracle import pose_graph as P
from overlapnet_b200 import pose_graph as pg, synth


def test_chain_graph_composes_the_odometry():
  rng = np.random.default_rng(0)
  odo = np.stack([P.update(np.eye(4), rng.normal(0, 0.3, 6)) for _ in range(5)])
  T0 = P.update(np.eye(4), rng.normal(0, 1, 6))
  g = pg.chain_graph(odo, (np.array([[0, 4]]), np.eye(4)[None]), T0=T0)
  assert g['poses'].shape == (6, 4, 4) and g['edges'].tolist() == [[0, 1], [1, 2], [2, 3], [3, 4], [4, 5], [0, 4]]
  np.testing.assert_array_equal(g['poses'][0], T0)
  for k in range(5):
    np.testing.assert_allclose(np.linalg.solve(g['poses'][k], g['poses'][k + 1]), odo[k], atol=1e-12)
  np.testing.assert_allclose(g['weights'][0], pg.sigma_weights(pg.ODOMETRY_SIGMA))
  np.testing.assert_allclose(g['weights'][-1], pg.sigma_weights(pg.LOOP_SIGMA))
  np.testing.assert_allclose(pg.sigma_weights((1.0, 0.2))[[0, 3]], [1 / np.deg2rad(1.0) ** 2, 25.0])
  assert pg.check_graph(g)['edges'].dtype == np.int32


def _bad(g, key, fn):
  g = {k: np.array(v, copy=True) for k, v in g.items()}
  fn(g[key])
  return g


REFUSALS = {
    'chain': lambda g: _bad(g, 'edges', lambda e: e.__setitem__((1, 1), 3)),
    'node out of range': lambda g: _bad(g, 'edges', lambda e: e.__setitem__((-1, 1), 99)),
    'a == b': lambda g: _bad(g, 'edges', lambda e: e.__setitem__((-1, 1), e[-1, 0])),
    'pose not finite': lambda g: _bad(g, 'poses', lambda T: T.__setitem__((2, 0, 3), np.nan)),
    'pose bottom row': lambda g: _bad(g, 'poses', lambda T: T.__setitem__((2, 3, 0), 1e-9)),
    'measurement not finite': lambda g: _bad(g, 'measurements', lambda T: T.__setitem__((0, 1, 1), np.inf)),
    'weight <= 0': lambda g: _bad(g, 'weights', lambda w: w.__setitem__((3, 2), 0.0)),
    'weight not finite': lambda g: _bad(g, 'weights', lambda w: w.__setitem__((3, 2), np.nan)),
    'one node': lambda g: {'poses': g['poses'][:1], 'edges': np.zeros((0, 2)), 'measurements': np.zeros((0, 4, 4)),
                           'weights': np.zeros((0, 6))},
    'missing chain edge': lambda g: {'poses': g['poses'], 'edges': g['edges'][1:],
                                     'measurements': g['measurements'][1:], 'weights': g['weights'][1:]},
}


@pytest.mark.parametrize('what', sorted(REFUSALS))
def test_check_graph_mirrors_the_library_refusals(what):
  g, _ = synth.pose_graph_scene(12, 2, seed=0)
  pg.check_graph(g)
  with pytest.raises(ValueError):
    pg.check_graph(REFUSALS[what](g))


def test_parameter_overrides_are_checked():
  p = pg.default_params({'phi': 9.0, 'max_iterations': 3})
  assert p.phi == 9.0 and p.max_iterations == 3 and p.cg_tol == 1e-12 and p.max_cg_iterations == 2000
  d = pg.default_params()
  assert (d.phi, d.lambda0, d.lambda_min, d.lambda_max, d.rel_cost_tol, d.step_tol, d.max_iterations) == \
      (P.DEFAULTS['phi'], 1e-6, 1e-12, 1e12, 1e-10, 1e-10, 50)
  with pytest.raises(KeyError):
    pg.default_params({'lambda': 1.0})


def test_trajectory_error_is_anchored_at_frame_zero():
  _, gt = synth.pose_graph_scene(20, 0, seed=4)
  A = P.update(np.eye(4), [0.1, -0.2, 0.3, 5, 6, 7])
  e = pg.trajectory_error(A @ gt, gt)              # the same trajectory from another origin: no error
  assert e['translation_max_m'] < 1e-9 and e['rotation_max_deg'] < 1e-9
  est = gt.copy()
  est[5, :3, 3] += [0.3, 0.4, 0.0]
  e = pg.trajectory_error(est, gt)
  assert abs(e['translation_max_m'] - 0.5) < 1e-12
  assert abs(e['translation_rmse_m'] - np.sqrt(0.25 / 20)) < 1e-12
  assert e['rotation_max_deg'] < 1e-9
