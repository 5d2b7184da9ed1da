"""Robust pose-graph optimization on the GPU (ovn_pgo_optimize_host): odometry chains closed by loop edges, with a
Geman-McClure kernel on the loops, batched over graphs in one launch.

The model (DESIGN.md section 7, "Pose-graph optimization"):
  nodes     float64 row-major 4x4 poses T_0 .. T_{n-1}; T_0 is fixed.
  update    T <- [R(omega) | v] T with xi = (omega, v), R by Rodrigues, as ICP updates its pose.
  edges     (a, b, Z, w): Z ~ T_a^-1 T_b, w six positive weights in (omega, v) order.  Edges 0 .. n-2 are the chain
            (k, k + 1); every later edge is a loop (a != b).
  residual  E = Z^-1 T_a^-1 T_b, e = (Log(R_E), t_E), chi2 = e^T diag(w) e.
  cost      F = 1/2 sum rho(chi2): rho(x) = x on the chain, rho(x) = phi x / (phi + x) on loops; s = phi / (phi + chi2)
            is the switch of the equivalent switchable constraint, and a loop is kept when s >= 1/2.
  solver    Levenberg-Marquardt on (H + lambda diag(H)) delta = -g, by preconditioned conjugate gradients.
None of the defaults is tuned on KITTI."""
import numpy as np

from . import _cabi

ODOMETRY_SIGMA = (0.2, 0.05)     # degrees, metres: the default weights of a chain edge are 1 / sigma^2
LOOP_SIGMA = (1.0, 0.2)          # degrees, metres: of a loop edge
KEEP_SCALE = 0.5                 # a loop edge is kept when s >= KEEP_SCALE, i.e. chi2 <= phi
STATUS = {v: k for k, v in _cabi.PGO_STATUS.items()}


def default_params(overrides=None):
  """ovn_pgo_default_params with ``overrides`` (a dict) applied; an unknown key raises KeyError."""
  prm = _cabi.PgoParams()
  _cabi.lib().ovn_pgo_default_params(prm)
  for key, value in (overrides or {}).items():
    if key not in dict(prm._fields_):
      raise KeyError('unknown pose-graph parameter %r' % key)
    setattr(prm, key, value)
  return prm


def sigma_weights(sigma):
  """w [6] = 1 / sigma^2 of (rotation sigma in degrees, translation sigma in metres), in (omega, v) order."""
  r, t = np.deg2rad(float(sigma[0])), float(sigma[1])
  return np.array([1 / r ** 2] * 3 + [1 / t ** 2] * 3)


def _rigid_rows(T):
  T = np.asarray(T)
  return np.isfinite(T).all(axis=(-2, -1)) & np.all(T[..., 3, :] == np.array([0.0, 0.0, 0.0, 1.0]), axis=-1)


def check_graph(graph):
  """The library's refusals of one graph, raised here as ValueError before anything reaches the device.  Returns the
  graph with contiguous arrays of the library's types."""
  poses = np.ascontiguousarray(graph['poses'], np.float64)
  edges = np.ascontiguousarray(graph['edges'], np.int64)
  Z = np.ascontiguousarray(graph['measurements'], np.float64)
  w = np.ascontiguousarray(graph['weights'], np.float64)
  if poses.ndim != 3 or poses.shape[1:] != (4, 4):
    raise ValueError('poses must be [n, 4, 4], got %s' % (poses.shape,))
  n = poses.shape[0]
  if not 2 <= n <= _cabi.PGO_MAX_NODES:
    raise ValueError('a graph has 2 .. %d nodes, got %d' % (_cabi.PGO_MAX_NODES, n))
  if edges.ndim != 2 or edges.shape[1] != 2 or Z.shape != (edges.shape[0], 4, 4) or w.shape != (edges.shape[0], 6):
    raise ValueError('edges [E, 2], measurements [E, 4, 4] and weights [E, 6] must agree')
  ne = edges.shape[0]
  if not n - 1 <= ne <= _cabi.PGO_MAX_EDGES:
    raise ValueError('a graph of %d nodes has %d .. %d edges, got %d' % (n, n - 1, _cabi.PGO_MAX_EDGES, ne))
  k = np.arange(n - 1)
  if not (np.array_equal(edges[:n - 1, 0], k) and np.array_equal(edges[:n - 1, 1], k + 1)):
    raise ValueError('the first n - 1 edges must be the chain (k, k + 1)')
  if edges.min() < 0 or edges.max() >= n or np.any(edges[:, 0] == edges[:, 1]):
    raise ValueError('an edge has a node outside [0, %d) or a == b' % n)
  if not _rigid_rows(poses).all():
    raise ValueError('a pose is not finite or its bottom row is not 0 0 0 1')
  if not _rigid_rows(Z).all():
    raise ValueError('a measurement is not finite or its bottom row is not 0 0 0 1')
  if not (np.isfinite(w).all() and (w > 0).all()):
    raise ValueError('every weight must be finite and > 0')
  return {'poses': poses, 'edges': edges.astype(np.int32), 'measurements': Z, 'weights': w}


def chain_graph(odometry, loops=None, odometry_sigma=ODOMETRY_SIGMA, loop_sigma=LOOP_SIGMA, T0=None):
  """A graph of n = len(odometry) + 1 nodes: the chain edges (k, k + 1) measure odometry[k] ~ T_k^-1 T_{k+1}, and
  ``loops`` = (edges [L, 2], measurements [L, 4, 4]) adds loop edges (a, b).  The initial poses are the composed
  odometry T_{k+1} = T_k odometry[k], anchored at ``T0`` (the identity by default).  The weights are
  sigma_weights of ``odometry_sigma`` and ``loop_sigma``."""
  odo = np.asarray(odometry, np.float64).reshape(-1, 4, 4)
  n = odo.shape[0] + 1
  T = np.empty((n, 4, 4))
  T[0] = np.eye(4) if T0 is None else np.asarray(T0, np.float64)
  for k in range(n - 1):
    T[k + 1] = T[k] @ odo[k]
  k = np.arange(n - 1)
  edges = [np.stack([k, k + 1], 1)]
  Z = [odo]
  w = [np.broadcast_to(sigma_weights(odometry_sigma), (n - 1, 6))]
  if loops is not None:
    le = np.asarray(loops[0], np.int64).reshape(-1, 2)
    lz = np.asarray(loops[1], np.float64).reshape(-1, 4, 4)
    edges.append(le)
    Z.append(lz)
    w.append(np.broadcast_to(sigma_weights(loop_sigma), (le.shape[0], 6)))
  return {'poses': T, 'edges': np.concatenate(edges).astype(np.int32), 'measurements': np.concatenate(Z),
          'weights': np.ascontiguousarray(np.concatenate(w))}


def optimize(engine, graphs, params=None, want_gradient=False, want_trace=False):
  """Engine.pose_graph on ``graphs`` (a list, one launch); each result also names its status ('status_name') and,
  for a graph with loops, marks them kept (s >= 1/2, 'loop_kept') with their scales ('loop_scale')."""
  out = engine.pose_graph(graphs, params, want_gradient, want_trace)
  for g, r in zip(graphs, out):
    n = np.asarray(g['poses']).shape[0]
    r['status_name'] = STATUS[r['status']]
    r['loop_scale'] = r['scale'][n - 1:]
    r['loop_kept'] = r['loop_scale'] >= KEEP_SCALE
  return out


def trajectory_error(est, gt):
  """The error of the trajectory ``est`` [n, 4, 4] against ``gt`` [n, 4, 4], anchored at frame 0 with no alignment:
  with A_i = est_0^-1 est_i and B_i = gt_0^-1 gt_i, the translation error of frame i is ||t(A_i) - t(B_i)|| (metres)
  and its rotation error the angle of R(B_i)^T R(A_i) (degrees, registration.pose_error's angle).  Returns a dict
  of translation_rmse_m, translation_max_m, rotation_rmse_deg and rotation_max_deg over every frame."""
  from .registration import pose_error
  est = np.asarray(est, np.float64)
  gt = np.asarray(gt, np.float64)
  A = np.linalg.solve(est[0], est)
  B = np.linalg.solve(gt[0], gt)
  t = np.linalg.norm(A[:, :3, 3] - B[:, :3, 3], axis=-1)
  Ar, Br = A.copy(), B.copy()
  Ar[:, :3, 3] = 0.0
  Br[:, :3, 3] = 0.0
  r = np.degrees(pose_error(Ar, Br)[1])
  return {'translation_rmse_m': float(np.sqrt(np.mean(t * t))), 'translation_max_m': float(t.max()),
          'rotation_rmse_deg': float(np.sqrt(np.mean(r * r))), 'rotation_max_deg': float(r.max())}
