"""Float64 NumPy model of the point-to-plane ICP of ``ovn_icp_pairs`` (TEST INFRASTRUCTURE, see oracle/__init__.py).

Restates DESIGN.md section 7 ("Registration of loop closures"): the projective association with the ground-truth
generator's float64 bin (the expression of ``oracle/gt.py:range_image_f64``, utils.py:75-104), the 29 sums of the
normal equations, the Cholesky solve, the Rodrigues update applied on the left, the distance schedule and the stopping
rules.  The reference has no ICP; nothing here claims parity with another implementation.  Every product and sum
that decides the association is evaluated in the device's order with separate roundings, so the association agrees
with the GPU's except where ``atan2`` / ``asin`` round differently at a bin edge.
"""
import numpy as np

from . import gt as G

F64 = np.float64

DEFAULTS = dict(d_start=2.0, d_end=0.3, gamma=0.8, cos_normal=float(np.cos(np.deg2rad(30.0))), eps_rot=1e-6,
                eps_trans=1e-5, iterations=30, min_inliers=100)
CONVERGED, MAX_ITERATIONS, DEGENERATE, TOO_FEW_INLIERS = 0, 1, 2, 3
PIVOT = 1e-12


def geometry(H=64, W=900, fov_up=3.0, fov_down=-25.0, max_range=50.0):
  """A handle's projection geometry; the angles and the range are float32 config values, as the handle stores them."""
  return G.geometry(H, W, fov_up, fov_down, max_range)


def bins_f64(x, y, z, g):
  """(keep, bx, by) of float64 points under range_projection (utils.py:75-104), the expression of
  oracle/gt.range_image_f64 (oracle/gt.range_angles and angle_bins)."""
  _, keep, yaw, pitch = G.range_angles(x, y, z, g)
  bx, by = G.angle_bins(yaw, pitch, g)
  return keep, bx, by


def _fill(n):
  return (n[..., 0] == -1) & (n[..., 1] == -1) & (n[..., 2] == -1)


def _apply(T, x, y, z, point):
  out = []
  for i in range(3):
    s = (T[i, 0] * x + T[i, 1] * y) + T[i, 2] * z
    out.append(s + T[i, 3] if point else s)
  return out


def valid_source(vertex, normal):
  """Pixels of a scan that take part: range > 0 (vertex w = 1) and a normal that is not the fill."""
  return (vertex[..., 3] > 0) & ~_fill(normal)


def associate(T, vs, ns, vt, nt, dk, cos_normal, g):
  """The inlier target pixel of every source pixel (or -1) under the pose T (4x4 float64), gate distance dk."""
  vs = vs.reshape(-1, 4)
  ns = ns.reshape(-1, 3)
  vt = vt.reshape(-1, 4)
  nt = nt.reshape(-1, 3)
  q = np.full(vs.shape[0], -1, np.int64)
  src = np.flatnonzero(valid_source(vs, ns))
  v = vs[src].astype(F64)
  n = ns[src].astype(F64)
  px, py, pz = _apply(T, v[:, 0], v[:, 1], v[:, 2], True)
  keep, bx, by = bins_f64(px, py, pz, g)
  j = by * g['W'] + bx
  w = vt[j].astype(F64)
  t = nt[j].astype(F64)
  ok = keep & (w[:, 3] > 0) & ~_fill(nt[j])
  mx, my, mz = _apply(T, n[:, 0], n[:, 1], n[:, 2], False)
  dx, dy, dz = px - w[:, 0], py - w[:, 1], pz - w[:, 2]
  d2 = (dx * dx + dy * dy) + dz * dz
  cn = (t[:, 0] * mx + t[:, 1] * my) + t[:, 2] * mz
  ok &= (d2 <= dk * dk) & (cn >= cos_normal)
  q[src[ok]] = j[ok]
  return q


def jacobian(T, vs, vt, nt, assoc):
  """(J [m, 6], e [m]) of the associated pixels: e = n_t . (p - q), J = [p x n_t, n_t]."""
  vs = vs.reshape(-1, 4)
  vt = vt.reshape(-1, 4)
  nt = nt.reshape(-1, 3)
  i = np.flatnonzero(assoc >= 0)
  j = assoc[i]
  v = vs[i].astype(F64)
  p = np.stack(_apply(T, v[:, 0], v[:, 1], v[:, 2], True), 1)
  q = vt[j, :3].astype(F64)
  n = nt[j].astype(F64)
  d = p - q
  e = (n[:, 0] * d[:, 0] + n[:, 1] * d[:, 1]) + n[:, 2] * d[:, 2]
  return np.concatenate([np.cross(p, n), n], 1), e


def system(T, vs, vt, nt, assoc):
  """(S, scale): the 29 sums (H's upper triangle row by row, g, inliers, sum e^2) from an association, and the sums of
  the absolute terms, the scale of each sum's rounding."""
  J, e = jacobian(T, vs, vt, nt, assoc)
  r, c = np.triu_indices(6)
  terms = np.concatenate([J[:, r] * J[:, c], J * e[:, None], np.ones((e.size, 1)), (e * e)[:, None]], 1)
  return terms.sum(0), np.abs(terms).sum(0)


def solve_update(S, T, dk, prm):
  """(status or None to go on, the updated pose) from the sums S: Cholesky of H delta = -g, R(omega) by Rodrigues,
  T <- [R(omega) | v] T, and the convergence test."""
  if S[27] < prm['min_inliers']:
    return TOO_FEW_INLIERS, T
  A = np.zeros((6, 6))
  r, c = np.triu_indices(6)
  A[r, c] = S[:21]
  A[c, r] = S[:21]
  tr = np.trace(A)
  L = np.zeros((6, 6))
  for j in range(6):
    s = A[j, j] - np.dot(L[j, :j], L[j, :j])
    if not s > PIVOT * tr:
      return DEGENERATE, T
    L[j, j] = np.sqrt(s)
    for i in range(j + 1, 6):
      L[i, j] = (A[i, j] - np.dot(L[i, :j], L[j, :j])) / L[j, j]
  y = np.zeros(6)
  for i in range(6):
    y[i] = (-S[21 + i] - np.dot(L[i, :i], y[:i])) / L[i, i]
  d = np.zeros(6)
  for i in range(5, -1, -1):
    d[i] = (y[i] - np.dot(L[i + 1:, i], d[i + 1:])) / L[i, i]
  th = np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
  R = np.eye(3)
  if th > 0:
    k = d[:3] / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = R + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)
  U = np.eye(4)
  U[:3, :3] = R
  U[:3, 3] = d[3:]
  T = U @ T
  tn = np.sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5])
  if dk == prm['d_end'] and th < prm['eps_rot'] and tn < prm['eps_trans']:
    return CONVERGED, T
  return None, T


def distances(prm):
  """d_k for k = 0 .. iterations - 1: d_start multiplied by gamma once per iteration, floored at d_end."""
  out, raw = [], F64(prm['d_start'])
  for _ in range(prm['iterations']):
    out.append(max(F64(prm['d_end']), raw))
    raw = raw * F64(prm['gamma'])
  return out


def register(vs, ns, vt, nt, init, g, params=None):
  """The whole registration of one pair: dict of pose, status, iterations, inliers, rms, valid."""
  prm = dict(DEFAULTS, **(params or {}))
  T = np.array(init, F64).reshape(4, 4)
  status, it, S = MAX_ITERATIONS, 0, np.zeros(29)
  for dk in distances(prm):
    q = associate(T, vs, ns, vt, nt, dk, prm['cos_normal'], g)
    S, _ = system(T, vs, vt, nt, q)
    it += 1
    end, T = solve_update(S, T, dk, prm)
    if end is not None:
      status = end
      break
  return dict(pose=T, status=status, iterations=it, inliers=int(S[27]),
              rms=float(np.sqrt(S[28] / S[27])) if S[27] > 0 else 0.0, valid=int(valid_source(vs, ns).sum()))
