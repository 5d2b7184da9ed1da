"""Float64 NumPy / SciPy model of the robust pose-graph optimizer (ovn_pgo_optimize_host, DESIGN.md section 7,
"Pose-graph optimization"): the residual, its exact Jacobians, the cost, the gradient, the sparse Gauss-Newton matrix,
and Levenberg-Marquardt with an exact sparse solve and the library's stopping rules.  Test infrastructure only.

A graph is a dict of poses [n, 4, 4], edges [E, 2] (chain (k, k + 1) first), measurements [E, 4, 4] and weights
[E, 6], as overlapnet_b200.pose_graph.chain_graph builds it.  The geometry (hat to jacobian, rho) keeps np.longdouble
inputs in long double, so that oracle/pgo_stages.py can take it as an exact reference for the kernel's float64."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

PI_BRANCH = 1e-2        # Log(R) above pi - PI_BRANCH takes its axis from the symmetric part of R (kPgoPiBranch)
SERIES_BELOW = 1e-2     # J_l^-1's K^2 coefficient takes its series below this angle (kPgoSeriesBelow)
DEFAULTS = dict(phi=25.0, lambda0=1e-6, lambda_min=1e-12, lambda_max=1e12, rel_cost_tol=1e-10, step_tol=1e-10,
                cg_tol=1e-12, max_iterations=50, max_cg_iterations=2000)
STATUS = ('converged', 'max_iterations', 'stalled', 'failed')


def _f(x):
  """x as float64, or as long double when it is long double"""
  x = np.asarray(x)
  return x if x.dtype == np.longdouble else x.astype(np.float64)


def inv_rigid(T):
  """[R | t]^-1 = [R^T | -R^T t], as the kernel inverts a pose or a measurement"""
  T = _f(T)
  out = np.zeros_like(T)
  Rt = np.swapaxes(T[..., :3, :3], -1, -2)
  out[..., :3, :3] = Rt
  out[..., :3, 3] = -np.einsum('...ij,...j->...i', Rt, T[..., :3, 3])
  out[..., 3, 3] = 1.0
  return out


def hat(v):
  v = _f(v)
  K = np.zeros(v.shape[:-1] + (3, 3), v.dtype)
  K[..., 0, 1], K[..., 0, 2], K[..., 1, 2] = -v[..., 2], v[..., 1], -v[..., 0]
  K[..., 1, 0], K[..., 2, 0], K[..., 2, 1] = v[..., 2], -v[..., 1], v[..., 0]
  return K


def rodrigues(w):
  """R(omega) [..., 3, 3] = I + sin(th) K + (1 - cos(th)) K^2, K the cross-product matrix of the unit axis."""
  w = _f(w)
  th = np.sqrt(np.sum(w * w, -1))
  safe = np.where(th > 0, th, 1.0)
  K = hat(w / safe[..., None])
  s, c1 = np.sin(th)[..., None, None], (1 - np.cos(th))[..., None, None]
  R = np.eye(3) + s * K + c1 * (K @ K)
  return np.where((th > 0)[..., None, None], R, np.eye(3))


def update(T, xi):
  """T <- [R(omega) | v] T of xi = (omega, v) [..., 6]."""
  xi = _f(xi)
  U = np.zeros(xi.shape[:-1] + (4, 4), xi.dtype)
  U[..., :3, :3] = rodrigues(xi[..., :3])
  U[..., :3, 3] = xi[..., 3:]
  U[..., 3, 3] = 1.0
  return U @ _f(T)


def log_so3(R):
  """phi [..., 3] of R [..., 3, 3]: the angle atan2(|axis| / 2, (tr R - 1) / 2) (registration.pose_error's), the axis
  from the antisymmetric part, or from the symmetric part above pi - PI_BRANCH."""
  R = _f(R)
  ax = np.stack([R[..., 2, 1] - R[..., 1, 2], R[..., 0, 2] - R[..., 2, 0], R[..., 1, 0] - R[..., 0, 1]], -1)
  sn = np.sqrt(np.sum(ax * ax, -1))
  cs = 0.5 * (np.trace(R, axis1=-2, axis2=-1) - 1.0)
  th = np.arctan2(0.5 * sn, cs)
  phi = np.where((sn > 0)[..., None], (th / np.where(sn > 0, sn, 1.0))[..., None] * ax, 0.0)
  near = th > np.pi - PI_BRANCH
  if np.any(near):
    Rn, csn, thn, axn = R[near], cs[near], th[near], ax[near]
    d = np.diagonal(Rn, axis1=-2, axis2=-1)
    i = np.argmax(d, -1)
    out = np.empty((Rn.shape[0], 3), R.dtype)
    for m in range(Rn.shape[0]):
      oc = 1.0 - csn[m]
      k = np.empty(3, R.dtype)
      k[i[m]] = np.sqrt(max((Rn[m, i[m], i[m]] - csn[m]) / oc, 0.0))
      for j in range(3):
        if j != i[m]:
          k[j] = (Rn[m, i[m], j] + Rn[m, j, i[m]]) / (2 * oc * k[i[m]])
      out[m] = (-1.0 if k @ axn[m] < 0 else 1.0) * thn[m] * k
    phi[near] = out
  return phi


def jl_inv(phi):
  """J_l^-1(phi) = I - K / 2 + c K^2, c = 1 / th^2 - (1 + cos th) / (2 th sin th) (a series below SERIES_BELOW)."""
  phi = _f(phi)
  t2 = np.sum(phi * phi, -1)
  th = np.sqrt(t2)
  with np.errstate(divide='ignore', invalid='ignore'):
    direct = 1.0 / t2 - (1.0 + np.cos(th)) / (2.0 * th * np.sin(th))
  c = np.where(th < SERIES_BELOW, 1 / 12 + t2 / 720 + t2 * t2 / 30240, direct)
  K = hat(phi)
  return np.eye(3) - 0.5 * K + c[..., None, None] * (K @ K)


def exp_so3(phi):
  return rodrigues(phi)


def residual(Ta, Tb, Z):
  """e [..., 6] = (Log(R_E), t_E) of E = Z^-1 T_a^-1 T_b, and C = Z^-1 T_a^-1 [..., 4, 4]."""
  C = inv_rigid(Z) @ inv_rigid(Ta)
  E = C @ Tb
  return np.concatenate([log_so3(E[..., :3, :3]), E[..., :3, 3]], -1), C


def jacobian(Ta, Tb, Z):
  """(e, A) with A = J_E Ad_C [..., 6, 6]: de/dxi_b = A and de/dxi_a = -A."""
  e, C = residual(Ta, Tb, Z)
  RC, tC = C[..., :3, :3], C[..., :3, 3]
  A = np.zeros(e.shape[:-1] + (6, 6), e.dtype)
  A[..., :3, :3] = jl_inv(e[..., :3]) @ RC
  A[..., 3:, :3] = hat(tC - e[..., 3:]) @ RC
  A[..., 3:, 3:] = RC
  return e, A


def rho(x, loop, phi):
  """(rho(chi2), s): least squares on the chain (and for phi = inf), Geman-McClure on loops."""
  x = _f(x)
  if np.isinf(phi):
    return x.copy(), np.ones_like(x)
  s = np.where(loop, phi / (phi + x), 1.0)
  return np.where(loop, s * x, x), s


def evaluate(graph, poses, phi):
  """F, chi2 [E], s [E] at ``poses``."""
  ed = np.asarray(graph['edges'], np.int64)
  n = poses.shape[0]
  e, _ = residual(poses[ed[:, 0]], poses[ed[:, 1]], graph['measurements'])
  chi2 = np.sum(graph['weights'] * e * e, -1)
  r, s = rho(chi2, np.arange(ed.shape[0]) >= n - 1, phi)
  return 0.5 * r.sum(), chi2, s


def linearize(graph, poses, phi):
  """F, chi2, s, the gradient g [n, 6] and the sparse H [6n, 6n] (every node) at ``poses``."""
  ed = np.asarray(graph['edges'], np.int64)
  n = poses.shape[0]
  E = ed.shape[0]
  e, A = jacobian(poses[ed[:, 0]], poses[ed[:, 1]], graph['measurements'])
  w = np.asarray(graph['weights'], np.float64)
  chi2 = np.sum(w * e * e, -1)
  r, s = rho(chi2, np.arange(E) >= n - 1, phi)
  d = s * s
  M = d[:, None, None] * np.einsum('kri,kr,krj->kij', A, w, A)
  q = d[:, None] * np.einsum('kri,kr,kr->ki', A, w, e)
  g = np.zeros((n, 6))
  np.add.at(g, ed[:, 1], q)
  np.add.at(g, ed[:, 0], -q)
  rows, cols, vals = [], [], []
  ii, jj = np.meshgrid(np.arange(6), np.arange(6), indexing='ij')
  for (u, v, sign) in ((0, 0, 1), (1, 1, 1), (0, 1, -1), (1, 0, -1)):
    rows.append((6 * ed[:, u])[:, None, None] + ii)
    cols.append((6 * ed[:, v])[:, None, None] + jj)
    vals.append(sign * M)
  H = sp.coo_matrix((np.concatenate([v.ravel() for v in vals]),
                     (np.concatenate([v.ravel() for v in rows]), np.concatenate([v.ravel() for v in cols]))),
                    shape=(6 * n, 6 * n)).tocsc()
  return 0.5 * r.sum(), chi2, s, g, H


def optimize(graph, params=None, lm_solve=None):
  """Levenberg-Marquardt with the library's rules (DESIGN section 7), each trial solved exactly by spsolve (or by
  ``lm_solve(A, b)``).  Returns a dict: poses, status (name), iterations, accepted, initial_cost, final_cost, lambda,
  max_gradient, chi2, scale, gradient [n, 6] and trace (a list of (F, lambda, accepted) per trial)."""
  p = dict(DEFAULTS, **(params or {}))
  T = np.asarray(graph['poses'], np.float64).copy()
  n = T.shape[0]
  F, chi2, s, g, H = linearize(graph, T, p['phi'])
  F0, lam, status, it, acc, trace = F, p['lambda0'], 'max_iterations', 0, 0, []
  while it < p['max_iterations']:
    Hr = H[6:, 6:]
    A = (Hr + lam * sp.diags(Hr.diagonal())).tocsc()
    b = -g[1:].ravel()
    delta = (lm_solve or spla.spsolve)(A, b) if np.any(b != 0) else np.zeros_like(b)
    it += 1
    dmax = float(np.max(np.abs(delta))) if delta.size else 0.0
    Tt = T.copy()
    Tt[1:] = update(T[1:], delta.reshape(-1, 6))
    Ft = evaluate(graph, Tt, p['phi'])[0]
    ok = Ft < F
    trace.append((Ft, lam, ok))
    if ok:
      T, Fold, acc = Tt, F, acc + 1
      lam = max(lam / 10, p['lambda_min'])
      F, chi2, s, g, H = linearize(graph, T, p['phi'])
      if Fold - F <= p['rel_cost_tol'] * Fold or dmax <= p['step_tol']:
        status = 'converged'
        break
    else:
      lam *= 10
      if dmax <= p['step_tol']:
        status = 'converged'
        break
      if lam > p['lambda_max']:
        status = 'stalled'
        break
  return {'poses': T, 'status': status, 'iterations': it, 'accepted': acc, 'initial_cost': F0, 'final_cost': F,
          'lambda': lam, 'max_gradient': float(np.abs(g[1:]).max()), 'chi2': chi2, 'scale': s, 'gradient': g,
          'trace': trace}


def replay(graph, trace_lambda, trace_accepted, params=None):
  """Trial costs of the oracle's LM when it takes the given accept / reject sequence and lambdas (the GPU's), from
  the same input: each trial is solved exactly at the oracle's own linearization."""
  p = dict(DEFAULTS, **(params or {}))
  T = np.asarray(graph['poses'], np.float64).copy()
  F, _, _, g, H = linearize(graph, T, p['phi'])
  out = []
  for lam, ok in zip(trace_lambda, trace_accepted):
    Hr = H[6:, 6:]
    delta = spla.spsolve((Hr + lam * sp.diags(Hr.diagonal())).tocsc(), -g[1:].ravel())
    Tt = T.copy()
    Tt[1:] = update(T[1:], delta.reshape(-1, 6))
    Ft = evaluate(graph, Tt, p['phi'])[0]
    out.append(Ft)
    if ok:
      T = Tt
      F, _, _, g, H = linearize(graph, T, p['phi'])
  return np.array(out), T
