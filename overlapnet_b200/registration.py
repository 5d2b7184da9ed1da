"""Geometric registration of loop-closure pairs on the GPU: point-to-plane ICP on the range images (ovn_icp_pairs),
seeded by the yaw head, as the OverlapNet paper initialises ICP with the predicted yaw when it closes loops.

The model (DESIGN.md section 7):
  direction  a pair (LEFT = a, RIGHT = b) estimates T = T_a^-1 T_b, which takes RIGHT's vertices into LEFT's frame:
             RIGHT is the source and LEFT's images are the target.  The heads' record of (a, b) predicts its yaw.
  seed       the heads' argmax a = 180 - yaw (evaluate.yaw_to_argmax) is a bin of gt.yaw_bin; its centre
             psi(a) = -(a - Wf // 2 + 1/2) 2 pi / Wf seeds T_0 = [Rz(psi) | 0].  The identity is the comparison.
  ICP        projective association, point-to-plane residuals, Cholesky solve and left update in float64, with
             the distance schedule and stopping rules of ovn_icp_pairs; the defaults are not tuned on KITTI."""
import numpy as np
import torch

PROJECT_CHUNK = 64          # scans projected per Engine.project call


def seed_yaw(argmax, Wf):
  """psi: the yaw at the centre of bin ``argmax`` of gt.yaw_bin at ``Wf`` bins, radians."""
  return -(np.asarray(argmax, np.float64) - Wf // 2 + 0.5) * (2 * np.pi / Wf)


def seed_pose(argmax, Wf):
  """T_0 = [Rz(seed_yaw(argmax, Wf)) | 0], (..., 4, 4) float64."""
  psi = seed_yaw(argmax, Wf)
  T = np.zeros(psi.shape + (4, 4))
  c, s = np.cos(psi), np.sin(psi)
  T[..., 0, 0], T[..., 0, 1], T[..., 1, 0], T[..., 1, 1] = c, -s, s, c
  T[..., 2, 2] = T[..., 3, 3] = 1.0
  return T


def pose_error(T_est, T_gt):
  """(translation norm in metres, rotation angle in radians) of T_gt^-1 T_est, over any leading dimensions."""
  E = np.linalg.solve(np.asarray(T_gt, np.float64), np.asarray(T_est, np.float64))
  R = E[..., :3, :3]
  axis = np.stack([R[..., 2, 1] - R[..., 1, 2], R[..., 0, 2] - R[..., 2, 0], R[..., 1, 0] - R[..., 0, 1]], -1)
  angle = np.arctan2(0.5 * np.linalg.norm(axis, axis=-1), 0.5 * (np.trace(R, axis1=-2, axis2=-1) - 1.0))
  return np.linalg.norm(E[..., :3, 3], axis=-1), angle


def images(engine, clouds, scans):
  """Vertex [n, H, W, 4] and normal [n, H, W, 3] maps of ``clouds[s]`` for s in ``scans``, projected on the device
  PROJECT_CHUNK scans at a time (Engine.project, Engine.normals)."""
  n = len(scans)
  vertex = torch.empty((n, engine.H, engine.W, 4), dtype=torch.float32, device=engine.device)
  normal = torch.empty((n, engine.H, engine.W, 3), dtype=torch.float32, device=engine.device)
  for s0 in range(0, n, PROJECT_CHUNK):
    s1 = min(n, s0 + PROJECT_CHUNK)
    batch = engine.upload_clouds([np.ascontiguousarray(clouds[s]() if callable(clouds[s]) else clouds[s], np.float32)
                                  for s in scans[s0:s1]])
    out = engine.project(batch, want=('range', 'vertex'))
    vertex[s0:s1] = out['vertex']
    normal[s0:s1] = engine.normals(out['range'], out['vertex'])
  return vertex, normal


def register(engine, clouds, left, right, init, params=None, pairs_per_call=1024):
  """Register the pairs (LEFT = clouds[left[i]], RIGHT = clouds[right[i]]) from ``init`` [np, 4, 4]: estimates
  T_LEFT^-1 T_RIGHT.  ``clouds``: (N, 4) float32 arrays or zero-argument callables returning one; only the scans the
  pairs touch are projected, ``pairs_per_call`` pairs at a time.  ``params``: overrides of ovn_icp_default_params.
  Returns host arrays: pose [np, 4, 4] f64, rms f64, inliers / valid / iterations / status i32.  A pair's result
  has the same bits whatever the chunking."""
  left = np.asarray(left, np.int64).reshape(-1)
  right = np.asarray(right, np.int64).reshape(-1)
  init = np.asarray(init, np.float64).reshape(-1, 4, 4)
  n = left.size
  if right.size != n or init.shape[0] != n:
    raise ValueError('left, right and init must have one entry per pair')
  if pairs_per_call < 1:
    raise ValueError('pairs_per_call must be >= 1')
  out = {'pose': np.zeros((n, 4, 4)), 'rms': np.zeros(n), 'inliers': np.zeros(n, np.int32),
         'valid': np.zeros(n, np.int32), 'iterations': np.zeros(n, np.int32), 'status': np.zeros(n, np.int32)}
  for p0 in range(0, n, pairs_per_call):
    p1 = min(n, p0 + pairs_per_call)
    scans, local = np.unique(np.concatenate([right[p0:p1], left[p0:p1]]), return_inverse=True)
    if scans.size and (scans[0] < 0 or scans[-1] >= len(clouds)):
      raise IndexError('a pair refers to a scan outside [0, %d)' % len(clouds))
    vertex, normal = images(engine, clouds, scans)
    res = engine.icp(vertex, normal, local[:p1 - p0], local[p1 - p0:], init[p0:p1], params)
    engine.check()
    for key in out:
      out[key][p0:p1] = res[key].cpu().numpy()
    del vertex, normal
  return out
