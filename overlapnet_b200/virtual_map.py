"""A map of virtual scans: range images rendered on the GPU at the points of a planar lattice, from the keyframe
clouds around each point, and encoded by the leg into a resident bank (DESIGN.md section 7).

  lattice   the points (i g, j g), anchored in the world frame, within max_distance of some keyframe's xy; each
            takes the rotation and z of its nearest keyframe (ties to the lowest index).
  entries   for each virtual frame, its m nearest keyframes within radius (by ascending planar distance, then index),
            each moved into the frame by inv(T_v) T_k, composed in NumPy float64.
  encode    the keyframe clouds uploaded once; ovn_render_preprocess_batch and the leg in chunks of max_batch_scans
            frames, giving the device bank [V, 360, 128].  With ``surfels``, the keyframes' surfel banks are built
            in chunks of max_batch_scans keyframes and the frames rendered from them
            (ovn_render_surfels_preprocess_batch, DESIGN.md section 7, "Surfel renders").
  pixel_rays  the float64 unit directions of the pixel centres that the surfel render intersects."""
import math

import numpy as np
import torch

FEAT_C = 128


def _nearest(xy, points):
  """For each of ``points`` (n, 2): the index of the nearest of ``xy`` (K, 2), ties to the lowest index, and the
  squared distance to it, both from exact float64 differences."""
  from scipy.spatial import cKDTree
  k = min(8, xy.shape[0])
  _, idx = cKDTree(xy).query(points, k=k)
  idx = np.asarray(idx).reshape(-1, k)
  diff = xy[idx] - points[:, None, :]
  d2 = diff[..., 0] ** 2 + diff[..., 1] ** 2
  best = d2.min(1)
  cand = np.where(d2 == best[:, None], idx, np.iinfo(np.int64).max).min(1)
  return cand, best


def lattice(keyframe_poses, spacing, max_distance):
  """[V, 4, 4] poses of the lattice points (i spacing, j spacing) within ``max_distance`` of some keyframe's xy,
  ordered by j, then i.  Each takes the rotation and z of its nearest keyframe, ties to the lowest index."""
  kp = np.asarray(keyframe_poses, np.float64).reshape(-1, 4, 4)
  g, md = float(spacing), float(max_distance)
  if kp.shape[0] < 1:
    raise ValueError('a lattice needs at least one keyframe')
  if not (g > 0 and md >= 0 and np.isfinite(g) and np.isfinite(md)):
    raise ValueError('spacing must be > 0 and max_distance >= 0')
  xy = kp[:, :2, 3]
  # candidates: the lattice points of each keyframe's bounding square, then the exact distance test
  reach = int(np.ceil(md / g)) + 1
  base = np.floor(xy / g).astype(np.int64)
  off = np.arange(-reach, reach + 1)
  oi, oj = np.meshgrid(off, off, indexing='xy')
  cand = (base[:, None, :] + np.stack([oi.reshape(-1), oj.reshape(-1)], 1)[None]).reshape(-1, 2)
  cand = np.unique(cand[:, ::-1], axis=0)[:, ::-1]             # unique (i, j), sorted by j then i
  pts = cand.astype(np.float64) * g
  k, d2 = _nearest(xy, pts)
  keep = d2 <= md * md
  k, pts = k[keep], pts[keep]
  out = kp[k].copy()
  out[:, 0, 3], out[:, 1, 3] = pts[:, 0], pts[:, 1]
  return out


def entries(virtual_poses, keyframe_poses, m, radius):
  """(entry_offsets [V + 1] int64, entry_cloud [E] int32, entry_pose [E, 4, 4] float64): for each virtual frame, its
  ``m`` nearest keyframes within ``radius`` (planar distance; by ascending distance, then index), each moved into the
  frame by inv(T_v) @ T_k in float64 with the bottom row set to exactly 0 0 0 1."""
  vp = np.asarray(virtual_poses, np.float64).reshape(-1, 4, 4)
  kp = np.asarray(keyframe_poses, np.float64).reshape(-1, 4, 4)
  m, radius = int(m), float(radius)
  if m < 1 or not radius >= 0:
    raise ValueError('m must be >= 1 and radius >= 0')
  from scipy.spatial import cKDTree
  kxy, vxy = kp[:, :2, 3], vp[:, :2, 3]
  near = cKDTree(kxy).query_ball_point(vxy, radius * (1 + 1e-9) + 1e-12) if kp.shape[0] and vp.shape[0] else \
      [[] for _ in range(vp.shape[0])]
  offsets = np.zeros(vp.shape[0] + 1, np.int64)
  clouds, poses = [], []
  for v, ids in enumerate(near):
    ids = np.asarray(ids, np.int64)
    d = kxy[ids] - vxy[v]
    d2 = d[:, 0] ** 2 + d[:, 1] ** 2
    ok = d2 <= radius * radius
    ids, d2 = ids[ok], d2[ok]
    ids = ids[np.lexsort((ids, d2))][:m]
    inv = np.linalg.inv(vp[v])
    for k in ids:
      M = inv @ kp[k]
      M[3] = (0.0, 0.0, 0.0, 1.0)
      poses.append(M)
      clouds.append(k)
    offsets[v + 1] = offsets[v] + ids.size
  return (offsets, np.asarray(clouds, np.int32).reshape(-1),
          np.asarray(poses, np.float64).reshape(-1, 4, 4))


def pixel_rays(H, W, fov_up, fov_down):
  """[H, W, 3] float64: u[y][x] the unit direction whose projection's pre-floor values (utils.py:86-95) are
  (x + 1/2, y + 1/2): azimuth pi (1 - 2 (x + 1/2) / W), pitch (1 - (y + 1/2) / H) fov - |fov_down|, u = (cos p cos a,
  cos p sin a, sin p).  Built with math.sin / math.cos (libm), one value at a time, so that every caller gets the same
  table."""
  fu = float(fov_up) / 180.0 * math.pi
  fd = float(fov_down) / 180.0 * math.pi
  fov = abs(fd) + abs(fu)
  az = [math.pi * (1.0 - 2.0 * (x + 0.5) / W) for x in range(W)]
  ca, sa = [math.cos(a) for a in az], [math.sin(a) for a in az]
  out = np.empty((H, W, 3), np.float64)
  for y in range(H):
    p = (1.0 - (y + 0.5) / H) * fov - abs(fd)
    cp, sp = math.cos(p), math.sin(p)
    out[y, :, 0] = [cp * c for c in ca]
    out[y, :, 1] = [cp * s for s in sa]
    out[y, :, 2] = sp
  return out


def bank_bytes(engine, n, n_surfel_banks=0):
  """Device bytes of a resident bank of ``n`` volumes: float32 [n, 360, 128], and on a tensor-core handle the
  operand copies ovn_bank_prepare keeps per row (an fp16 [360][128] copy, six 32 KB correlation tiles, a flag); plus
  ``n_surfel_banks`` keyframe surfel banks of [H, W, 8] float32 (1.84 MB at 64 x 900)."""
  row = engine.Wf * FEAT_C * 4
  if engine.precision == 'f16_tc':
    row += engine.Wf * FEAT_C * 2 + 6 * 32768 + 4
  return int(n) * row + int(n_surfel_banks) * engine.H * engine.W * 8 * 4


def encode(infer, clouds, keyframe_poses, virtual_poses, m, radius, surfels=None):
  """The feature volumes [V, 360, 128] (device) of the virtual frames at ``virtual_poses``, rendered from their m
  nearest keyframe clouds within ``radius`` (``clouds``: (N, 4) float32 arrays or callables returning one).  With
  ``surfels`` (a dict of surfel parameters, Engine.surfel_params; {} for the defaults) the frames are rendered from
  the keyframes' surfels instead of their points.  Refused before anything is rendered when the bank, its
  tensor-core copies and the keyframes' surfel banks do not fit in the device's free memory."""
  eng = infer._engine
  vp = np.asarray(virtual_poses, np.float64).reshape(-1, 4, 4)
  kp = np.asarray(keyframe_poses, np.float64).reshape(-1, 4, 4)
  if len(clouds) != kp.shape[0]:
    raise ValueError('%d keyframe clouds for %d keyframe poses' % (len(clouds), kp.shape[0]))
  V = vp.shape[0]
  if surfels is not None:
    eng.surfel_params(surfels)                                   # unknown keys are refused before anything runs
  need = bank_bytes(eng, V, 0 if surfels is None else kp.shape[0])
  free, _ = torch.cuda.mem_get_info(eng.device)
  if need > free:
    raise MemoryError('virtual map: the bank of %d frames needs %d bytes (float32 and tensor-core copies%s), but the '
                      'device has %d bytes free' % (V, need, '' if surfels is None else ', keyframe surfels', free))
  eo, ec, ep = entries(vp, kp, m, radius)
  load = lambda c: np.ascontiguousarray(c() if callable(c) else c, np.float32)
  if surfels is None:
    batch = eng.upload_clouds([load(c) for c in clouds])
  else:
    # the surfel banks from max_batch_scans keyframe clouds at a time: no more clouds on the device at once
    src = torch.empty((kp.shape[0], eng.H, eng.W, 8), dtype=torch.float32, device=eng.device)
    for k0 in range(0, kp.shape[0], eng.max_batch_scans):
      k1 = min(kp.shape[0], k0 + eng.max_batch_scans)
      eng.surfels(eng.upload_clouds([load(c) for c in clouds[k0:k1]]), surfels, out=src[k0:k1])
  bank = torch.empty((V, eng.Wf, FEAT_C), dtype=torch.float32, device=eng.device)
  x = None
  for v0 in range(0, V, eng.max_batch_scans):
    v1 = min(V, v0 + eng.max_batch_scans)
    e0, e1 = int(eo[v0]), int(eo[v1])
    if x is None or x.shape[0] != v1 - v0:
      x = torch.empty((v1 - v0, eng.H, eng.W, eng.C), dtype=torch.float32, device=eng.device)
    if surfels is None:
      eng.render_preprocess(batch, eo[v0:v1 + 1] - e0, ec[e0:e1], ep[e0:e1], out=x)
    else:
      eng.render_surfels_preprocess(src, eo[v0:v1 + 1] - e0, ec[e0:e1], ep[e0:e1], surfels, out=x)
    eng.leg(x, out=bank[v0:v1])
  return bank
