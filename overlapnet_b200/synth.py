"""Seeded synthetic inputs shaped like the reference's data (SURVEY.md section 8d).

Used by bench.py and the tests; there is no network for KITTI, so every benchmark input is
generated here and labelled ``"data": "synthetic"``.
"""
import numpy as np

KITTI_POINTS = 124668   # point count of the reference fixture data/scans/000000.bin


def kitti_like_cloud(seed, n_points=KITTI_POINTS, zero_points=0, far_fraction=0.02):
  """HDL-64-shaped cloud: 64 beams with pitch in [-24.8, +2] deg (+ jitter), uniform azimuth,
  log-normal range clipped to (0.5, 80) m so that about ``far_fraction`` exceed max_range=50,
  intensity U[0,1) quantised to 0.01.  Returns (n_points, 4) float32 [x, y, z, intensity].
  ``zero_points`` rows are overwritten with [0,0,0,0] to exercise the depth>0 filter."""
  rng = np.random.default_rng(seed)
  beam = rng.integers(0, 64, size=n_points)
  pitch = np.deg2rad(-24.8 + (2.0 + 24.8) * (beam + 0.5) / 64.0 + rng.normal(0.0, 0.05, n_points))
  az = rng.uniform(-np.pi, np.pi, n_points)
  # median ~9 m; sigma chosen so P(r > 50) ~= far_fraction
  sigma = np.log(50.0 / 9.0) / 2.054 if far_fraction > 0 else 0.5
  r = np.clip(np.exp(rng.normal(np.log(9.0), sigma, n_points)), 0.5, 80.0)
  pts = np.empty((n_points, 4), dtype=np.float32)
  pts[:, 0] = r * np.cos(pitch) * np.cos(az)
  pts[:, 1] = r * np.cos(pitch) * np.sin(az)
  pts[:, 2] = r * np.sin(pitch)
  pts[:, 3] = np.floor(rng.uniform(0, 1, n_points) * 100.0) / 100.0
  if zero_points:
    pts[rng.choice(n_points, size=zero_points, replace=False)] = 0.0
  return pts


def random_probs(seed, n_points, n_classes=20):
  """Per-point class probabilities (softmax of N(0,1)), float32 (n_points, n_classes)."""
  rng = np.random.default_rng(seed)
  logits = rng.standard_normal((n_points, n_classes)).astype(np.float32)
  e = np.exp(logits - logits.max(axis=1, keepdims=True))
  return (e / e.sum(axis=1, keepdims=True)).astype(np.float32)


def range_like_images(seed, n, channels=4, H=64, W=900, empty_fraction=0.22):
  """Synthetic preprocessed network inputs (n, H, W, C) float32 in the reference's channel order
  (depth, normal x3, [probabilities], [intensity]); ``empty_fraction`` of the pixels hold -1."""
  rng = np.random.default_rng(seed)
  x = np.empty((n, H, W, channels), dtype=np.float32)
  x[..., 0] = rng.uniform(0.0, 50.0, (n, H, W))
  if channels >= 4:
    nrm = rng.standard_normal((n, H, W, 3))
    nrm /= np.linalg.norm(nrm, axis=-1, keepdims=True)
    x[..., 1:4] = nrm
  if channels > 4:
    x[..., 4:] = rng.uniform(0.0, 1.0, (n, H, W, channels - 4))
  empty = rng.uniform(0, 1, (n, H, W)) < empty_fraction
  x[empty] = -1.0
  return x


def feature_volumes(seed, n, width=360, channels=128, sparsity=0.5, scale=1.0):
  """Synthetic leg outputs (n, 1, width, channels) float32: non-negative (post-ReLU) with about
  ``sparsity`` exact zeros."""
  rng = np.random.default_rng(seed)
  v = rng.standard_normal((n, 1, width, channels)).astype(np.float32) * np.float32(scale)
  v = np.maximum(v + np.float32(scale * (0.0 if sparsity == 0.5 else 0.3)), 0)
  return np.ascontiguousarray(v, dtype=np.float32)


# ---- an analytic street scene, ray-cast from any pose -----------------------------------------------------------
HDL64_PITCH_DEG = (-24.8, 2.0)     # the 64 beams' elevations span this range evenly
STREET_CELL = 40.0                 # roads run along x = 40 i and y = 40 j
STREET_HALF_WIDTH = 7.0


def _street_cell_objects(seed, i, j):
  """Boxes [(x0, x1, y0, y1, z1)] and poles [(x, y, radius, height)] of the city block whose corner is (40 i, 40 j):
  two or three buildings set back from the roads, parked boxes and poles along its kerbs.  Seeded by (seed, i, j)
  only, so a block is the same from every pose."""
  rng = np.random.default_rng([int(seed) & 0xFFFFFFFF, int(i) & 0xFFFFFFFF, int(j) & 0xFFFFFFFF])
  x0, y0 = STREET_CELL * i, STREET_CELL * j
  lo, hi = STREET_HALF_WIDTH + 2.0 + rng.uniform(0, 2, 2), STREET_CELL - STREET_HALF_WIDTH - 2.0 - rng.uniform(0, 2, 2)
  boxes, poles = [], []
  cuts = np.sort(rng.uniform(lo[0] + 6, hi[0] - 6, rng.integers(1, 3)))
  edges = np.concatenate([[lo[0]], cuts, [hi[0]]])
  for a, b in zip(edges[:-1], edges[1:]):          # buildings side by side, a 1.5 m gap between neighbours
    boxes.append((x0 + a, x0 + b - 1.5, y0 + lo[1], y0 + hi[1], rng.uniform(6.0, 20.0)))
  for side in range(4):                            # kerbside boxes (parked cars, kiosks) and poles
    for _ in range(rng.integers(1, 4)):
      s = rng.uniform(4.0, STREET_CELL - 8.0)
      w, l, h = rng.uniform(1.6, 2.2), rng.uniform(3.5, 5.0), rng.uniform(1.4, 2.5)
      off = STREET_HALF_WIDTH - 2.0 - w
      if side == 0: boxes.append((x0 + s, x0 + s + l, y0 + off, y0 + off + w, h))
      elif side == 1: boxes.append((x0 + off, x0 + off + w, y0 + s, y0 + s + l, h))
      elif side == 2: boxes.append((x0 + s, x0 + s + l, y0 + STREET_CELL - off - w, y0 + STREET_CELL - off, h))
      else: boxes.append((x0 + STREET_CELL - off - w, x0 + STREET_CELL - off, y0 + s, y0 + s + l, h))
    for _ in range(rng.integers(1, 3)):
      s = rng.uniform(2.0, STREET_CELL - 2.0)
      r = STREET_HALF_WIDTH - 0.5
      xy = [(x0 + s, y0 + r), (x0 + r, y0 + s), (x0 + s, y0 + STREET_CELL - r), (x0 + STREET_CELL - r, y0 + s)][side]
      poles.append((xy[0], xy[1], rng.uniform(0.1, 0.25), rng.uniform(4.0, 8.0)))
  return boxes, poles


def street_scene_cloud(pose, seed=0, noise=0.0, n_azimuth=1800, max_hit=80.0, ground_only=False):
  """A HDL-64-like scan of a seeded street scene from the LiDAR pose ``pose`` (4x4 float64, world from sensor): a
  ground plane z = 0, blocks of buildings between roads along x = 40 i and y = 40 j (14 m wide), parked boxes and
  poles along the kerbs.  64 beams span -24.8 .. +2 degrees, ``n_azimuth`` columns per turn; a ray keeps its nearest
  hit closer than ``max_hit`` metres, plus N(0, ``noise``) metres along the ray.  Ground hits sit at z = 0 exactly
  in the world, so a level scan's ground points share one float32 z.  Returns (N, 4) float32 x, y, z, intensity
  in the sensor frame.  Sensors ride at about 1.73 m (KITTI's mounting height)."""
  T = np.asarray(pose, np.float64).reshape(4, 4)
  R, o = T[:3, :3], T[:3, 3]
  pitch = np.deg2rad(np.linspace(HDL64_PITCH_DEG[0], HDL64_PITCH_DEG[1], 64))
  az = (np.arange(n_azimuth) + 0.5) * (2 * np.pi / n_azimuth)
  pp, aa = np.meshgrid(pitch, az, indexing='ij')
  d_local = np.stack([np.cos(pp) * np.cos(aa), np.cos(pp) * np.sin(aa), np.sin(pp)], -1).reshape(-1, 3)
  d = d_local @ R.T
  t = np.full(d.shape[0], np.inf)
  with np.errstate(divide='ignore', invalid='ignore'):
    tg = np.where(d[:, 2] < 0, -o[2] / d[:, 2], np.inf)
  ground = tg < t
  t = np.where(ground, tg, t)
  if not ground_only:
    t = t.reshape(64, n_azimuth)
    ground = ground.reshape(64, n_azimuth)
    dd = d.reshape(64, n_azimuth, 3)
    level = abs(R[2, 2] - 1.0) < 1e-12
    heading = np.arctan2(R[1, 0], R[0, 0])
    step = 2 * np.pi / n_azimuth

    def columns(xy, half=0.0):
      """The columns whose rays can reach points xy (k, 2) widened by the angle `half`; every column unless level."""
      if not level:
        return slice(None)
      rel = np.arctan2(xy[:, 1] - o[1], xy[:, 0] - o[0]) - heading
      c = np.angle(np.exp(1j * rel).mean())                  # the points lie within a half turn of their mean
      dev = np.angle(np.exp(1j * (rel - c)))
      lo, hi = c + dev.min() - half - 2 * step, c + dev.max() + half + 2 * step
      k0, k1 = int(np.floor(lo / step)), int(np.ceil(hi / step))
      return np.arange(k0, k1 + 1) % n_azimuth

    reach = max_hit + STREET_CELL
    i0, i1 = int(np.floor((o[0] - reach) / STREET_CELL)), int(np.floor((o[0] + reach) / STREET_CELL))
    j0, j1 = int(np.floor((o[1] - reach) / STREET_CELL)), int(np.floor((o[1] + reach) / STREET_CELL))
    with np.errstate(invalid='ignore', divide='ignore'):
      for i in range(i0, i1 + 1):
        for j in range(j0, j1 + 1):
          boxes, poles = _street_cell_objects(seed, i, j)
          for (bx0, bx1, by0, by1, bz1) in boxes:          # slab test of an axis-aligned box on the ground
            near = np.hypot(max(bx0 - o[0], 0, o[0] - bx1), max(by0 - o[1], 0, o[1] - by1))
            if near >= max_hit:
              continue
            inside = bx0 <= o[0] <= bx1 and by0 <= o[1] <= by1
            cols = slice(None) if inside else columns(np.array([[bx0, by0], [bx0, by1], [bx1, by0], [bx1, by1]]))
            dc = dd[:, cols]
            inv = 1.0 / dc
            ta = (np.array([bx0, by0, 0.0]) - o) * inv
            tb = (np.array([bx1, by1, bz1]) - o) * inv
            tn = np.nanmax(np.minimum(ta, tb), -1)
            tf = np.nanmin(np.maximum(ta, tb), -1)
            tc = t[:, cols]
            hit = (tn <= tf) & (tn > 0) & (tn < tc)
            t[:, cols] = np.where(hit, tn, tc)
            ground[:, cols] &= ~hit
          for (cx, cy, r, h) in poles:                     # vertical cylinder, entry point only
            dist = np.hypot(cx - o[0], cy - o[1])
            if dist - r >= max_hit or dist <= r:
              continue
            cols = columns(np.array([[cx, cy]]), np.arcsin(r / dist))
            dc = dd[:, cols]
            a = dc[..., 0] ** 2 + dc[..., 1] ** 2
            b = 2 * (dc[..., 0] * (o[0] - cx) + dc[..., 1] * (o[1] - cy))
            c = (o[0] - cx) ** 2 + (o[1] - cy) ** 2 - r * r
            disc = b * b - 4 * a * c
            tq = (-b - np.sqrt(np.maximum(disc, 0))) / (2 * np.where(a > 0, a, 1))
            z = o[2] + tq * dc[..., 2]
            tc = t[:, cols]
            hit = (disc > 0) & (a > 0) & (tq > 0) & (tq < tc) & (z >= 0) & (z <= h)
            t[:, cols] = np.where(hit, tq, tc)
            ground[:, cols] &= ~hit
    t = t.reshape(-1)
    ground = ground.reshape(-1)
  keep = t < max_hit
  if noise > 0:
    t = t + np.random.default_rng(int(seed) + 1).normal(0.0, noise, t.shape)
    keep &= t > 0.1
  pw = o + t[keep, None] * d[keep]
  pw[ground[keep] & (noise <= 0), 2] = 0.0
  local = (pw - o) @ R                                     # R^T (p - o), row by row
  out = np.empty((local.shape[0], 4), np.float32)
  out[:, :3] = local
  out[:, 3] = 0.5
  return out


def _rotation(axis_angle):
  w = np.asarray(axis_angle, np.float64)
  th = np.linalg.norm(w)
  if th == 0:
    return np.eye(3)
  k = w / th
  K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
  return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def pose_graph_scene(n, n_loops, seed=0, n_false=0, step=1.0, init_noise=(0.02, 0.005), min_gap=10):
  """A seeded pose graph of a random drive: ground-truth poses [n, 4, 4] (mostly yaw turns, ``step`` metres per
  node), exact odometry T_k^-1 T_{k+1}, ``n_loops`` exact loop edges (a, b) with |a - b| >= ``min_gap``, then
  ``n_false`` false loops with random measurements (any rotation, up to 20 m).  The initial poses compose the
  odometry with increments perturbed by N(0, init_noise) (degrees, metres) per axis.  Returns (graph, gt) with the
  graph as pose_graph.chain_graph builds it (default weights) and its initial poses replaced."""
  from .pose_graph import chain_graph
  rng = np.random.default_rng(seed)
  gt = np.empty((n, 4, 4))
  gt[0] = np.eye(4)
  for k in range(1, n):
    D = np.eye(4)
    D[:3, :3] = _rotation([rng.normal(0, 0.002), rng.normal(0, 0.002), rng.normal(0, 0.05)])
    D[:3, 3] = [step, rng.normal(0, 0.02), rng.normal(0, 0.01)]
    gt[k] = gt[k - 1] @ D
  odo = np.linalg.solve(gt[:-1], gt[1:])
  pairs = []
  while len(pairs) < n_loops + n_false:
    a, b = sorted(rng.integers(0, n, 2))
    if b - a >= min_gap:
      pairs.append((a, b))
  pairs = np.array(pairs, np.int64).reshape(-1, 2)
  Z = np.linalg.solve(gt[pairs[:, 0]], gt[pairs[:, 1]]) if len(pairs) else np.zeros((0, 4, 4))
  for m in range(n_loops, n_loops + n_false):
    Z[m] = np.eye(4)
    Z[m, :3, :3] = _rotation(rng.normal(0, 1, 3) / np.sqrt(3) * rng.uniform(0, np.pi))
    Z[m, :3, 3] = rng.uniform(-20, 20, 3)
  g = chain_graph(odo, (pairs, Z))
  T = np.empty((n, 4, 4))
  T[0] = gt[0]
  r, t = np.deg2rad(init_noise[0]), init_noise[1]
  for k in range(n - 1):
    D = np.eye(4)
    D[:3, :3] = _rotation(rng.normal(0, r, 3))
    D[:3, 3] = rng.normal(0, t, 3)
    T[k + 1] = T[k] @ odo[k] @ D
  g['poses'] = T
  return g, gt
