"""NumPy model of the render (ovn_render_batch, DESIGN.md section 4): each entry's cloud moved by its float64 pose in
the kernel's operation order, the entries concatenated in order, and the concatenation fed to oracle/projection.py's
range_projection and gen_normal_map."""
import numpy as np

from oracle import projection as oproj


def transform(points, M):
  """fl32(M (x, y, z, 1)) of (N, 4) float32 points, intensity kept: every coordinate ((M_i0 x + M_i1 y) + M_i2 z)
  + M_i3 in float64, each product and sum a separate NumPy operation (rounded once, never contracted)."""
  p = np.asarray(points, np.float32).reshape(-1, 4)
  M = np.asarray(M, np.float64).reshape(4, 4)
  x, y, z = (p[:, i].astype(np.float64) for i in range(3))
  out = np.empty_like(p)
  for i in range(3):
    out[:, i] = ((((M[i, 0] * x) + (M[i, 1] * y)) + (M[i, 2] * z)) + M[i, 3]).astype(np.float32)
  out[:, 3] = p[:, 3]
  return out


def concatenate(clouds, entry_cloud, entry_pose):
  """The cloud of one image: the entries' transformed clouds, in entry order."""
  parts = [transform(clouds[c], M) for c, M in zip(entry_cloud, entry_pose)]
  return np.concatenate(parts) if parts else np.zeros((0, 4), np.float32)


def render(clouds, entry_cloud, entry_pose, H=64, W=900, fov_up=3.0, fov_down=-25.0, max_range=50.0):
  """(range, vertex, intensity, winner, normal) of one image; winner indexes the concatenated cloud, -1 where
  empty."""
  cat = concatenate(clouds, entry_cloud, entry_pose)
  rng, vert, inten, fidx = oproj.range_projection(cat, fov_up, fov_down, H, W, max_range)
  valid, _, _, _ = oproj.projection_bins(cat, fov_up, fov_down, H, W, max_range)
  sel = np.flatnonzero(valid)
  winner = np.where(fidx >= 0, sel[np.maximum(fidx, 0)] if sel.size else -1, -1).astype(np.int32)
  return rng, vert, inten, winner, oproj.gen_normal_map(rng, vert, H, W)


def overlap(rendered_range, real_range):
  """com_overlap_yaw's rule: rendered pixels within 1 m of the real scan's valid pixels, over those pixels."""
  a, b = np.asarray(rendered_range, np.float32), np.asarray(real_range, np.float32)
  valid = b > 0
  return float(np.count_nonzero((a > 0) & valid & (np.abs(a - b) < 1)) / max(1, np.count_nonzero(valid)))
