"""NumPy model of the surfel render (ovn_surfels_batch / ovn_render_surfels_batch, DESIGN.md section 7, "Surfel
renders"), in the kernels' operation order: every float64 product, sum, quotient and square root a separate NumPy
operation, rounded once and never contracted.  The keyframes' projections and the rendered images' normals come
from oracle/projection.py."""
import math

import numpy as np

from oracle import projection as oproj

F32, F64 = np.float32, np.float64
DEFAULTS = dict(kappa=1.0, c_min=0.5, max_splat=8)


def delta(H, W, fov_up, fov_down):
  """max(2 pi / W, fov / H) from the handle's float32 degrees, as the library computes it."""
  fu = float(F32(fov_up)) / 180.0 * math.pi
  fd = float(F32(fov_down)) / 180.0 * math.pi
  return max(2.0 * math.pi / W, (abs(fd) + abs(fu)) / H)


def build(rng, vert, inten, normal, kappa=1.0, c_min=0.5, fov_up=3.0, fov_down=-25.0):
  """The [H, W, 8] surfel bank of one projection (range, vertex, intensity, normal images): (c, r, n, intensity) per
  valid pixel, zeros elsewhere."""
  H, W = rng.shape
  out = np.zeros((H, W, 8), F32)
  ok = rng > 0
  c = vert[ok][:, :3].astype(F32)
  n = normal[ok].astype(F32).copy()
  cx, cy, cz = (c[:, i].astype(F64) for i in range(3))
  fill = (n[:, 0] == -1) & (n[:, 1] == -1) & (n[:, 2] == -1)
  nc = np.sqrt((cx * cx + cy * cy) + cz * cz)
  for i, ci in enumerate((cx, cy, cz)):
    n[:, i] = np.where(fill, (-ci / nc).astype(F32), n[:, i])
  dot = (n[:, 0].astype(F64) * cx + n[:, 1].astype(F64) * cy) + n[:, 2].astype(F64) * cz
  d = rng[ok].astype(F64)
  den = np.maximum(np.abs(dot) / d, F64(c_min))
  r = (((F64(kappa) * d) * delta(H, W, fov_up, fov_down)) / den).astype(F32)
  out[ok] = np.concatenate([c, r[:, None], n, inten[ok][:, None].astype(F32)], 1)
  return out


def surfels(cloud, H=64, W=900, fov_up=3.0, fov_down=-25.0, max_range=50.0, kappa=1.0, c_min=0.5):
  """The surfel bank of one raw cloud: its projection at the handle's geometry and max_range, then build."""
  rng, vert, inten, _ = oproj.range_projection(cloud, fov_up, fov_down, H, W, max_range)
  return build(rng, vert, inten, oproj.gen_normal_map(rng, vert, H, W), kappa, c_min, fov_up, fov_down)


def pose(bank, M):
  """(q, m, r, intensity, slot) of the bank's surfels (r > 0) moved by the float64 pose M: q = M (c, 1) in
  mat4_apply's order, m = R n."""
  flat = bank.reshape(-1, 8)
  slot = np.flatnonzero(flat[:, 3] > 0)
  s = flat[slot]
  M = np.asarray(M, F64)
  c = [s[:, i].astype(F64) for i in range(3)]
  n = [s[:, 4 + i].astype(F64) for i in range(3)]
  q = np.stack([(((M[i, 0] * c[0]) + (M[i, 1] * c[1])) + (M[i, 2] * c[2])) + M[i, 3] for i in range(3)], 1)
  m = np.stack([((M[i, 0] * n[0]) + (M[i, 1] * n[1])) + (M[i, 2] * n[2]) for i in range(3)], 1)
  return q, m, s[:, 3].astype(F64), s[:, 7], slot


def window(q, nq, r, S, H, W, fov_up, fov_down):
  """The kernel's half-widths (hy, hx) of the box that holds every pixel a surfel can draw (surfel_window), in host
  libm: S where r >= |q| or where the azimuth bound reaches a pole."""
  fu, fd = fov_up / 180.0 * math.pi, fov_down / 180.0 * math.pi
  rows_per_rad, cols_per_rad = H / (abs(fd) + abs(fu)), W / (2.0 * math.pi)
  hy = np.full(q.shape[0], S, np.int64)
  hx = hy.copy()
  with np.errstate(all='ignore'):
    small = r < nq
    a = np.arcsin(r / nq)
    hy = np.where(small, np.fmin(S, np.ceil(a * rows_per_rad) + 1.0), S).astype(np.int64)
    p = np.abs(np.arcsin(q[:, 2] / nq)) + a
    s = np.sin(0.5 * a) / np.cos(p)
    ok = small & (p < 1.5707963267948966) & (s < 1.0)
    hx = np.where(ok, np.fmin(S, np.ceil(2.0 * np.arcsin(s) * cols_per_rad) + 1.0), S).astype(np.int64)
  return hy, hx


def _hit(q, m, r, u, max_range):
  """(drawn, t) of surfels (q, m, r) at rays u, the draw rule in the kernel's order."""
  den = (m[:, 0] * u[:, 0] + m[:, 1] * u[:, 1]) + m[:, 2] * u[:, 2]
  num = (m[:, 0] * q[:, 0] + m[:, 1] * q[:, 1]) + m[:, 2] * q[:, 2]
  with np.errstate(all='ignore'):
    t = num / den
    d = t[:, None] * u - q
    dist2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    drawn = (np.abs(den) > 1e-6) & (t > 0) & (t.astype(F32) < F32(max_range)) & (dist2 <= r * r)
  return drawn, t


def render(banks, entry_cloud, entry_pose, rays, H=64, W=900, fov_up=3.0, fov_down=-25.0, max_range=50.0,
           max_splat=8, full_window=False):
  """(range, vertex, intensity, winner, normal) of one image z-buffered from the entries' surfel banks.  winner is
  (entry ordinal) H W + slot, -1 where empty.  The boxes are the kernel's windows (surfel_window); with
  ``full_window`` every surfel is tested on its whole (2 S + 1)^2 box instead, which must give the same image."""
  HW = H * W
  S = int(max_splat)
  keys = np.full(HW, np.iinfo(np.uint64).max, np.uint64)
  per = []
  for k, (c, M) in enumerate(zip(entry_cloud, entry_pose)):
    q, m, r, inten, slot = pose(banks[c], M)
    nq = np.sqrt((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2])
    keep = (nq > 0) & ((nq - r) < F64(F32(max_range)))
    q32 = q.astype(F32)
    keep &= oproj.point_depth(np.concatenate([q32, np.zeros((q32.shape[0], 1), F32)], 1)) > 0
    q, m, r, inten, slot, nq, q32 = q[keep], m[keep], r[keep], inten[keep], slot[keep], nq[keep], q32[keep]
    pts = np.concatenate([q32, np.zeros((q32.shape[0], 1), F32)], 1)
    _, _, by, bx = oproj.projection_bins(pts, fov_up, fov_down, H, W, np.inf)
    if full_window:
      hy = hx = np.full(q.shape[0], S, np.int64)
    else:
      hy, hx = window(q, nq, r, S, H, W, fov_up, fov_down)
    per.append((q, m, r, inten, slot))
    key_lo = (k * HW + slot).astype(np.uint64)
    ny, nx = 2 * hy + 1, 2 * hx + 1
    area = ny * nx
    # every (surfel, box pixel) pair, in chunks of about 2^22 pairs
    ends = np.cumsum(area)
    s0 = 0
    while s0 < q.shape[0]:
      s1 = max(s0 + 1, int(np.searchsorted(ends, (ends[s0 - 1] if s0 else 0) + (1 << 22), 'right')))
      a = area[s0:s1]
      sel = np.repeat(np.arange(s0, s1), a)
      local = np.arange(sel.size) - np.repeat(np.cumsum(a) - a, a)
      y = by[sel].astype(np.int64) + local // nx[sel] - hy[sel]
      x = bx[sel].astype(np.int64) + local % nx[sel] - hx[sel]
      inside = (y >= 0) & (y < H)
      sel, y, x = sel[inside], y[inside], np.mod(x[inside], W)
      drawn, t = _hit(q[sel], m[sel], r[sel], rays[y, x], max_range)
      key = (t[drawn].astype(F32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | key_lo[sel[drawn]]
      np.minimum.at(keys, (y * W + x)[drawn], key)
      s0 = s1
  rng = np.full(HW, -1, F32)
  vert = np.full((HW, 4), -1, F32)
  inten_img = np.full(HW, -1, F32)
  winner = np.full(HW, -1, np.int32)
  depth = (keys >> np.uint64(32)).astype(np.uint32).view(F32)
  has = (keys != np.iinfo(np.uint64).max) & (depth > 0)
  pix = np.flatnonzero(has)
  lo = (keys[pix] & np.uint64(0xFFFFFFFF)).astype(np.int64)
  for k in np.unique(lo // HW):
    q, m, r, inten, slot = per[k]
    at = np.flatnonzero(lo // HW == k)
    j = np.searchsorted(slot, lo[at] % HW)
    p = pix[at]
    u = rays.reshape(-1, 3)[p]
    qq, mm = q[j], m[j]
    den = (mm[:, 0] * u[:, 0] + mm[:, 1] * u[:, 1]) + mm[:, 2] * u[:, 2]
    num = (mm[:, 0] * qq[:, 0] + mm[:, 1] * qq[:, 1]) + mm[:, 2] * qq[:, 2]
    t = num / den
    rng[p] = t.astype(F32)
    vert[p, :3] = (t[:, None] * u).astype(F32)
    vert[p, 3] = 1.0
    inten_img[p] = inten[j]
    winner[p] = lo[at].astype(np.int32)
  assert np.array_equal(rng[pix].view(np.uint32), depth[pix].view(np.uint32))
  rng, vert = rng.reshape(H, W), vert.reshape(H, W, 4)
  return rng, vert, inten_img.reshape(H, W), winner.reshape(H, W), oproj.gen_normal_map(rng, vert, H, W)
