"""NumPy float64 restatement of the Monte Carlo localization filter (csrc/mcl.cu, DESIGN.md sections 4 and 7).

Every stage takes its inputs as arguments, so the GPU tests model each stage from the GPU's own input to it.
Philox4x32-10 is reproduced bit for bit; the float64 arithmetic is the kernels' up to the last bits of the
transcendental functions and of contracted multiply-adds."""
import numpy as np

STREAM_MOTION, STREAM_INIT, STREAM_RESAMPLE = 0, 1, 2
M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = np.uint64(0xFFFFFFFF)
TWO_PI = 6.283185307179586
PI = 3.141592653589793


def philox(seed, ctr):
  """Philox4x32-10 words [n, 4] uint32 of the counters ``ctr`` [n, 4] under the 64-bit ``seed``."""
  c = np.asarray(ctr, np.uint64).reshape(-1, 4)
  c0, c1, c2, c3 = (c[:, j].copy() for j in range(4))
  k0, k1 = int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF
  for _ in range(10):
    p0 = M0 * c0
    p1 = M1 * c2
    hi0, lo0 = p0 >> np.uint64(32), p0 & MASK
    hi1, lo1 = p1 >> np.uint64(32), p1 & MASK
    c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
    k0 = (k0 + W0) & 0xFFFFFFFF
    k1 = (k1 + W1) & 0xFFFFFFFF
  return np.stack([c0, c1, c2, c3], 1).astype(np.uint32)


def counters(i, step, stream, block):
  i = np.asarray(i, np.uint64).reshape(-1)
  out = np.zeros((i.size, 4), np.uint64)
  out[:, 0] = i
  out[:, 1] = step
  out[:, 2] = stream
  out[:, 3] = block
  return out


def u53(a, b):
  """k = (a >> 5) 2^26 + (b >> 6), u = k 2^-53 with k = 0 read as 1/2: in (0, 1)."""
  k = (np.asarray(a, np.uint64) >> np.uint64(5)) * np.uint64(1 << 26) + (np.asarray(b, np.uint64) >> np.uint64(6))
  kf = k.astype(np.float64)
  return np.where(k == 0, 0.5, kf) * 2.0 ** -53


def box_muller(w):
  r = np.sqrt(-2.0 * np.log(u53(w[:, 0], w[:, 1])))
  a = TWO_PI * u53(w[:, 2], w[:, 3])
  return r * np.cos(a), r * np.sin(a)


def wrap_pi(a):
  r = np.fmod(np.asarray(a, np.float64) + PI, TWO_PI)
  r = np.where(r <= 0.0, r + TWO_PI, r)
  return r - PI


# ---- stages -------------------------------------------------------------------------------------------------
def init_global(n, seed, kf, radius):
  kf = np.asarray(kf, np.float64)
  i = np.arange(n)
  b0 = philox(seed, counters(i, 0, STREAM_INIT, 0))
  b1 = philox(seed, counters(i, 0, STREAM_INIT, 1))
  K = kf.shape[0]
  k = np.minimum((u53(b0[:, 0], b0[:, 1]) * K).astype(np.int64), K - 1)
  r = radius * np.sqrt(u53(b0[:, 2], b0[:, 3]))
  phi = TWO_PI * u53(b1[:, 0], b1[:, 1])
  th = PI - TWO_PI * u53(b1[:, 2], b1[:, 3])
  return np.stack([kf[k, 0] + r * np.cos(phi), kf[k, 1] + r * np.sin(phi), th, np.full(n, -np.log(n))])


def init_pose(n, seed, pose, sigma):
  i = np.arange(n)
  n0, n1 = box_muller(philox(seed, counters(i, 0, STREAM_INIT, 0)))
  n2, _ = box_muller(philox(seed, counters(i, 0, STREAM_INIT, 1)))
  return np.stack([pose[0] + sigma[0] * n0, pose[1] + sigma[1] * n1, wrap_pi(pose[2] + sigma[2] * n2),
                   np.full(n, -np.log(n))])


def motion(x, y, th, seed, step, odom, sigma):
  """(x', y', theta') of the particles after one predict with odometry (dx, dy, dtheta) and noise sigma."""
  i = np.arange(np.size(x))
  n0, n1 = box_muller(philox(seed, counters(i, step, STREAM_MOTION, 0)))
  n2, _ = box_muller(philox(seed, counters(i, step, STREAM_MOTION, 1)))
  c, s = np.cos(th), np.sin(th)
  ex = odom[0] + sigma[0] * n0
  ey = odom[1] + sigma[1] * n1
  return x + c * ex - s * ey, y + s * ex + c * ey, wrap_pi(th + odom[2] + sigma[2] * n2)


def lookup(x, y, raster, x0, y0, cell):
  """The keyframe under each (x, y), -1 outside the raster."""
  raster = np.asarray(raster)
  with np.errstate(invalid='ignore'):
    fy = np.floor((np.asarray(y, np.float64) - y0) / cell)
    fx = np.floor((np.asarray(x, np.float64) - x0) / cell)
    inside = (fy >= 0) & (fy < raster.shape[0]) & (fx >= 0) & (fx < raster.shape[1])
  k = np.full(np.shape(x), -1, np.int64)
  k[inside] = raster[fy[inside].astype(np.int64), fx[inside].astype(np.int64)]
  return k


def touched(k, K):
  """The keyframes with at least one particle, ascending."""
  return np.flatnonzero(np.bincount(np.asarray(k)[np.asarray(k) >= 0], minlength=K) > 0)


def expected_bin(psi, width):
  """gt.yaw_bin's expression on the relative yaw psi, mod width."""
  return (np.floor(-(np.asarray(psi) / np.pi) * width * 0.5) + width // 2).astype(np.int64) % width


def loglik(k, th, kf_theta, touched_ids, overlap, yaw, width, sigma_o, sigma_psi):
  """log l_i: -1/2 ((1 - O) / s_o)^2 - 1/2 (D / s_psi)^2 with the overlap / yaw of the particle's keyframe."""
  k = np.asarray(k)
  slot = np.full(np.size(kf_theta), -1, np.int64)
  slot[np.asarray(touched_ids, np.int64)] = np.arange(len(touched_ids))
  inside = k >= 0
  O = np.zeros(k.size)
  D = np.full(k.size, np.pi)
  j = slot[k[inside]]
  O[inside] = np.asarray(overlap, np.float32)[j].astype(np.float64)
  a = 180 - np.asarray(yaw, np.int64)[j]
  e = expected_bin(wrap_pi(np.asarray(th)[inside] - np.asarray(kf_theta)[k[inside]]), width)
  d = (a - e) % width
  d = np.minimum(d, width - d)
  D[inside] = d * (TWO_PI / width)
  return -0.5 * ((1.0 - O) / sigma_o) ** 2 - 0.5 * (D / sigma_psi) ** 2


def normalize(lw):
  """(normalised log-weights, weights)."""
  m = np.max(lw)
  lw = lw - (m + np.log(np.sum(np.exp(lw - m))))
  return lw, np.exp(lw)


def estimate(w, x, y, th):
  sw = np.sum(w)
  return {'x': np.sum(w * x) / sw, 'y': np.sum(w * y) / sw, 'theta': np.arctan2(np.sum(w * np.sin(th)),
                                                                                  np.sum(w * np.cos(th))),
          'ess': 1.0 / np.sum(w * w)}


def resample_u0(seed, step):
  w = philox(seed, counters([0], step, STREAM_RESAMPLE, 0))
  return float(u53(w[:, 0], w[:, 1])[0])


def systematic(cdf, u0):
  """Ancestors a_j = min{i : C_i > (j + u0) / N}, clamped to N - 1."""
  n = np.size(cdf)
  t = (np.arange(n, dtype=np.float64) + u0) / n
  return np.minimum(np.searchsorted(np.asarray(cdf), t, side='right'), n - 1)


# ---- the whole filter ---------------------------------------------------------------------------------------
class Filter:
  """The filter of csrc/mcl.cu on the host: ``observe(ids)`` gives (overlap, yaw) of the touched keyframes."""

  def __init__(self, kf, raster, x0, y0, cell, width=360):
    self.kf, self.raster, self.x0, self.y0, self.cell, self.width = np.asarray(kf, np.float64), raster, x0, y0, cell, width

  def init_global(self, n, seed, radius):
    self.p, self.seed, self.step_no = init_global(n, seed, self.kf, radius), seed, 0

  def step(self, odom, sigma, observe, sigma_o, sigma_psi, rho=0.5):
    self.step_no += 1
    x, y, th = motion(self.p[0], self.p[1], self.p[2], self.seed, self.step_no, odom, sigma)
    k = lookup(x, y, self.raster, self.x0, self.y0, self.cell)
    ids = touched(k, self.kf.shape[0])
    ov, yaw = observe(ids) if ids.size else (np.zeros(0, np.float32), np.zeros(0, np.int32))
    ll = loglik(k, th, self.kf[:, 2], ids, ov, yaw, self.width, sigma_o, sigma_psi)
    lw, w = normalize(self.p[3] + ll)
    est = estimate(w, x, y, th)
    est['n_touched'] = int(ids.size)
    est['resampled'] = bool(est['ess'] < rho * w.size)
    self.p = np.stack([x, y, th, lw])
    if est['resampled']:
      a = systematic(np.cumsum(w), resample_u0(self.seed, self.step_no))
      self.p = np.stack([x[a], y[a], th[a], np.full(w.size, -np.log(w.size))])
    return est


# ---- a synthetic localization scenario with a sensor that knows the true pose --------------------------------
def scenario(spacing=1.0):
  """A 3.3 km drive: twice round a 700 m x 300 m loop with rounded corners, the second lap 3 m to the left of the
  first (a revisit in another lane), then 500 m back along the start in the opposite direction.  Frames every
  ``spacing`` metres; returns (n, 3) planar poses x, y, theta."""
  pts = []

  def lap(offset):
    a, b, r = 700.0, 300.0, 40.0
    segs = []
    # straight edges and quarter circles, counter-clockwise, driven at the inner offset
    corners = [(a - r, r, -np.pi / 2), (a - r, b - r, 0.0), (r, b - r, np.pi / 2), (r, r, np.pi)]
    for (cx, cy, a0) in corners:
      segs.append(('arc', cx, cy, a0, r - offset))
    s = []
    for cx, cy, a0, rr in [(c[1], c[2], c[3], c[4]) for c in segs]:
      for t in np.arange(0.0, np.pi / 2, spacing / rr):
        s.append((cx + rr * np.cos(a0 + t), cy + rr * np.sin(a0 + t), wrap_pi(a0 + t + np.pi / 2)))
      # the straight edge after the corner
      end = a0 + np.pi / 2
      ex, ey = cx + rr * np.cos(end), cy + rr * np.sin(end)
      th = wrap_pi(end + np.pi / 2)
      length = (a if abs(np.cos(th)) > 0.5 else b) - 2 * r
      for d in np.arange(0.0, length, spacing):
        s.append((ex + d * np.cos(th), ey + d * np.sin(th), th))
    return s
  pts += lap(0.0)
  pts += lap(3.0)
  # back along the bottom edge, westwards, 6 m to the right of the first lap
  for d in np.arange(0.0, 500.0, spacing):
    pts.append((600.0 - d, -6.0, np.pi))
  return np.asarray(pts, np.float64)


def fake_sensor(truth, keyframes, width=360, reach=15.0):
  """observe(ids) of a query at the true pose ``truth`` (x, y, theta): overlap max(0, 1 - d / reach) with d the
  distance to the keyframe, and the heads' yaw 180 - (the yaw bin of the true relative pose)."""
  kf = np.asarray(keyframes, np.float64)

  def observe(ids):
    ids = np.asarray(ids, np.int64)
    d = np.hypot(kf[ids, 0] - truth[0], kf[ids, 1] - truth[1])
    ov = np.maximum(0.0, 1.0 - d / reach).astype(np.float32)
    yaw = (180 - expected_bin(wrap_pi(truth[2] - kf[ids, 2]), width)).astype(np.int32)
    return ov, yaw
  return observe
