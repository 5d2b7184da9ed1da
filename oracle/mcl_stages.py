"""Float64 stage model of Monte Carlo localization (csrc/mcl.cu) and the gate each stage, read back by
Engine.mcl_stage / Engine.mcl_particles, must pass.  Test infrastructure only; it builds on oracle/mcl.py.  Every
check takes the stage's inputs as arguments, so each GPU stage is checked from the GPU's own input to it.  The
``restate_*`` functions are a NumPy restatement of each kernel in its own order; the CPU tests run them in place of
the GPU, with and without planted defects (``mutant``).

Rounding rules.  u = 2^-53, and an ulp of a normal double v is at most 2 u |v|.  Each IEEE + - * / and sqrt rounds
once (|err| <= u |result|, or 2^-1074 absolute where the result is subnormal); fmod, floor, negation, scaling by 1/2
and the integer-to-double conversions are exact.  A product that the compiler contracts with an add into a DFMA
rounds once instead of twice; every bound below counts the product's rounding as well, so it covers both forms.
The sm_90a build does contract: the log-likelihood's final subtraction is DFMA(q1, -0.5, -0.5 q2), whose product
by -1/2 is exact, so there both forms give the same bits.  The device's double functions are within the maximum
ulp errors of the CUDA C++ Programming Guide (CUDA 12.9, "Mathematical Functions", double-precision table):
exp 1, log 1, sin 2, cos 2, atan2 2 ulp; sqrt is correctly rounded.  So exp and log carry 2 u relative, sin, cos
and atan2 4 u.  The host side of every bound is evaluated in np.longdouble (80-bit, 63 mantissa bits, checked at
import): NumPy's float64 transcendentals may use SIMD routines that are not correctly rounded.  Host rounding adds
at most 2^-58 of the magnitudes involved (pairwise sums of up to 2^24 long double terms), which each bound includes.
First-order bounds are scaled by 1 + 2^-40 for the second-order terms.

Gates (ratio = |GPU - reference| / bound, pass <= 1; "exact" = bit equality):

  philox, u53        exact (oracle/mcl.py restates them; tests/test_gpu_mcl.py compares the words).
  init global        keyframe k = min(floor(fl(u K)), K - 1) exact; r = fl(radius fl(sqrt u)) and phi = fl(2 pi u)
                     exact; x = kf_x + r cos(phi): |err| <= 5 u |r cos| + u |x| (cos 4 u, product, add).  theta =
                     pi - fl(2 pi u) (or one DFMA): u |2 pi u| + u |theta|.  lw = -log n: 2 u log n.
  init pose, motion  Box-Muller: r = sqrt(-2 log u_a) within 2 u (log's 2 u halves under sqrt, then sqrt rounds),
                     n0 = r cos a and n1 = r sin a within 7 u.  e = d + s n: 8 u |s n| + u |e|.  Motion's x' = (x +
                     c ex) - s ey: 5 u |c ex| + |c| E_ex + 5 u |s ey| + |s| E_ey + u |x + c ex| + u |x'|.  theta'
                     = wrap_pi(v), v = fl(theta + dtheta) + s_t n2 (exactly v when s_t = 0) within E_v = 8 u |s_t n2|
                     + u |v|; wrap_pi is restated exactly and is monotone between its wraps, so theta' must lie in
                     wrap_pi of the double interval [v - E_v, v + E_v] (crossing the wrap: at or above the low end
                     or at or below the high end).  The ratio printed is the distance modulo 2 pi over E_v + u (|v| +
                     pi) + 3 pi u (wrap_pi's three adds).
  lookup, touched    exact: the raster lookup (oracle/mcl.lookup), and k_mcl_compact restated tile by tile with its
                     ballots and warp prefix.
  loglik             O, the expected bin e, d, D, t1 = fl(fl(1 - O) / s_o), t2 = fl(D / s_psi) are exact; ll =
                     -(t1^2 + t2^2) / 2 within u (t1^2 / 2 + t2^2 / 2 + |ll|) + 3 2^-1074; -inf exactly where the
                     restated float64 squares overflow.
  max                m = max_i fl(lw_i + ll_i): exact (order-free).
  S                  terms exp(fl(z_i - m)), z_i = fl(lw_i + ll_i): each within e_i (u |z_i - m| + 2 u) + 2^-1074;
                     the sum in the kernel's order (grid-stride chains over min(ceil(N / 256), 1024) blocks, the 256-
                     thread tree, k_mcl_final's 1024-slot tree) adds u sum_k |s_k| over every partial sum s_k.
  L, weights, lw     L = m + log S (GPU's m and S) within E_L = 2 u |log S| + u |L|; lw' = z - L within E_L + u
                     |lw'|; w = exp(lw') within w (E_lw' + 2 u) + 2 2^-1074.
  six sums           from the GPU's weights: w exact, w^2, w x, w y within u |t| + 2^-1074, w sin, w cos within 5 u |t|
                     + 2^-1074; plus u sum_k |s_k| in the kernel's order.  ESS = 1 / S2 within ess (b2 / S2) / (1 - b2
                     / S2) + u ess; x = Sx / Sw within (bx + |x| bw) / (Sw - bw) + u |x|, likewise y; theta =
                     atan2(Ss, Sc) within r / (1 - r) + 4 u |theta|, r = hypot(bs, bc) / hypot(Ss, Sc) (the
                     1 / hypot conditioning), compared modulo 2 pi.
  decision           fl(rho N) restated; the GPU's decision must be its own ESS < fl(rho N), and equal the model's
                     unless the reference ESS lies within its bound of fl(rho N) (a tie band: counted).
  prefix, u0         exact: 8 sequential weights per thread, the Hillis-Steele scan, the tile totals, the exclusive
                     tile offsets in order; u0 from Philox.
  ancestors, gather  exact: the kernel's binary search over the GPU's prefix with t_j = fl(fl(j + u0) / N); the new
                     set is the motion output at the ancestors, log-weights the bits of -log N.
"""
import numpy as np

from . import mcl as om

U = 2.0 ** -53
TINY = 2.0 ** -1074
HOST = 2.0 ** -58
SECOND = 1.0 + 2.0 ** -40
THREADS = 256
RED_BLOCKS = 1024
SCAN_PER = 8
SCAN_TILE = THREADS * SCAN_PER
COMPACT = 1024
PI, TWO_PI = om.PI, om.TWO_PI
REL = {'exp': 2 * U, 'log': 2 * U, 'sin': 4 * U, 'cos': 4 * U, 'atan2': 4 * U}   # 1, 1, 2, 2, 2 ulp
MUTANTS = ('drop_last', 'final_256', 'scan_shift', 'offsets_inclusive', 'warp_le', 'slot_plus_one', 'bin_trunc',
           'wrap_minus_pi', 'motion_new_theta', 'box_muller_swapped', 'resample_ge', 'estimate_unnormalized',
           'normalize_no_m')

if np.finfo(np.longdouble).nmant != 63:
  raise ImportError('oracle.mcl_stages needs an 80-bit np.longdouble (x86) for the host side of its bounds')
LD = np.longdouble


def _ld(a):
  return np.asarray(a, LD)


def dev(fn, *a):
  """The restatement's stand-in for a device function: the long double value rounded to float64 (within 1/2 ulp
  plus 2^-63 relative, inside the device's documented error)."""
  return getattr(np, fn)(*[_ld(x) for x in a]).astype(np.float64)


def red_blocks(n):
  return max(1, min((n + THREADS - 1) // THREADS, RED_BLOCKS))


def _ratio(err, bound):
  err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
  with np.errstate(invalid='ignore', divide='ignore'):
    r = np.where(err == 0, 0.0, err / bound)
  return np.where(np.isnan(r), np.inf, r)


# ---- exact restatements ---------------------------------------------------------------------------------------------
def wrap_pi(a, mutant=None):
  r = om.wrap_pi(a)
  if mutant == 'wrap_minus_pi':
    r = np.where(r == PI, -PI, r)
  return r


def box_muller(w, mutant=None):
  r = np.sqrt(-2.0 * dev('log', om.u53(w[:, 0], w[:, 1])))
  a = TWO_PI * om.u53(w[:, 2], w[:, 3])
  c, s = dev('cos', a), dev('sin', a)
  if mutant == 'box_muller_swapped':
    c, s = s, c
  return r * c, r * s


def _normals(seed, i, step, stream):
  """(n0, n1, n2) of particles i: the reference values in long double and the Box-Muller inputs."""
  w0 = om.philox(seed, om.counters(i, step, stream, 0))
  w1 = om.philox(seed, om.counters(i, step, stream, 1))
  out = []
  for w, keep in ((w0, 2), (w1, 1)):
    r = np.sqrt(-2.0 * np.log(_ld(om.u53(w[:, 0], w[:, 1]))))
    a = TWO_PI * om.u53(w[:, 2], w[:, 3])
    out += [r * np.cos(_ld(a)), r * np.sin(_ld(a))][:keep]
  return out


def restate_init_global(n, seed, kf, radius, mutant=None):
  kf = np.asarray(kf, np.float64)
  i = np.arange(n)
  b0 = om.philox(seed, om.counters(i, 0, om.STREAM_INIT, 0))
  b1 = om.philox(seed, om.counters(i, 0, om.STREAM_INIT, 1))
  K = kf.shape[0]
  k = np.minimum((om.u53(b0[:, 0], b0[:, 1]) * K).astype(np.int64), K - 1)
  r = radius * np.sqrt(om.u53(b0[:, 2], b0[:, 3]))
  phi = TWO_PI * om.u53(b1[:, 0], b1[:, 1])
  th = PI - TWO_PI * om.u53(b1[:, 2], b1[:, 3])
  lw = -dev('log', float(n))
  return np.stack([kf[k, 0] + r * dev('cos', phi), kf[k, 1] + r * dev('sin', phi), th, np.full(n, lw)])


def restate_init_pose(n, seed, pose, sigma, mutant=None):
  i = np.arange(n)
  n0, n1 = box_muller(om.philox(seed, om.counters(i, 0, om.STREAM_INIT, 0)), mutant)
  n2, _ = box_muller(om.philox(seed, om.counters(i, 0, om.STREAM_INIT, 1)), mutant)
  return np.stack([pose[0] + sigma[0] * n0, pose[1] + sigma[1] * n1, wrap_pi(pose[2] + sigma[2] * n2, mutant),
                   np.full(n, -dev('log', float(n)))])


def restate_motion(x, y, th, seed, step, odom, sigma, mutant=None):
  i = np.arange(np.size(x))
  n0, n1 = box_muller(om.philox(seed, om.counters(i, step, om.STREAM_MOTION, 0)), mutant)
  n2, _ = box_muller(om.philox(seed, om.counters(i, step, om.STREAM_MOTION, 1)), mutant)
  th2 = wrap_pi(th + odom[2] + sigma[2] * n2, mutant)
  a = th2 if mutant == 'motion_new_theta' else th
  c, s = dev('cos', a), dev('sin', a)
  ex = odom[0] + sigma[0] * n0
  ey = odom[1] + sigma[1] * n1
  return x + c * ex - s * ey, y + s * ex + c * ey, th2


def restate_compact(k, K, mutant=None):
  """k_mcl_compact over the lookup ``k``: (touched [count], slot [K]), tile by tile of 1024 keyframes with the
  warps' ballots and the warp-sum prefix.  Positions the kernel does not write hold -1."""
  flags = np.zeros(K, np.int64)
  k = np.asarray(k)
  flags[k[k >= 0]] = 1
  touched = np.full(K + 1, -1, np.int64)
  slot = np.full(K, -1, np.int64)
  base = 0
  lane = np.arange(32)
  below = (lane[None, :] < lane[:, None]) if mutant != 'warp_le' else (lane[None, :] <= lane[:, None])
  for k0 in range(0, K, COMPACT):
    f = np.zeros(COMPACT, np.int64)
    m = min(COMPACT, K - k0)
    f[:m] = flags[k0:k0 + m]
    fw = f.reshape(COMPACT // 32, 32)
    in_warp = fw @ below.T.astype(np.int64)                 # popc(ballot & lanes below)
    warp_sum = fw.sum(1)
    before = np.concatenate([[0], np.cumsum(warp_sum)[:-1]])
    pos = (base + before[:, None] + in_warp).reshape(-1)[:m]
    fk = f[:m] == 1
    slot[k0:k0 + m] = np.where(fk, pos + (1 if mutant == 'slot_plus_one' else 0), -1)
    touched[pos[fk]] = np.arange(k0, k0 + m)[fk]
    base += int(warp_sum.sum())
  return touched[:base], slot


def expected_bin(psi, width, mutant=None):
  q = -(np.asarray(psi) / PI) * width * 0.5
  f = np.trunc(q) if mutant == 'bin_trunc' else np.floor(q)
  return (f + width // 2).astype(np.int64)


def _loglik_terms(k, th, kf_theta, slot, overlap, yaw, width, s_o, s_psi, mutant=None):
  """(t1, t2) of every particle, exact: the kernel's O, D and divisions."""
  k = np.asarray(k)
  inside = k >= 0
  O = np.zeros(k.size)
  D = np.full(k.size, PI)
  j = np.asarray(slot)[k[inside]]
  ov = np.asarray(overlap, np.float32)
  jj = np.minimum(j, ov.size - 1)                          # a defective slot may point past the list
  O[inside] = ov[jj].astype(np.float64)
  a = 180 - np.asarray(yaw, np.int64)[jj]
  psi = om.wrap_pi(np.asarray(th, np.float64)[inside] - np.asarray(kf_theta, np.float64)[k[inside]])
  e = expected_bin(psi, width, mutant)
  d = (a - e) % width
  d = np.minimum(d, width - d)
  D[inside] = d * (TWO_PI / width)
  with np.errstate(over='ignore', invalid='ignore'):
    return (1.0 - O) / s_o, D / s_psi


def restate_loglik(k, th, kf_theta, slot, overlap, yaw, width, s_o, s_psi, mutant=None):
  t1, t2 = _loglik_terms(k, th, kf_theta, slot, overlap, yaw, width, s_o, s_psi, mutant)
  with np.errstate(over='ignore', invalid='ignore'):
    return -0.5 * (t1 * t1) - 0.5 * (t2 * t2)


def kernel_sum(t, mutant=None):
  """(value, sum of |every partial sum|) of the terms ``t`` [n] reduced as k_mcl_* and k_mcl_final do."""
  t = np.asarray(t, np.float64)
  n = t.size
  G = red_blocks(n)
  T = G * THREADS
  if mutant == 'drop_last':
    t = t[:-1]
  rows = -(-n // T)
  a = np.zeros(rows * T)
  a[:t.size] = t
  a = a.reshape(rows, T)
  mag = 0.0
  acc = np.zeros(T)
  for r in range(rows):                                    # each thread's grid-stride chain
    acc = acc + a[r]
    mag += float(np.abs(acc).sum())
  sm = acc.reshape(G, THREADS)
  s = THREADS // 2
  while s >= 1:                                            # the block's tree
    sm[:, :s] = sm[:, :s] + sm[:, s:2 * s]
    mag += float(np.abs(sm[:, :s]).sum())
    s //= 2
  p = np.zeros(RED_BLOCKS)
  p[:G] = sm[:, 0]
  s = RED_BLOCKS // (4 if mutant == 'final_256' else 2)
  while s >= 1:                                            # k_mcl_final's tree
    p[:s] = p[:s] + p[s:2 * s]
    mag += float(np.abs(p[:s]).sum())
    s //= 2
  return float(p[0]), mag


def restate_update(lw, ll, x, y, th, rho, seed, step, mutant=None):
  """The update from the set's log-weights ``lw`` and the GPU's ``ll``: dict of the scalars (m, S, ess, x, y,
  theta, resampled, u0), the new log-weights 'lw' and the weights 'w'."""
  n = np.size(lw)
  z = np.asarray(lw, np.float64) + np.asarray(ll, np.float64)
  m = float(np.max(z))
  S, _ = kernel_sum(dev('exp', z - m), mutant)
  L = (0.0 if mutant == 'normalize_no_m' else m) + float(dev('log', S))
  lw2 = z - L
  w = dev('exp', lw2)
  we = dev('exp', z - m) if mutant == 'estimate_unnormalized' else w
  with np.errstate(under='ignore'):
    sums = [kernel_sum(v, mutant)[0] for v in (we, we * we, we * x, we * y, we * dev('sin', th), we * dev('cos', th))]
  ess = 1.0 / sums[1]
  return {'m': m, 'S': S, 'ess': ess, 'x': sums[2] / sums[0], 'y': sums[3] / sums[0],
          'theta': float(dev('arctan2', sums[4], sums[5])), 'resampled': float(ess < rho * float(n)),
          'u0': om.resample_u0(seed, step), 'lw': lw2, 'w': w}


def restate_prefix(w, mutant=None):
  """The inclusive prefix sum of k_mcl_tile_sums, k_mcl_tile_offsets and k_mcl_prefix, bit for bit."""
  w = np.asarray(w, np.float64)
  n = w.size
  tiles = -(-n // SCAN_TILE)
  own = np.zeros(tiles * SCAN_TILE)
  own[:n] = w
  own = own.reshape(tiles, THREADS, SCAN_PER)
  t = np.zeros((tiles, THREADS))
  for j in range(SCAN_PER):
    t = t + own[:, :, j]
  sm = t
  s = 1
  while s < THREADS:                                       # Hillis-Steele over the threads
    new = sm.copy()
    lag = s - 1 if mutant == 'scan_shift' else s
    new[:, s:] = sm[:, s:] + sm[:, s - lag:THREADS - lag] if lag else sm[:, s:] + sm[:, s:]
    sm = new
    s *= 2
  excl = np.concatenate([np.zeros((tiles, 1)), sm[:, :-1]], 1)
  total = sm[:, -1]
  off = np.zeros(tiles)
  run = 0.0
  for b in range(tiles):                                   # exclusive, in tile order
    if mutant == 'offsets_inclusive':
      run += total[b]
      off[b] = run
    else:
      off[b] = run
      run += total[b]
  c = off[:, None] + excl
  out = np.zeros((tiles, THREADS, SCAN_PER))
  for j in range(SCAN_PER):
    c = c + own[:, :, j]
    out[:, :, j] = c
  return out.reshape(-1)[:n]


def restate_ancestors(cdf, u0, mutant=None):
  """k_mcl_resample's binary search: the least i with C_i > t_j (clamped to n - 1), t_j = fl(fl(j + u0) / n)."""
  cdf = np.asarray(cdf, np.float64)
  n = cdf.size
  t = (np.arange(n, dtype=np.float64) + u0) / float(n)
  lo = np.zeros(n, np.int64)
  hi = np.full(n, n - 1, np.int64)
  while True:
    act = lo < hi
    if not act.any():
      return lo
    mid = lo + (hi - lo) // 2
    up = cdf[mid] >= t if mutant == 'resample_ge' else cdf[mid] > t
    hi = np.where(act & up, mid, hi)
    lo = np.where(act & ~up, mid + 1, lo)


# ---- gates ----------------------------------------------------------------------------------------------------------
def _mod(d, period):
  d = _ld(d)
  return d - np.round(d / _ld(period)) * _ld(period)


def _theta_gate(got, v_ref, bound_v):
  """(ratio, outside) of wrapped angles ``got`` against the exact v_ref known within bound_v (0: v is exact)."""
  got = np.asarray(got, np.float64)
  v64 = v_ref.astype(np.float64)
  exact = bound_v == 0
  lo = np.where(exact, v64, np.nextafter((v_ref - bound_v).astype(np.float64), -np.inf))
  hi = np.where(exact, v64, np.nextafter((v_ref + bound_v).astype(np.float64), np.inf))
  olo, ohi = om.wrap_pi(lo), om.wrap_pi(hi)
  inside = np.where(olo <= ohi, (got >= olo) & (got <= ohi), (got >= olo) | (got <= ohi))
  bound = (bound_v + U * (np.abs(v_ref) + PI) + 3 * PI * U) * SECOND
  r = _ratio(np.abs(_mod(_ld(got) - v_ref, TWO_PI)).astype(np.float64), np.asarray(bound, np.float64))
  return np.where(inside, r, np.inf), int(np.count_nonzero(~inside))


def _lw0_gate(got, n):
  ref = -np.log(LD(n))
  return _ratio(np.abs(_ld(got) - ref).astype(np.float64), float(2 * U * abs(ref) * SECOND + TINY))


def check_init_global(n, seed, kf, radius, got):
  """Ratios [4, n] (x, y, theta, lw) of the GPU's initial set ``got`` [4, n]."""
  kf = np.asarray(kf, np.float64)
  got = np.asarray(got, np.float64)
  i = np.arange(n)
  b0 = om.philox(seed, om.counters(i, 0, om.STREAM_INIT, 0))
  b1 = om.philox(seed, om.counters(i, 0, om.STREAM_INIT, 1))
  K = kf.shape[0]
  k = np.minimum((om.u53(b0[:, 0], b0[:, 1]) * K).astype(np.int64), K - 1)
  r = radius * np.sqrt(om.u53(b0[:, 2], b0[:, 3]))
  phi = _ld(TWO_PI * om.u53(b1[:, 0], b1[:, 1]))
  out = np.zeros((4, n))
  for row, f in ((0, np.cos), (1, np.sin)):
    rc = _ld(r) * f(phi)
    ref = _ld(kf[k, row]) + rc
    bound = (5 * U * np.abs(rc) + U * np.abs(ref)) * SECOND + HOST * (np.abs(rc) + np.abs(_ld(kf[k, row]))) + 2 * TINY
    out[row] = _ratio(np.abs(_ld(got[row]) - ref).astype(np.float64), bound.astype(np.float64))
  q = _ld(TWO_PI) * _ld(om.u53(b1[:, 2], b1[:, 3]))
  ref = _ld(PI) - q
  bound = (U * q + U * np.abs(ref)) * SECOND + HOST * _ld(PI)
  out[2] = _ratio(np.abs(_ld(got[2]) - ref).astype(np.float64), bound.astype(np.float64))
  out[3] = _lw0_gate(got[3], n)
  return out


def _affine_gate(base, s, nrm):
  """(reference, bound) of fl(base + s n) with n = nrm (long double reference of a 7 u Box-Muller normal)."""
  sn = _ld(s) * nrm
  ref = _ld(base) + sn
  return ref, np.where(sn == 0, 0.0, (8 * U * np.abs(sn) + U * np.abs(ref)) * SECOND + HOST * (np.abs(sn) + np.abs(
      _ld(base))) + 2 * TINY)


def check_init_pose(n, seed, pose, sigma, got):
  got = np.asarray(got, np.float64)
  n0, n1, n2 = _normals(seed, np.arange(n), 0, om.STREAM_INIT)
  out = np.zeros((4, n))
  for row, nrm in ((0, n0), (1, n1)):
    ref, bound = _affine_gate(pose[row], sigma[row], nrm)
    out[row] = _ratio(np.abs(_ld(got[row]) - ref).astype(np.float64), np.asarray(bound, np.float64))
  v, bv = _affine_gate(pose[2], sigma[2], n2)
  out[2], _ = _theta_gate(got[2], v, bv)
  out[3] = _lw0_gate(got[3], n)
  return out


def check_motion(x, y, th, seed, step, odom, sigma, got):
  """Ratios [3, n] of the GPU's motion output ``got`` [3, n] from the set (x, y, theta) before the predict."""
  x, y, th = (np.asarray(a, np.float64) for a in (x, y, th))
  got = np.asarray(got, np.float64)
  n0, n1, n2 = _normals(seed, np.arange(x.size), step, om.STREAM_MOTION)
  ex, bex = _affine_gate(odom[0], sigma[0], n0)
  ey, bey = _affine_gate(odom[1], sigma[1], n1)
  c, s = np.cos(_ld(th)), np.sin(_ld(th))
  out = np.zeros((3, x.size))
  # x' = (x + c ex) - s ey, y' = (y + s ex) + c ey
  for row, p, ca, cb, sign in ((0, x, c, s, -1), (1, y, s, c, 1)):
    pa, pb = ca * ex, cb * ey
    mid = _ld(p) + pa
    ref = mid + sign * pb
    bound = ((5 * U * np.abs(pa) + np.abs(ca) * bex + 5 * U * np.abs(pb) + np.abs(cb) * bey + U * np.abs(mid)
              + U * np.abs(ref)) * SECOND + HOST * (np.abs(_ld(p)) + np.abs(pa) + np.abs(pb)) + 4 * TINY)
    out[row] = _ratio(np.abs(_ld(got[row]) - ref).astype(np.float64), bound.astype(np.float64))
  a = th + odom[2]                                          # fl(theta + dtheta): exact restatement
  v, bv = _affine_gate(a, sigma[2], n2)
  out[2], _ = _theta_gate(got[2], v, bv)
  return out


def check_touched(k, K, touched, count):
  """Entries of the GPU's touched list (and its count) that differ from the model's; 0 passes."""
  want, _ = restate_compact(k, K)
  got = np.asarray(touched, np.int64)[:count]
  if count != want.size:
    return max(count, want.size)
  return int(np.count_nonzero(got != want))


def check_loglik(k, th, kf_theta, touched, overlap, yaw, width, s_o, s_psi, got):
  """Ratios [n] of the GPU's log-likelihood ``got`` from its lookup, headings and touched list."""
  K = np.size(kf_theta)
  slot = np.full(K, -1, np.int64)
  slot[np.asarray(touched, np.int64)] = np.arange(np.size(touched))
  t1, t2 = _loglik_terms(k, th, kf_theta, slot, overlap, yaw, width, s_o, s_psi)
  with np.errstate(over='ignore', invalid='ignore'):
    ovf = ~np.isfinite(-0.5 * (t1 * t1) - 0.5 * (t2 * t2))
  h = 0.5 * _ld(t1) ** 2 + 0.5 * _ld(t2) ** 2
  ref = -h
  got = np.asarray(got, np.float64)
  bound = (U * (h + np.abs(ref))) * SECOND + HOST * h + 3 * TINY
  with np.errstate(invalid='ignore'):
    r = _ratio(np.abs(_ld(got) - ref).astype(np.float64), bound.astype(np.float64))
  return np.where(ovf, np.where(got == -np.inf, 0.0, np.inf), r)


def check_update(lw, ll, x, y, th, n_rho, scal, w, lw_new=None, seed=None, step=None):
  """Gates of one update from the set's log-weights ``lw``, the GPU's ``ll`` and motion output (x, y, th), with the
  GPU's SCALARS ``scal`` [8], weights ``w`` and, when it did not resample, new log-weights ``lw_new``.
  ``n_rho`` = fl(rho N).  Returns a dict of the largest ratio per stage (weights, lw as arrays), the mismatches
  'exact' of the exact stages and 'tie' (1 when the decision lay in its tie band)."""
  lw, ll, x, y, th, w = (np.asarray(a, np.float64) for a in (lw, ll, x, y, th, w))
  scal = np.asarray(scal, np.float64)
  m_gpu, S_gpu, ess_gpu, x_gpu, y_gpu, th_gpu, dec_gpu, u0_gpu = scal
  rep = {'exact': 0, 'tie': 0}
  z = lw + ll
  fin = np.isfinite(z)
  m = float(np.max(z))
  rep['exact'] += int(m_gpu != m)
  # S from the GPU's m; a term at -inf is exactly 0 on both sides
  dz = _ld(z) - LD(m_gpu)
  e = np.exp(dz)
  _, mag = kernel_sum(dev('exp', z - m_gpu))
  S_ref = np.sum(e)
  terr = np.where(fin, e * (U * np.abs(np.where(fin, dz, 0)) + REL['exp']), 0)
  bound_S = (np.sum(terr) + z.size * TINY + U * mag) * SECOND + HOST * S_ref
  rep['S'] = float(_ratio(float(abs(LD(S_gpu) - S_ref)), float(bound_S)))
  # L, the log-weights and the weights from the GPU's m and S
  logS = np.log(LD(S_gpu))
  L = LD(m_gpu) + logS
  bound_L = (REL['log'] * abs(logS) + U * abs(L)) * SECOND + HOST * (abs(L) + abs(logS))
  lw_ref = np.where(fin, _ld(z) - L, 0)
  bound_lw = bound_L + U * np.abs(lw_ref) * SECOND + HOST * np.abs(lw_ref)
  if lw_new is not None:                                   # -inf stays -inf
    r = _ratio(np.abs(_ld(lw_new) - lw_ref).astype(np.float64), bound_lw.astype(np.float64))
    rep['lw'] = np.where(fin, r, np.where(np.asarray(lw_new) == -np.inf, 0.0, np.inf))
  w_ref = np.where(fin, np.exp(lw_ref), 0)
  bound_w = w_ref * ((bound_lw * SECOND + REL['exp']) * SECOND + HOST) + 2 * TINY
  rep['weights'] = _ratio(np.abs(_ld(w) - w_ref).astype(np.float64), bound_w.astype(np.float64))
  # the six sums from the GPU's weights, then the estimate
  wl = _ld(w)
  ref, bnd = [], []
  for j, rel in enumerate((0.0, U, U, U, 5 * U, 5 * U)):
    f = (None, wl, _ld(x), _ld(y), np.sin(_ld(th)), np.cos(_ld(th)))[j]
    t = wl if f is None else wl * f
    with np.errstate(under='ignore'):
      _, mag = kernel_sum(t.astype(np.float64))               # the partial sums' magnitudes, to first order
    at = np.abs(t)
    ref.append(np.sum(t))
    bnd.append(float((rel * np.sum(at) + (w.size * TINY if rel else 0.0) + U * mag) * SECOND + HOST * np.sum(at)))
    del t, at
  Sw, S2, Sx, Sy, Ss, Sc = ref
  bw, b2, bx, by, bs, bc = bnd
  ess_ref = 1 / S2
  q = b2 / S2
  bound_ess = ess_ref * (q / (1 - q) + U) * SECOND + HOST * ess_ref
  rep['ess'] = float(_ratio(float(abs(LD(ess_gpu) - ess_ref)), float(bound_ess)))
  for key, Sv, bv, got in (('x', Sx, bx, x_gpu), ('y', Sy, by, y_gpu)):
    v = Sv / Sw
    bound = ((bv + abs(v) * bw) / (Sw - bw) + U * abs(v)) * SECOND + HOST * abs(v)
    rep[key] = float(_ratio(float(abs(LD(got) - v)), float(bound)))
  th_ref = np.arctan2(Ss, Sc)
  r = float(np.hypot(float(bs), float(bc)) / np.hypot(float(Ss), float(Sc)))
  bound_th = (r / (1 - r) if r < 1 else np.inf) * SECOND + REL['atan2'] * float(abs(th_ref)) * SECOND + HOST
  rep['theta'] = float(_ratio(float(abs(_mod(LD(th_gpu) - th_ref, 2 * np.pi))), bound_th))
  # the decision and u0
  rep['exact'] += int(dec_gpu != float(ess_gpu < n_rho))
  if abs(ess_ref - LD(n_rho)) <= bound_ess:
    rep['tie'] = 1
  else:
    rep['exact'] += int(dec_gpu != float(ess_ref < LD(n_rho)))
  if seed is not None:
    rep['exact'] += int(u0_gpu != om.resample_u0(seed, step))
  return rep


def check_prefix(w, got):
  """Entries of the GPU's prefix sum that differ from the model's in bits."""
  return int(np.count_nonzero(np.asarray(got, np.float64).view(np.uint64) != restate_prefix(w).view(np.uint64)))


def check_ancestors(cdf, u0, got):
  return int(np.count_nonzero(np.asarray(got, np.int64) != restate_ancestors(cdf, u0)))
