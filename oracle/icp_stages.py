"""Float64 stage model of point-to-plane ICP (k_icp_pairs, csrc/icp.cu) and the gate each stage of one iteration, read
back by Engine.icp(..., want_stage=True), must pass.  Test infrastructure only; it builds on oracle/icp.py and the bin
classifier oracle/gt.bin_candidates.  Running a pair with iterations = k + 1 from the same init returns iteration k's
association and sums and the pose after it; the pose after k iterations is that iteration's input (a pair has the
same bits in any call).

Notation: u = 2^-53, gamma(k) = k u / (1 - k u), n = 6.

Gates:

  association  from the GPU's input pose T.  p = T v, the rotated normal m, d2 = |p - q|^2, cn = n_t . m and the tests
               d2 <= fl(d_k d_k), cn >= cos_normal are separately rounded IEEE operations in the kernel (apply3, dot3
               use __dmul_rn / __dadd_rn), restated bit for bit; only atan2 / asin of the bin are not.  Where
               bin_candidates calls the bin certain, the GPU's value must equal the model's; where it is ambiguous, it
               must equal the model's outcome at one of the candidate bins.  Gate: zero unexplained pixels; the
               ambiguous ones are counted.
  sums         from the GPU's own association.  J and e per pixel are bit-exact (explicit _rn operations; np.cross
               forms a_1 b_2 - a_2 b_1 with separate roundings like the kernel).  The error of each sum against the
               exact sum of the exact terms t_i (computed exactly: Dekker products and fsum) is at most
               u sum w_i |t_i| / (1 - u w_max), w_i the roundings term i passes: in thread tid = i mod 384's chain over
               pixels tid, tid + 384, .. a term at inlier position m of n_t takes its product rounding and the
               n_t - m + 1 adds after it (n_t for m = 1, whose add to 0 is exact); a contracted DFMA rounds once per
               add, which this covers; then the 5 xor-tree levels and thread 0's sum over the 12 warps (11 for warps
               0 and 1, 12 - w for warp w >= 2).  The inlier count S[27] is exact.
  update       from the GPU's S and input pose.  d* solves H d = -g exactly (fractions).  Higham Thm 10.4 gives
               (H + dH) d^ = -g with |dH| <= gamma(3n + 1) |L^| |L^T|, and (|L^| |L^T|)_ij <= |L^_i| |L^_j| =
               sqrt(H_ii H_jj) (1 + O(gamma(n + 1))), so with M = |H^-1| D, D_ij = gamma(3n + 1) sqrt(H_ii H_jj) /
               (1 - gamma(n + 1)): |d^ - d*| <= b = M |d*| + (M 1) |M |d*||_inf / (1 - |M|_inf).  The pose
               T' = [R(w) | v] T then moves by at most |dw|_2 sum_k |T_kj| (|R(a) - R(b)|_2 <= |a - b|_2 for the
               exponential of skew matrices) plus |dv_i| in column 3, and each of the GPU's Rodrigues and the
               reference's adds u (6 + 14 th + 18 th^2) sum_k |T_kj| (sqrt, division, sin / cos within 2 ulp,
               1 - cos, K^2 and the adds to I) and gamma(4) (sum_k |R_ik| |T_kj| + |v_i|) for the 4-term products.
               Row 3 is exactly 0 0 0 1.  A pair that ends DEGENERATE or TOO_FEW_INLIERS keeps its pose bit for bit.
  decisions    TOO_FEW_INLIERS (S[27] < min_inliers) is exact.  DEGENERATE: the kernel's trace and threshold
               fl(1e-12 fl(sum H_ii)) are restated bit for bit and compared with the exact pivots s_j of H (LDL^T in
               fractions); the GPU's pivot is the exact pivot of H + dH, off by at most x^T D x + gamma(n + 1) 2 H_jj,
               x = (-H_<j^-1 h_j, 1).  CONVERGED: d_k == d_end exactly, |w*| < eps_rot and |v*| < eps_trans with the
               GPU's norms within |b| + 3 u |d*| of the exact ones.  A quantity within its bound of its threshold
               lets either outcome pass; those are counted.
  result       rms = sqrt(S28 / S27) (0 without inliers), inliers = S27, valid and iterations: exact.
"""
import math
from fractions import Fraction

import numpy as np

from . import gt as G
from . import icp

U = 2.0 ** -53
THREADS = 384
WARPS = THREADS // 32
N = 6
MUTANTS_ASSOC = ('cos_unrotated', 'atan2_plus', 'schedule_advanced')
MUTANTS_SUMS = ('sums_float32', 'chain_drop_last', 'cross_reversed')
MUTANTS_DECISION = ('pivot_no_trace', 'converge_early')


def gamma(k):
  return k * U / (1 - k * U)


# ---- association ---------------------------------------------------------------------------------------------------
def _flat(vs, ns, vt, nt):
  return vs.reshape(-1, 4), ns.reshape(-1, 3), vt.reshape(-1, 4), nt.reshape(-1, 3)


def outcomes(T, vs, ns, vt, nt, dk, cos_normal, g, mutant=None, ulps=G.BIN_ULPS):
  """(src, cand [m, 4], out [m, 4], ambiguous [m]): the valid source pixels, their candidate target pixels
  (gt.candidate_pixels, the model's bin first) and the kernel's association at each candidate, -1 where the pair
  fails a test."""
  vs, ns, vt, nt = _flat(vs, ns, vt, nt)
  src = np.flatnonzero(icp.valid_source(vs, ns))
  v = vs[src].astype(np.float64)
  n = ns[src].astype(np.float64)
  px, py, pz = icp._apply(T, v[:, 0], v[:, 1], v[:, 2], True)
  c = G.bin_candidates(px, py, pz, g, ulps)
  if mutant == 'atan2_plus':
    _, _, yaw, pitch = G.range_angles(px, py, pz, g)
    c['bx'], c['by'] = G.angle_bins(-yaw, pitch, g)
    c['alt_x'], c['alt_y'] = c['bx'], c['by']
  cand = G.candidate_pixels(c, g['W'])
  if mutant == 'cos_unrotated':
    mx, my, mz = n[:, 0], n[:, 1], n[:, 2]
  else:
    mx, my, mz = icp._apply(T, n[:, 0], n[:, 1], n[:, 2], False)
  out = np.full(cand.shape, -1, np.int64)
  d2max = np.float64(dk) * np.float64(dk)
  for col in range(4):
    j = cand[:, col]
    w = vt[j].astype(np.float64)
    t = nt[j].astype(np.float64)
    dx, dy, dz = px - w[:, 0], py - w[:, 1], pz - w[:, 2]
    d2 = (dx * dx + dy * dy) + dz * dz
    cn = (t[:, 0] * mx + t[:, 1] * my) + t[:, 2] * mz
    ok = c['keep'] & (w[:, 3] > 0) & ~icp._fill(nt[j]) & (d2 <= d2max) & (cn >= cos_normal)
    out[ok, col] = j[ok]
  return src, cand, out, c['amb_x'] | c['amb_y']


def restate_association(T, vs, ns, vt, nt, dk, cos_normal, g, mutant=None):
  """The association at the model's bins, [HW] (-1 where none)."""
  src, _, out, _ = outcomes(T, vs, ns, vt, nt, dk, cos_normal, g, mutant)
  q = np.full(vs.reshape(-1, 4).shape[0], -1, np.int64)
  q[src] = out[:, 0]
  return q


def association_gate(T, vs, ns, vt, nt, dk, cos_normal, g, got):
  """(unexplained pixels, ambiguous pixels) of the GPU's association ``got`` [HW] from the input pose T."""
  got = np.asarray(got, np.int64).reshape(-1)
  src, _, out, amb = outcomes(T, vs, ns, vt, nt, dk, cos_normal, g)
  gs = got[src]
  explained = np.where(amb, np.any(out == gs[:, None], 1), out[:, 0] == gs)
  rest = np.ones(got.size, bool)
  rest[src] = False
  return int(np.count_nonzero(~explained) + np.count_nonzero(got[rest] != -1)), int(np.count_nonzero(amb))


# ---- sums ----------------------------------------------------------------------------------------------------------
def terms(T, vs, vt, nt, assoc, mutant=None):
  """(pixel index [m], terms [m, 29]) of the associated pixels in the kernel's per-pixel arithmetic (bit-exact)."""
  vs = vs.reshape(-1, 4)
  vt = vt.reshape(-1, 4)
  nt = nt.reshape(-1, 3)
  assoc = np.asarray(assoc, np.int64).reshape(-1)
  i = np.flatnonzero(assoc >= 0)
  J, e = icp.jacobian(T, vs, vt, nt, assoc)
  if mutant == 'cross_reversed':
    J[:, :3] = -J[:, :3]
  r, c = np.triu_indices(6)
  return i, np.concatenate([J[:, r] * J[:, c], J * e[:, None], np.ones((e.size, 1)), (e * e)[:, None]], 1)


def _factors(T, vs, vt, nt, assoc):
  vs = vs.reshape(-1, 4)
  vt = vt.reshape(-1, 4)
  nt = nt.reshape(-1, 3)
  J, e = icp.jacobian(T, vs, vt, nt, np.asarray(assoc, np.int64).reshape(-1))
  r, c = np.triu_indices(6)
  one = np.ones((e.size, 1))
  a = np.concatenate([J[:, r], J, one, e[:, None]], 1)
  b = np.concatenate([J[:, c], np.repeat(e[:, None], 6, 1), one, e[:, None]], 1)
  return a, b


def _two_prod(a, b):
  """(p, r) with p + r == a b exactly (Dekker; no overflow or underflow at these magnitudes)."""
  p = a * b
  s = 134217729.0
  ca, cb = s * a, s * b
  ah = ca - (ca - a)
  bh = cb - (cb - b)
  al, bl = a - ah, b - bh
  return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def weights(pix, HW):
  """w_i of each associated pixel (ascending pixel order): chain, xor tree and warp roundings (module docstring)."""
  tid = pix % THREADS
  order = np.argsort(tid, kind='stable')
  n_t = np.bincount(tid, minlength=THREADS)
  start = np.concatenate([[0], np.cumsum(n_t)[:-1]])
  m = np.empty(pix.size, np.int64)
  m[order] = np.arange(pix.size) - start[tid[order]] + 1
  chain = np.where(m == 1, n_t[tid], n_t[tid] - m + 2)
  warp = tid // 32
  return chain + 5 + np.where(warp == 0, WARPS - 1, WARPS - warp)


def sums_gate(T, vs, vt, nt, assoc, S):
  """(err / bound [29], exact count ok): the GPU's sums S against the exact sums of the exact terms."""
  a, b = _factors(T, vs, vt, nt, assoc)
  pix = np.flatnonzero(np.asarray(assoc).reshape(-1) >= 0)
  HW = np.asarray(assoc).size
  w = weights(pix, HW).astype(np.float64)
  p, r = _two_prod(a, b)
  wmax = float(w.max()) if w.size else 0.0
  bound = U * (w @ (np.abs(p) * (1 + U))) / (1 - U * wmax)
  ratio = np.zeros(29)
  for k in range(29):
    err = abs(math.fsum([float(S[k])] + (-p[:, k]).tolist() + (-r[:, k]).tolist()))
    ratio[k] = err / bound[k] if bound[k] > 0 else (0.0 if err == 0 else np.inf)
  return ratio, bool(S[27] == pix.size)


def restate_sums(T, vs, vt, nt, assoc, mutant=None):
  """The 29 sums in the kernel's order without contraction: each thread's chain, the xor tree, the warps in order."""
  pix, t = terms(T, vs, vt, nt, assoc, 'cross_reversed' if mutant == 'cross_reversed' else None)
  HW = np.asarray(assoc).size
  dt = np.float32 if mutant == 'sums_float32' else np.float64
  if mutant == 'chain_drop_last' and pix.size:
    tid = pix % THREADS
    keep = np.ones(pix.size, bool)
    keep[np.flatnonzero(tid == tid[-1])[-1]] = False
    pix, t = pix[keep], t[keep]
  steps = (HW + THREADS - 1) // THREADS
  full = np.zeros((steps * THREADS, 29), dt)
  full[pix] = t.astype(dt)
  full = full.reshape(steps, THREADS, 29)
  acc = np.zeros((THREADS, 29), dt)
  for s in range(steps):
    acc = acc + full[s]
  acc = acc.reshape(WARPS, 32, 29)
  lanes = np.arange(32)
  for o in (16, 8, 4, 2, 1):
    acc = acc + acc[:, lanes ^ o]
  x = acc[0, 0]
  for wp in range(1, WARPS):
    x = x + acc[wp, 0]
  return x.astype(np.float64)


# ---- solve, update and decisions ----------------------------------------------------------------------------------
def _H(S):
  A = np.zeros((6, 6))
  r, c = np.triu_indices(6)
  A[r, c] = S[:21]
  A[c, r] = S[:21]
  return A


def _frac_matrix(A):
  return [[Fraction(float(x)) for x in row] for row in A]


def exact_pivots(H):
  """The exact pivots s_0 .. of H's LDL^T (fractions), up to and including the first that is <= 0."""
  A = _frac_matrix(H)
  piv = []
  for j in range(6):
    s = A[j][j]
    piv.append(s)
    if s <= 0:
      break
    for i in range(j + 1, 6):
      f = A[i][j] / s
      for k in range(j + 1, 6):
        A[i][k] -= f * A[j][k]
  return piv


def exact_inverse(H):
  n = 6
  A = _frac_matrix(H)
  I = [[Fraction(int(i == j)) for j in range(n)] for i in range(n)]
  for j in range(n):
    p = next(i for i in range(j, n) if A[i][j] != 0)
    A[j], A[p] = A[p], A[j]
    I[j], I[p] = I[p], I[j]
    inv = 1 / A[j][j]
    A[j] = [x * inv for x in A[j]]
    I[j] = [x * inv for x in I[j]]
    for i in range(n):
      if i != j and A[i][j] != 0:
        f = A[i][j]
        A[i] = [x - f * y for x, y in zip(A[i], A[j])]
        I[i] = [x - f * y for x, y in zip(I[i], I[j])]
  return I


def _backward_D(H):
  dg = np.sqrt(np.maximum(np.diag(H), 0.0))
  return gamma(3 * N + 1) / (1 - gamma(N + 1)) * np.outer(dg, dg)


def pivot_threshold(S):
  """fl(1e-12 tr) with tr summed in the kernel's order from 0.0 (bit-exact)."""
  tr = 0.0
  for i in range(6):
    tr += float(S[[0, 6, 11, 15, 18, 20][i]])
  return icp.PIVOT * tr


def rodrigues_err(th):
  return U * (6 + 14 * th + 18 * th * th)


def model_step(S, dk, prm, mutant=None):
  """The model's decision on the GPU's sums: dict(status (None: go on), tie, d (exact solution, float64), b (its
  bound), kind of the tie)."""
  S = np.asarray(S, np.float64)
  if S[27] < prm['min_inliers']:
    return dict(status=icp.TOO_FEW_INLIERS, tie=False)
  H = _H(S)
  thr = icp.PIVOT if mutant == 'pivot_no_trace' else pivot_threshold(S)
  piv = exact_pivots(H)
  D = _backward_D(H)
  tie = False
  degenerate = False
  for j, s in enumerate(piv):
    if j == 0:
      band = D[0, 0]
    else:
      Hj = H[:j, :j]
      x = np.append(-np.linalg.lstsq(Hj, H[:j, j], rcond=None)[0], 1.0)
      band = float(np.abs(x) @ D[:j + 1, :j + 1] @ np.abs(x)) * (1 + 1e-6)
    band += gamma(N + 1) * 2 * H[j, j]
    if abs(float(s) - thr) <= band or not np.isfinite(band):
      tie = True
    if not s > thr:
      degenerate = True
      break
  if degenerate:
    return dict(status=icp.DEGENERATE, tie=tie)
  Hinv = exact_inverse(H)
  g = [Fraction(float(x)) for x in S[21:27]]
  d = np.array([float(-sum(Hinv[i][k] * g[k] for k in range(6))) for i in range(6)])
  M = np.abs(np.array([[float(x) for x in row] for row in Hinv])) @ D
  rho = float(np.abs(M).sum(1).max())
  b0 = M @ np.abs(d)
  b = b0 + M.sum(1) * (np.abs(b0).max() / (1 - rho)) if rho < 1 else np.full(6, np.inf)
  th, tn = float(np.linalg.norm(d[:3])), float(np.linalg.norm(d[3:]))
  bth = float(np.linalg.norm(b[:3])) + 3 * U * th
  btn = float(np.linalg.norm(b[3:])) + 3 * U * tn
  at_end = mutant == 'converge_early' or dk == prm['d_end']
  status = icp.CONVERGED if at_end and th < prm['eps_rot'] and tn < prm['eps_trans'] else None
  if at_end and (abs(th - prm['eps_rot']) <= bth or abs(tn - prm['eps_trans']) <= btn):
    tie = True
  return dict(status=status, tie=tie, d=d, b=b)


def decision_gate(m, got):
  """(mismatch, tie) of the status ``got`` against the model's decision ``m`` (model_step): within a tie band any
  outcome but TOO_FEW_INLIERS, which is exact, passes."""
  want = icp.MAX_ITERATIONS if m['status'] is None else m['status']
  if m['tie']:
    return int((got == icp.TOO_FEW_INLIERS) != (want == icp.TOO_FEW_INLIERS)), 1
  return int(got != want), 0


def pose_bound(T, d, b):
  """(reference pose [4, 4], per-element bound [4, 4]) of T' = [R(d) | v] T, d the exact update with bound b."""
  th = float(np.linalg.norm(d[:3]))
  R = np.eye(3)
  if th > 0:
    k = d[:3] / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = R + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)
  Uu = np.eye(4)
  Uu[:3, :3] = R
  Uu[:3, 3] = d[3:]
  ref = Uu @ T
  colT = np.abs(T[:3]).sum(0)                                     # sum_k |T_kj|, j = 0 .. 3
  dw = float(np.linalg.norm(b[:3])) + U * th
  dv = np.abs(b[3:]) + U * np.abs(d[3:])
  last = np.zeros(4)
  last[3] = 1.0
  bound = np.zeros((4, 4))
  bound[:3] = dw * colT[None, :] + np.outer(dv, last) + 2 * (
      rodrigues_err(th + float(np.linalg.norm(b[:3]))) * colT[None, :]
      + gamma(4) * (np.abs(R) @ np.abs(T[:3]) + np.outer(np.abs(d[3:]), last)))
  return ref, bound * (1 + 1e-10)


def ratio_max(err, bound):
  """max err / bound, an exact 0 / 0 counting as 0"""
  err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
  r = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err == 0, 0.0, np.inf))
  return float(r.max())


# ---- one iteration of one pair ---------------------------------------------------------------------------------------
def check_iteration(T, k, prm, g, vs, ns, vt, nt, stage):
  """Every gate of iteration k (0-based) of one pair from its input pose T.  ``stage``: the GPU's (or a restatement's)
  assoc [HW], system [29], pose [4, 4], status, iterations, inliers, rms, valid after iterations = k + 1.  Returns a
  report dict: unexplained / ambiguous pixels, sums and pose err / bound, decision mismatch and tie counts, result
  field mismatches."""
  dk = icp.distances(dict(prm, iterations=k + 1))[k]
  rep = {}
  rep['unexplained'], rep['ambiguous'] = association_gate(T, vs, ns, vt, nt, dk, prm['cos_normal'], g, stage['assoc'])
  ratio, count_ok = sums_gate(T, vs, vt, nt, stage['assoc'], stage['system'])
  rep['sums'] = float(ratio.max())
  S = np.asarray(stage['system'], np.float64)
  m = model_step(S, dk, prm)
  rep['decision'], rep['tie'] = decision_gate(m, stage['status'])
  rep['pose'] = 0.0
  if stage['status'] in (icp.DEGENERATE, icp.TOO_FEW_INLIERS):
    rep['pose'] = 0.0 if np.array_equal(np.asarray(stage['pose']).view(np.uint64), T.view(np.uint64)) else np.inf
  elif 'd' in m:
    ref, bound = pose_bound(T, m['d'], m['b'])
    P = np.asarray(stage['pose'])
    rep['pose'] = ratio_max(np.abs(P[:3] - ref[:3]), bound[:3])
    if not np.array_equal(P[3], [0.0, 0.0, 0.0, 1.0]):
      rep['pose'] = np.inf
  elif not m['tie']:
    rep['pose'] = np.inf                                  # the GPU went on where the model is degenerate
  rms = math.sqrt(S[28] / S[27]) if S[27] > 0 else 0.0
  valid = int(icp.valid_source(vs.reshape(-1, 4), ns.reshape(-1, 3)).sum())
  rep['fields'] = int((not count_ok) + (stage['rms'] != rms) + (stage['inliers'] != int(S[27]))
                      + (stage['valid'] != valid) + (stage['iterations'] != k + 1))
  return rep


def restate_iteration(T, k, prm, g, vs, ns, vt, nt, mutant=None):
  """A NumPy restatement of iteration k of the kernel from the pose T, in the form check_iteration reads (sums
  without contraction).  ``mutant`` names a defect to plant (MUTANTS_*)."""
  d = icp.distances(dict(prm, iterations=k + 2))
  dk = d[k + 1] if mutant == 'schedule_advanced' else d[k]
  assoc = restate_association(T, vs, ns, vt, nt, dk, prm['cos_normal'], g,
                              mutant if mutant in MUTANTS_ASSOC else None)
  S = restate_sums(T, vs, vt, nt, assoc, mutant if mutant in MUTANTS_SUMS else None)
  end, P = icp.solve_update(S, T, dk, prm)
  if mutant in MUTANTS_DECISION:
    end = model_step(S, dk, prm, mutant)['status']
    if end != icp.DEGENERATE:
      P = icp.solve_update(S, T, -1.0, dict(prm, min_inliers=0))[1]
  valid = int(icp.valid_source(vs.reshape(-1, 4), ns.reshape(-1, 3)).sum())
  return dict(assoc=assoc, system=S, pose=P, status=icp.MAX_ITERATIONS if end is None else end, iterations=k + 1,
              inliers=int(S[27]), rms=math.sqrt(S[28] / S[27]) if S[27] > 0 else 0.0, valid=valid)
