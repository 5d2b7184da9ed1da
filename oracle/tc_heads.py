"""Float64 model of the tensor-core heads (precision ``f16_tc``), stage by stage (TEST INFRASTRUCTURE).

Each function models one kernel from the GPU's own inputs to that kernel (read back with
``Engine.heads_stage``), so an error is caught in the stage that makes it and does not carry over.  Each
returns ``(model, tol)``: the value the kernel must store, computed in float64 with every fp16 rounding the
kernel makes, and a per-element bound on ``|gpu - model|``.  ``rounding=False`` switches the fp16 roundings
off; the stages then chain to the float64 oracle (``oracle.network.delta_head``) exactly.

Rounding points (``csrc/network_tc.cu``); ``h`` = fp16 round-to-nearest-even with subnormals kept:
* o1 (``k_gather_rows_f16``, ``k_delta_conv1_wgmma``): the operand copies are ``h(fp32(x - mu))``, the
  fp32 subtraction rounded first; ``|l - r|`` is one HSUB2 of two fp16 values, i.e. the exact difference
  rounded once to fp16; W1 is ``h(W1)``; the accumulators start at ``h(-mu_o1)`` and the result is stored
  as ``h(acc)``.  Bound: 1 fp16 ulp of the result plus ``2^-15 (sum |d| |W1| + |mu_o1|)`` for the fp32
  tensor-core accumulation, which truncates (120 K16 steps of at most 2^-22 relative each).
* x3 (``k_conv2_wgmma``): ``h(max(sum o1 (W2hi + W2lo) + b2eff, 0) - mu_x3)``, W2 split on the host as
  ``hi = h(W2)``, ``lo = h(W2 - hi)``.  Same form of bound (K = 960: 120 MMA steps with hi and lo).
  ReLU is 1-Lipschitz, so elements whose pre-activation lies within the bound of 0 need no exemption;
  ``near_kink`` counts them for the report.
* Dense partials (``k_conv3_wgmma``): ``sum_m relu(sum x3 h(W3) + b3eff) wd`` over each half of the 256
  channels, in fp32 (fmaf chain and two shuffles): the conv bound times ``|wd|`` plus ``2^-16`` of the
  sum of ``|relu wd|``.  Invalid rows (ib or jb >= 22) are exactly 0.
* overlap (``k_dense_finalize``): ``sigmoid(sum partial + bd)``, a fixed fp32 tree of 1152 values.
* b2eff / b3eff (``tc_pack_weights`` in double, ``k_fold_bias2`` / ``k_fold_bias3`` as fp32 fmaf chains of
  960 / 1152 terms): ``2^-13`` of the sum of the magnitudes of the terms.
* corr (``k_pack_corr``, ``k_corr_wgmma``, ``k_corr_finalize``): against the exact float64 correlation of
  the float32 volumes.  Each value is split as ``x = hi + lo + e``, ``hi = h(x)``, ``lo = h(x - hi)``:
  ``|e| <= 2^-22 |x|`` while lo is a normal number, and ``|e| <= 2^-25`` once lo is subnormal.  The product
  ``l r`` is formed as ``lhi rhi + llo rhi + lhi rlo``; the dropped ``llo rlo`` is at most ``2^-22 |l r|``.
  So the split contributes at most ``2^-20 A[k] + 2^-25 (|L|_1 + |R|_1)`` to bin k, with ``A`` the
  correlation of ``|L|`` and ``|R|``.  The fp32 accumulation (24 truncating MMA steps over K = 128, the
  diagonal sums of at most 64 terms, the 18-partial finalize) adds an allowance of ``2^-19 A[k]``.  This
  allowance is NOT a worst case: the worst case, ``(24 + 64 + 18) 2^-24`` relative, is 6e-6 and would not
  tell the three-term split from plain fp16 (which is 1e-5 off on leg-like volumes).  It is four times the
  mean truncation bias of the 24 MMA steps and far above the spread of the round-to-nearest sums; the GPU
  tests print the measured ratio of error to bound.
"""
import numpy as np

S15 = 15
U15 = 2.0 ** -15


def h(x):
  """fp16 round-to-nearest-even (subnormals kept) of float64 / float32 values, back in float64."""
  return np.asarray(x, np.float64).astype(np.float16).astype(np.float64)


def ulp16(x):
  """Spacing of the fp16 numbers at |x| (2^-24 at 0)."""
  a = np.minimum(np.abs(np.asarray(x, np.float64)), 65504.0).astype(np.float16)
  return np.spacing(a).astype(np.float64)


def operand(x, mu, rounding=True):
  """The fp16 operand copy of a volume (k_gather_rows_f16): h(fp32(x - mu))."""
  if not rounding:
    return np.asarray(x, np.float64) - np.asarray(mu, np.float64)
  return h(np.asarray(x, np.float32) - np.asarray(mu, np.float32))


def o1_stage(l, r, mu, w1, mu_o1, rounding=True):
  """o1[i, jb, o] of one pair (i < W, jb < W / 15): sum_{dj, c} |L[i, c] - R[15 jb + dj, c]| W1[dj, c, o] - mu_o1[o].
  l, r: (W, 128) volumes; mu: (128,) feature centre; w1: c_conv1 kernel (1, 15, 128, 64); mu_o1: (64,)."""
  L, R = operand(l, mu, rounding), operand(r, mu, rounding)
  W = np.asarray(w1, np.float64)[0]
  m0 = -np.asarray(mu_o1, np.float64)
  if rounding:
    W, m0 = h(W), h(m0)
  Wf = W.reshape(-1, W.shape[-1])
  Wa = np.abs(Wf)
  nb = L.shape[0] // S15
  acc = np.empty((L.shape[0], nb, W.shape[-1]))
  mag = np.empty_like(acc)
  for jb in range(nb):
    d = np.abs(L[:, None, :] - R[None, S15 * jb:S15 * jb + S15, :])      # exact difference of two fp16 values
    if rounding:
      d = h(d)                                                            # HSUB2 rounds it once
    d = d.reshape(L.shape[0], -1)
    acc[:, jb] = d @ Wf
    mag[:, jb] = d @ Wa
  acc += m0
  if not rounding:
    return acc, np.zeros_like(acc)
  err = U15 * (mag + np.abs(m0))
  model = h(acc)
  return model, ulp16(np.abs(model) + err) + err


def w2_split(w2):
  """W2 as the kernel applies it: hi + lo with hi = h(W2), lo = h(W2 - hi) (tc_pack_weights)."""
  w = np.asarray(w2, np.float32)
  hi = w.astype(np.float16)
  lo = (w - hi.astype(np.float32)).astype(np.float16)
  return hi.astype(np.float64) + lo.astype(np.float64)


def x3_stage(o1, w2, b2eff, mu_x3, rounding=True):
  """x3[ib, jb, n] of one pair from its o1 (W, nb, 64): max(sum_{di, o} o1[15 ib + di, jb, o] W2[di, o, n] + b2eff[n], 0)
  - mu_x3[n].  Returns (model, tol, near_kink): near_kink counts the elements whose pre-activation is within tol of 0."""
  W = w2_split(w2)[:, 0] if rounding else np.asarray(w2, np.float64)[:, 0]        # (15, 64, 128)
  o = np.asarray(o1, np.float64)
  nb = o.shape[0] // S15
  o = o.reshape(nb, S15, o.shape[1], o.shape[2])                                    # (ib, di, jb, o)
  b = np.asarray(b2eff, np.float64)
  m = np.asarray(mu_x3, np.float64)
  pre = np.einsum('adbo,don->abn', o, W) + b
  y = np.maximum(pre, 0) - m
  if not rounding:
    return y, np.zeros_like(y), 0
  err = U15 * (np.einsum('adbo,don->abn', np.abs(o), np.abs(W)) + np.abs(b) + np.abs(m))
  model = h(y)
  return model, ulp16(np.abs(model) + err) + err, int((np.abs(pre) <= err).sum())


def _conv3(x3, W3):
  nb = x3.shape[0]
  nv = nb - 2
  out = np.zeros((nv, nv, W3.shape[-1]))
  for kh in range(3):
    for kw in range(3):
      out += np.einsum('abc,cm->abm', x3[kh:kh + nv, kw:kw + nv], W3[kh, kw])
  return out


def dense_stage(x3, w3, b3eff, wd, rounding=True):
  """Dense partials of one pair from its x3 (nb, nb, 128): part[ib, jb, half] = sum over the channels m of that half
  of relu(c_conv3(x3)[ib, jb, m] + b3eff[m]) wd[(ib (nb-2) + jb) 256 + m]; 0 (tolerance 0) where ib or jb >= nb - 2."""
  x = np.asarray(x3, np.float64)
  nb = x.shape[0]
  nv = nb - 2
  W3 = np.asarray(w3, np.float64)
  if rounding:
    W3 = h(W3)
  b = np.asarray(b3eff, np.float64)
  pre = _conv3(x, W3) + b
  a = np.maximum(pre, 0)
  wdr = np.asarray(wd, np.float64).reshape(nv, nv, -1)
  half = W3.shape[-1] // 2
  model = np.zeros((nb, nb, 2))
  tol = np.zeros((nb, nb, 2))
  model[:nv, :nv] = (a * wdr).reshape(nv, nv, 2, half).sum(-1)
  if rounding:
    err = U15 * (_conv3(np.abs(x), np.abs(W3)) + np.abs(b))
    t = np.abs(wdr) * err + 2.0 ** -16 * np.abs(a * wdr)
    tol[:nv, :nv] = t.reshape(nv, nv, 2, half).sum(-1) + 2.0 ** -40
  return model, tol


def overlap_stage(partial, bd):
  """sigmoid(sum of a pair's Dense partials + bd) and its bound (k_dense_finalize)."""
  p = np.asarray(partial, np.float64)
  z = p.sum() + float(np.asarray(bd).reshape(-1)[0])
  ov = 1.0 / (1.0 + np.exp(-z))
  return ov, 0.25 * (2.0 ** -20 * np.abs(p).sum() + 2.0 ** -23 * abs(z)) + 2.0 ** -22


def b2eff_model(w, mu_o1):
  """b2eff = b2 + sum_{di, o} (b1[o] + mu_o1[o]) W2[di, o, n] (c_conv1 bias and o1 centre through c_conv2)."""
  k1, b1 = w['c_conv1']
  k2, b2 = w['c_conv2']
  W = np.asarray(k2, np.float64)[:, 0]                                             # (15, 64, 128)
  t1 = np.einsum('o,don->n', np.asarray(b1, np.float64), W)
  t2 = np.einsum('o,don->n', np.asarray(mu_o1, np.float64), W)
  base = np.asarray(b2, np.float64) + t1
  mag1 = np.abs(b2) + np.einsum('o,don->n', np.abs(np.asarray(b1, np.float64)), np.abs(W))
  mag2 = np.abs(base) + np.einsum('o,don->n', np.abs(np.asarray(mu_o1, np.float64)), np.abs(W))
  return base + t2, 2.0 ** -23 * mag1 + 2.0 ** -13 * mag2


def b3eff_model(w, mu_x3):
  """b3eff = b3 + sum_{tap, n} mu_x3[n] W3[tap, n, m] with the fp32 W3."""
  k3, b3 = w['c_conv3']
  W = np.asarray(k3, np.float64).reshape(9, 128, -1)
  m = np.asarray(mu_x3, np.float64)
  return (np.asarray(b3, np.float64) + np.einsum('n,tnm->m', m, W),
          2.0 ** -13 * (np.abs(b3) + np.einsum('n,tnm->m', np.abs(m), np.abs(W))))


def correlation(l, r):
  """Exact float64 correlation of two (W, C) volumes: corr[k] = sum_j <L[(k + j + W/2) mod W], R[j]>."""
  L = np.asarray(l, np.float64)
  R = np.asarray(r, np.float64)
  n = L.shape[0]
  G = L @ R.T
  j = np.arange(n)
  return np.array([G[(k + j + n // 2) % n, j].sum() for k in range(n)])


def corr_stage(l, r):
  """The exact correlation of one pair and the per-bin gate of the hi/lo split path: the split's derived bound plus
  the empirical allowance for the fp32 accumulation (module docstring)."""
  A = correlation(np.abs(l), np.abs(r))
  absolute = 2.0 ** -25 * (np.abs(np.asarray(l, np.float64)).sum() + np.abs(np.asarray(r, np.float64)).sum())
  return correlation(l, r), (2.0 ** -20 + 2.0 ** -19) * A + absolute


def corr_split(l, r, terms=('hh', 'lh', 'hl')):
  """The correlation the split operands give with exact accumulation, from the chosen products of the halves
  (hh = Lhi Rhi, lh = Llo Rhi, hl = Lhi Rlo): the kernel uses all three."""
  def split(x):
    x = np.asarray(x, np.float32)
    hi = x.astype(np.float16)
    return hi.astype(np.float64), (x - hi.astype(np.float32)).astype(np.float16).astype(np.float64)
  (lh, ll), (rh, rl) = split(l), split(r)
  parts = {'hh': (lh, rh), 'lh': (ll, rh), 'hl': (lh, rl)}
  return sum(correlation(*parts[t]) for t in terms)


def calibrate(v0, w, rounding=True):
  """Centres in the manner of calibrate_all (float64 means, so not bit for bit the GPU's): mu = h(channel means of
  V0); mu_o1 = h(channel means of o1 over the pair (V0, V0 rolled by half a turn)); mu_x3 = means of x3 there."""
  v0 = np.asarray(v0, np.float32)
  r0 = np.roll(v0, -v0.shape[0] // 2, axis=0)
  mu = h(v0.astype(np.float64).mean(0)) if rounding else v0.astype(np.float64).mean(0)
  o1, _ = o1_stage(v0, r0, mu, w['c_conv1'][0], np.zeros(64), rounding)
  mu_o1 = o1.reshape(-1, 64).mean(0)
  mu_o1 = h(mu_o1) if rounding else mu_o1
  o1, _ = o1_stage(v0, r0, mu, w['c_conv1'][0], mu_o1, rounding)
  b2eff, _ = b2eff_model(w, mu_o1)
  x3, _, _ = x3_stage(o1, w['c_conv2'][0], b2eff, np.zeros(128), rounding)
  return mu, mu_o1, x3.reshape(-1, 128).mean(0)
