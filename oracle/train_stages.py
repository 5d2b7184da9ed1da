"""Float64 model of every stage of a training step, with a per-element bound on the kernel's rounding (TEST
INFRASTRUCTURE).

Each function models one stage from the GPU's own inputs to that stage (read back with ``Engine.train_stage``), so
an error is caught in the stage that makes it.  ReLU masks are taken from the GPU's own activations and the signs
of ``l - r`` from its own fp32 volumes (the sign of an fp32 difference is the sign of the exact one), so no mask or
sign can flip between the GPU and the model and the gates are per element.  Every function takes and returns
float64 torch tensors on the caller's device (the GPU in ``tests/test_gpu_train_stages.py``) and returns
``(model, bound)`` pairs; ``ratio(gpu, model, bound)`` is the largest ``|gpu - model| / bound``.

The bound of a product ``sum_k a_k b_k`` is ``u sum_k w_k |a_k| |b_k|`` (``u = 2^-24``, half an fp32 ulp relative),
where ``w_k`` counts the roundings the product of term k passes through in the kernel's own summation order, times
``1 / (1 - u max w)`` for the higher-order terms.  ``w_k`` depends on k alone, so it is folded into one operand and
the bound is one more float64 product of absolute values.
* fp32 (``k_simt_gemm``, ``k_delta_dgrad``, ``k_corr_backward``, ``k_dense_*``): an ``fmaf`` chain over the K slice
  in order; term j of an n-term chain passes through ``n - j`` roundings.  ``wgrad_gemm`` splits the reduction into
  ``nsplit`` slices of ``kchunk`` rows (``split_w`` restates its choice) that ``k_splitk_reduce`` adds in slice
  order: ``nsplit - z`` more for slice z.  An operand formed in fp32 (``|l - r|``) adds 1, a bias add 1.
* tf32x3 (``k_tc_gemm``, ``k_delta_dgrad_tc``): a product is ``lo_a hi_b + hi_a lo_b + hi_a hi_b`` with
  ``|x - hi - lo| <= 2^-22 |x|``; with the dropped ``lo_a lo_b`` a term is off by at most ``3 * 2^-22 = 12 u`` of
  ``|a b|`` (``TF32X3_SPLIT``).  The six MMAs of a K16 tile start from zero and truncate when they add into the
  accumulator: ``MMA_ULPS = 2`` fp32 ulps (4 u) of the tile's ``sum |a b|`` each, 24 u (``TF32X3_MMA``), an
  allowance for the tensor core's alignment like ``oracle/tc_leg.py``'s, not a proven worst case.  Each tile's
  partial is added to the running sum with one rounded FADD: tile t of T passes through ``T - t``.
* ``k_train_loss`` forms dz in double from the fp32 yhat and y and rounds once: dz is held to ``2^-22 |dz|``
  (2 ulps) of the exact derivative at those inputs.  The cancellation of ``1 - yhat`` as yhat -> 1 is exact
  (Sterbenz, yhat >= 1/2); what remains is the rounding of the stored yhat itself, which the overlap stage bounds
  absolutely (a relative bound would need the logit, which ``k_dense_sigmoid`` does not keep).
* ``k_dense_sigmoid``: a thread's strided ``fmaf`` chain, a 256-way tree (8 adds), the bias; then ``expf``
  (2 ulps), ``1 + e`` and the division: yhat within ``6 u yhat + sigmoid'(|z| - bz) bz`` of the model.
* ``k_corr_readout``: the diagonal sum of the Gram matrix in j order (``Wf - j`` adds).
* ``k_corr_dlogit``: ``expf``, the sigmoid and four fp32 operations, an absolute bound from their relative errors,
  plus fp32's range: past corr = 88.7 ``expf`` overflows and sigmoid(-corr) < 2^-126 is 0.
* ``k_delta_dgrad_reduce``: ``dfv_corr + part_0 + part_1 + ...`` in that order.
"""
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24
TF32X3_SPLIT = 12.0
MMA_ULPS = 2.0
TF32X3_MMA = 6 * 2 * MMA_ULPS
TF32X3_TERM = TF32X3_SPLIT + TF32X3_MMA
SPLIT_BLOCKS, MAX_SPLIT = 528, 32     # wgrad_gemm's target CTAs and most slices
PART_R_ADDS = 20                      # k_delta_dgrad: 4 rows of a thread + 16 thread rows (tc: 4 + 3 + 1)
f64 = torch.float64


def _cdiv(a, b):
  return -(-a // b)


def _factor(wmax):
  return 1.0 / (1.0 - float(wmax) * U)


def chain_w(K, prec, device=None):
  """w_k of one unsplit K-long product of k_simt_gemm (fp32) or k_tc_gemm (tf32x3), k in the kernel's order."""
  k = torch.arange(K, dtype=f64, device=device)
  if prec == 'fp32':
    return K - k
  return TF32X3_TERM + (_cdiv(K, 16) - torch.div(k, 16, rounding_mode='floor'))


def split_plan(Kred, M, N):
  """(nsplit, kchunk) of wgrad_gemm for an [M][N] result reduced over Kred rows."""
  tiles = _cdiv(M, 64) * _cdiv(N, 64)
  nsplit = min(_cdiv(SPLIT_BLOCKS, tiles), MAX_SPLIT)
  kchunk = _cdiv(_cdiv(Kred, nsplit), 16) * 16
  return _cdiv(Kred, kchunk), kchunk


def split_w(Kred, M, N, prec, device=None):
  """(w_m, slice z of row m) of the Kred reduction rows of wgrad_gemm."""
  nsplit, kchunk = split_plan(Kred, M, N)
  m = torch.arange(Kred, dtype=torch.int64, device=device)
  z = torch.div(m, kchunk, rounding_mode='floor')
  j = m - z * kchunk
  length = torch.clamp(Kred - z * kchunk, max=kchunk)
  if prec == 'fp32':
    w = (length - j) + (nsplit - z)
  else:
    w = TF32X3_TERM + (_cdiv_t(length, 16) - torch.div(j, 16, rounding_mode='floor')) + (nsplit - z)
  return w.to(f64), z


def _cdiv_t(a, b):
  return torch.div(a + b - 1, b, rounding_mode='floor')


def ratio(gpu, model, bound):
  """max |gpu - model| / bound (0 / 0 = 0, x / 0 = inf)."""
  err = (torch.as_tensor(gpu).to(model) - model).abs()
  r = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                  torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
  return float(r.max()) if r.numel() else 0.0


def exceeded(gpu, model, bound):
  """The fraction of elements outside their bound."""
  err = (torch.as_tensor(gpu).to(model) - model).abs()
  return float((err > bound).to(f64).mean())


def _nchw(x):
  return x.permute(0, 3, 1, 2)


def _oihw(w):
  return w.permute(3, 2, 0, 1)


# ---- forward ---------------------------------------------------------------------------------------------------
def conv_forward(x, w, b, stride, relu, prec):
  """A valid NHWC conv (leg layers, c_conv2, c_conv3) on x [n, H, W, C]: K = (dh, dw, c), the bias added after
  the chain, then the ReLU (1-Lipschitz)."""
  kh, kw, cin, _ = w.shape
  wk = (chain_w(kh * kw * cin, prec, x.device) + 1).reshape(kh, kw, cin, 1)
  model = F.conv2d(_nchw(x), _oihw(w), b, stride=stride).permute(0, 2, 3, 1)
  bound = F.conv2d(_nchw(x.abs()), _oihw(w.abs() * wk), b.abs(), stride=stride).permute(0, 2, 3, 1)
  if relu:
    model = model.clamp(min=0)
  return model, U * _factor(wk.max()) * bound


def delta_forward(L, R, w1, b1, prec):
  """c_conv1 on |l - r| (DeltaOperand) for volumes L, R [n, Wf, 128], w1 [1, s, 128, 64]: o1 [n, Wf, nb, 64]."""
  n, Wf, C = L.shape
  s = w1.shape[1]
  nb = Wf // s
  W = w1.reshape(s * C, -1)
  wk = chain_w(s * C, prec, L.device) + 2                 # the fp32 subtraction and the bias add
  Wa = W.abs() * wk[:, None]
  out, bnd = [], []
  for p in range(n):
    D = (L[p][:, None, None, :] - R[p][:nb * s].reshape(nb, s, C)[None]).abs().reshape(Wf * nb, s * C)
    out.append((D @ W + b1).reshape(Wf, nb, -1))
    bnd.append((D @ Wa + b1.abs()).reshape(Wf, nb, -1))
  return torch.stack(out), U * _factor(wk.max()) * torch.stack(bnd)


def dense_forward(x4, wd, bd):
  """k_dense_sigmoid on x4 [n, n_in]: (yhat model, bound)."""
  n_in = x4.shape[1]
  i = torch.arange(n_in, device=x4.device)
  t = i % 256
  w = (_cdiv_t(n_in - t, 256) - torch.div(i, 256, rounding_mode='floor') + 9).to(f64)
  z = x4 @ wd.reshape(-1) + bd.reshape(())
  bz = U * _factor(w.max()) * (x4.abs() @ (wd.reshape(-1).abs() * w) + bd.abs().reshape(()))
  y = torch.sigmoid(z)
  zz = (z.abs() - bz).clamp(min=0)
  sp = torch.sigmoid(zz) * (1 - torch.sigmoid(zz))
  return y, (1 + 1e-6) * (sp * bz + 6 * U * y)


def corr_forward(L, R, prec):
  """The Gram matrix (GramOperand, K = 128) and k_corr_readout's diagonal sums: corr [n, Wf]."""
  n, Wf, C = L.shape
  wc = chain_w(C, prec, L.device)
  k = torch.arange(Wf, device=L.device)
  idx = (k[:, None] + k[None, :] + Wf // 2) % Wf              # [k, j] -> row of G
  jj = k[None, :].expand(Wf, Wf)
  wj = (Wf - k).to(f64)
  out, bnd = [], []
  for p in range(n):
    G = L[p] @ R[p].T
    Gb = (L[p].abs() * wc) @ R[p].abs().T + (L[p].abs() @ R[p].abs().T) * wj[None, :]
    out.append(G[idx, jj].sum(1))
    bnd.append(Gb[idx, jj].sum(1))
  return torch.stack(out), U * _factor(wc.max() + Wf) * torch.stack(bnd)


# ---- loss and Dense --------------------------------------------------------------------------------------------
def dz(yhat, y):
  """dL/d(Dense logit) of k_train_loss per pair for the n pairs of one chunk, from the stored fp32 yhat."""
  n = yhat.numel()
  d = yhat - y
  u = (d.abs() + 0.25) * 24 - 12
  e = torch.exp(-u)
  model = 120.0 * e / (1 + e) ** 2 * torch.sign(d) / n * yhat * (1 - yhat)
  return model, 2.0 ** -22 * model.abs()


def dense_backward(x4, dzv, wd):
  """k_dense_backward of one chunk: (dWd [n_in], bound), (db, bound) from the GPU's dz, and (dpre3, bound) with
  the mask x4 > 0."""
  n = dzv.numel()
  w = (n - torch.arange(n, device=x4.device)).to(f64)
  g = dzv @ x4
  gb = U * _factor(n) * ((dzv.abs() * w) @ x4.abs())
  db = dzv.sum()
  dbb = U * _factor(n) * (dzv.abs() * w).sum()
  pre = torch.where(x4 > 0, dzv[:, None] * wd.reshape(1, -1), torch.zeros_like(x4))
  return (g, gb), (db, dbb), (pre, U * pre.abs())


def corr_dlogit(corr, gt_or, gt_ov, min_ov, Wf):
  """k_corr_dlogit of one chunk: dcorr [n, Wf]."""
  n = corr.shape[0]
  t = torch.zeros_like(corr)
  on = gt_ov > min_ov
  t[torch.arange(n, device=corr.device)[on], gt_or.long()[on]] = 1.0
  sg = torch.sigmoid(-corr)
  coef = 1 + (Wf - 1) * t
  num = (1 - t) - coef * sg
  model = num / (n * Wf)
  # expf overflows to inf past corr = 88.7, where sg < 2^-126 becomes 0; the result may be subnormal (2^-149)
  dsg = 4 * U * sg * (1 - sg) + 3 * U * sg + 2.0 ** -126
  bound = (1 + 1e-6) * ((coef * (dsg + U * sg) + 2 * U * num.abs()) / (n * Wf) + U * model.abs() + 2.0 ** -149)
  return model, bound


# ---- backward of the heads -------------------------------------------------------------------------------------
def conv_wgrad(x, dy, kshape, stride, prec, drop_slice=None, double_slice=None, no_ones=False):
  """wgrad_gemm of one chunk through ConvWgradOperand: x [n, H, W, C], dy [n, Ho, Wo, N] -> (dW [kh, kw, C, N],
  bound), (db [N], bound).  drop_slice / double_slice / no_ones plant defects for the mutation tests."""
  kh, kw = kshape
  n, Ho, Wo, N = dy.shape
  C = x.shape[3]
  Kred = n * Ho * Wo
  w, z = split_w(Kred, kh * kw * C + 1, N, prec, x.device)
  w = w.reshape(n, Ho, Wo, 1)
  z = z.reshape(n, Ho, Wo, 1)
  dyu = dy
  if drop_slice is not None:
    dyu = torch.where(z == drop_slice, torch.zeros_like(dy), dy)
  if double_slice is not None:
    dyu = torch.where(z == double_slice, 2 * dy, dyu)
  size = (N, C, kh, kw)
  dW = torch.nn.grad.conv2d_weight(_nchw(x), size, _nchw(dyu), stride=stride).permute(2, 3, 1, 0)
  bW = torch.nn.grad.conv2d_weight(_nchw(x.abs()), size, _nchw(dy.abs() * w), stride=stride).permute(2, 3, 1, 0)
  db = torch.zeros(N, dtype=f64, device=x.device) if no_ones else dyu.sum((0, 1, 2))
  bb = (dy.abs() * w).sum((0, 1, 2))
  fac = U * _factor(w.max())
  return (dW, fac * bW), (db, fac * bb)


def conv_dgrad(dy, w, in_hw, stride, prec, mask=None):
  """The input gradient (ConvDgradOperand / ConvDgradStridedOperand) of dy [n, Ho, Wo, N] through w [kh, kw, C,
  N] to an [n, H, W, C] input, K = (dh, dw, n), rows no output reads 0; masked by ``mask`` (the input > 0)."""
  kh, kw, C, N = w.shape
  n = dy.shape[0]
  wk = chain_w(kh * kw * N, prec, dy.device).reshape(kh, kw, 1, N)
  size = (n, C) + tuple(in_hw)
  dx = torch.nn.grad.conv2d_input(size, _oihw(w), _nchw(dy), stride=stride).permute(0, 2, 3, 1)
  bx = torch.nn.grad.conv2d_input(size, _oihw(w.abs() * wk), _nchw(dy.abs()), stride=stride).permute(0, 2, 3, 1)
  bx = U * _factor(wk.max()) * bx
  if mask is not None:
    dx = torch.where(mask, dx, torch.zeros_like(dx))
    bx = torch.where(mask, bx, torch.zeros_like(bx))
  return dx, bx


def do1(dx3, w2, prec):
  """c_conv2's input gradient dx3 [n, ho, jb, 128] W2^T, stored [n, ho, jb, dh, 64] (K = the 128 outputs)."""
  s = w2.shape[0]
  W = w2.reshape(s, w2.shape[2], w2.shape[3])               # [dh, c, no]
  wk = chain_w(W.shape[2], prec, dx3.device)
  model = torch.einsum('phjn,dcn->phjdc', dx3, W)
  bound = torch.einsum('phjn,dcn->phjdc', dx3.abs(), W.abs() * wk)
  return model, U * _factor(wk.max()) * bound


def _do1_rows(d, s):
  """do1 [n, nho, nb, s, 64] -> [n, Wf = nho s, nb, 64] (row i = s ho + dh)."""
  n, nho, nb, _, o = d.shape
  return d.permute(0, 1, 3, 2, 4).reshape(n, nho * s, nb, o)


def delta_wgrad(L, R, d1, s, prec):
  """wgrad_gemm through DeltaWgradOperand of one chunk: L, R [n, Wf, 128], d1 = do1 [n, nho, nb, s, 64] ->
  (dW1 [1, s, 128, 64], bound), (db1 [64], bound)."""
  n, nho, nb, _, O = d1.shape
  C = L.shape[2]
  Kred = n * nho * nb * s
  w, _ = split_w(Kred, s * C + 1, O, prec, L.device)
  w = _do1_rows(w.reshape(n, nho, nb, s, 1), s)              # [n, Wf, nb, 1]
  d = _do1_rows(d1, s)
  dW = torch.zeros(s, C, O, dtype=f64, device=L.device)
  bW = torch.zeros_like(dW)
  for p in range(n):
    D = (L[p][:nho * s, None, None, :] - R[p][:nb * s].reshape(nb, s, C)[None]).abs()   # [i, jb, dj, c]
    dW += torch.einsum('ijdc,ijo->dco', D, d[p])
    bW += torch.einsum('ijdc,ijo->dco', D, d[p].abs() * (w[p] + 1))
  db = d.sum((0, 1, 2))
  bb = (d.abs() * w).sum((0, 1, 2))
  fac = U * _factor(w.max() + 1)
  return (dW[None], fac * bW[None]), (db, fac * bb)


# ---- backward into the volumes ---------------------------------------------------------------------------------
def corr_backward(dc, L, R, half=None, shift=0):
  """k_corr_backward: dL = C0 R, dR = C1 L with C0[i, q] = dc[(i - q - half) mod Wf], C1[j, q] =
  dc[(q - j - half) mod Wf], q in order.  -> (dfv [2, n, Wf, 128], bound).  ``half`` / ``shift``: planted defects."""
  n, Wf, _ = L.shape
  half = Wf // 2 if half is None else half
  i = torch.arange(Wf, device=L.device)
  wq = (Wf - i).to(f64)
  i0 = (i[:, None] - i[None, :] - half + shift) % Wf
  i1 = (i[None, :] - i[:, None] - half + shift) % Wf
  out, bnd = [], []
  for side, (idx, X) in enumerate(((i0, R), (i1, L))):
    Cm = dc[:, idx]                                           # [n, row, q]
    out.append(Cm @ X)
    bnd.append((Cm.abs() * wq) @ X.abs())
  return torch.stack(out), U * _factor(Wf) * torch.stack(bnd)


def delta_dgrad(d1, w1, L, R, prec, sign0=0.0):
  """k_delta_dgrad(_tc) partials for do1 d1 [n, nho, nb, s, 64], w1 [1, s, 128, 64], volumes L, R [n, Wf, 128]:
  (part_l [n, nb, Wf, 128], bound), (part_r [n, nit, Wf, 128], bound).  ``sign0``: the sign a planted defect gives
  l == r."""
  n, nho, nb, s, O = d1.shape
  Wf, C = L.shape[1], L.shape[2]
  nit = _cdiv(Wf, 64)
  W = w1.reshape(s, C, O)
  wo = chain_w(O, prec, L.device)
  d = _do1_rows(d1, s)                                         # [n, Wf, nb, O]
  pl, bl, pr, br = [], [], [], []
  wdj = (s - torch.arange(s, device=L.device)).to(f64).reshape(1, 1, s, 1)
  tile = torch.div(torch.arange(Wf, device=L.device), 64, rounding_mode='floor')
  for p in range(n):
    G = torch.einsum('ijo,dco->ijdc', d[p], W)                 # [i, jb, dj, c]
    Ga = torch.einsum('ijo,dco->ijdc', d[p].abs(), W.abs())
    Gb = torch.einsum('ijo,dco->ijdc', d[p].abs(), W.abs() * wo)
    diff = L[p][:, None, None, :] - R[p][:nb * s].reshape(nb, s, C)[None]
    sg = torch.sign(diff)
    if sign0:
      sg = torch.where(diff == 0, torch.full_like(sg, sign0), sg)
    v = sg * G
    pl.append(v.sum(2).permute(1, 0, 2))                        # [jb, i, c]
    bl.append((sg.abs() * (Gb + wdj * Ga)).sum(2).permute(1, 0, 2))
    vr = torch.zeros(nit, Wf, C, dtype=f64, device=L.device)
    brr = torch.zeros_like(vr)
    vb = sg.abs() * (Gb + PART_R_ADDS * Ga)
    vr.index_add_(0, tile, -v.reshape(Wf, nb * s, C))
    brr.index_add_(0, tile, vb.reshape(Wf, nb * s, C))
    pr.append(vr)
    br.append(brr)
  fac = U * _factor(wo.max() + max(s, PART_R_ADDS))
  return (torch.stack(pl), fac * torch.stack(bl)), (torch.stack(pr), fac * torch.stack(br))


def images_order(x, offsets):
  """[2, n, ...] (LEFT, RIGHT over the pairs) -> [2n, ...] in the gathered images' order: chunk after chunk, the
  chunk's LEFT then its RIGHT."""
  out = []
  for a, b in zip(offsets[:-1], offsets[1:]):
    out += [x[0, a:b], x[1, a:b]]
  return torch.cat(out)


def volume_dy(dfv_corr, part_l, part_r, fv, offsets):
  """The top leg layer's dy: k_delta_dgrad_reduce (dfv_corr, then the partials in order) masked by the volumes
  fv [2n, Wf, 128] (images order).  -> ([2n, Wf, 128] images order, bound)."""
  nb, nit = part_l.shape[1], part_r.shape[1]
  sides = []
  for parts, k in ((part_l, nb), (part_r, nit)):
    w = (k - torch.arange(k, device=parts.device)).to(f64).reshape(1, k, 1, 1)
    sides.append((parts.sum(1), (parts.abs() * w).sum(1)))
  tot = torch.stack([dfv_corr[0] + sides[0][0], dfv_corr[1] + sides[1][0]])
  bnd = torch.stack([nb * dfv_corr[0].abs() + sides[0][1], nit * dfv_corr[1].abs() + sides[1][1]])
  tot, bnd = images_order(tot, offsets), images_order(bnd, offsets)
  mask = fv > 0
  fac = U * _factor(max(nb, nit))
  return torch.where(mask, tot, torch.zeros_like(tot)), torch.where(mask, fac * bnd, torch.zeros_like(bnd))
