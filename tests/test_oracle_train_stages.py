"""oracle/train_stages.py on the CPU at small shapes: a float32 restatement of each kernel's summation order stays
within the bound, and planted defects exceed it (the fraction of elements outside is printed)."""
import numpy as np
import pytest
import torch

from oracle import train_stages as S

f64 = torch.float64


def _f32_chain(terms):
  """fmaf chain over the first axis, float32 result after every step (terms [K, ...] exact float64 products)."""
  acc = np.zeros(terms.shape[1:], np.float32)
  for t in terms:
    acc = (acc.astype(np.float64) + t).astype(np.float32)
  return acc


def _split_gemm(A, B, kchunk):
  """k_simt_gemm split-K + k_splitk_reduce: A [K, M], B [K, N] float32 -> [M, N] float32."""
  K = A.shape[0]
  tot = np.zeros((A.shape[1], B.shape[1]), np.float32)
  for z0 in range(0, K, kchunk):
    part = _f32_chain(np.einsum('km,kn->kmn', A[z0:z0 + kchunk].astype(np.float64), B[z0:z0 + kchunk]))
    tot = (tot + part).astype(np.float32)
  return tot


def _rng(seed):
  return np.random.default_rng(seed)


def _wgrad_case(seed=0):
  rng = _rng(seed)
  x = np.maximum(rng.standard_normal((2, 7, 20, 3)), 0).astype(np.float32)
  w_shape = (3, 5)
  ho, wo = (7 - 3) // 2 + 1, 20 - 5 + 1
  dy = rng.standard_normal((2, ho, wo, 6)).astype(np.float32)
  return x, dy, w_shape, (2, 1)


def _patches(x, kshape, stride):
  kh, kw = kshape
  n, H, W, C = x.shape
  ho, wo = (H - kh) // stride[0] + 1, (W - kw) // stride[1] + 1
  cols = np.empty((n, ho, wo, kh, kw, C), np.float32)
  for dh in range(kh):
    for dw in range(kw):
      cols[:, :, :, dh, dw] = x[:, dh:dh + (ho - 1) * stride[0] + 1:stride[0], dw:dw + (wo - 1) * stride[1] + 1:stride[1]]
  return cols.reshape(n * ho * wo, kh * kw * C)


@pytest.mark.parametrize('defect', [None, 'drop_slice', 'double_slice', 'no_ones'])
def test_wgrad_split_k(defect):
  x, dy, k, stride = _wgrad_case()
  A = np.concatenate([_patches(x, k, stride), np.ones((_patches(x, k, stride).shape[0], 1), np.float32)], 1)
  Dy = dy.reshape(-1, dy.shape[-1])
  Kred = A.shape[0]
  nsplit, kchunk = S.split_plan(Kred, A.shape[1], Dy.shape[1])
  assert nsplit > 2
  G = _split_gemm(A, Dy, kchunk)
  (dW, bW), (db, bb) = S.conv_wgrad(torch.tensor(x, dtype=f64), torch.tensor(dy, dtype=f64), k, stride, 'fp32')
  gk = torch.tensor(G[:-1].reshape(dW.shape), dtype=f64)
  gb = torch.tensor(G[-1], dtype=f64)
  if defect is None:
    assert S.ratio(gk, dW, bW) <= 1 and S.ratio(gb, db, bb) <= 1
    print('wgrad: %.3f %.3f' % (S.ratio(gk, dW, bW), S.ratio(gb, db, bb)))
    return
  kw = {'drop_slice': dict(drop_slice=1), 'double_slice': dict(double_slice=1), 'no_ones': dict(no_ones=True)}[defect]
  (mW, _), (mb, _) = S.conv_wgrad(torch.tensor(x, dtype=f64), torch.tensor(dy, dtype=f64), k, stride, 'fp32', **kw)
  frac = max(S.exceeded(mW, dW, bW), S.exceeded(mb, db, bb))
  print('%s: %.1f %% of the elements outside their bound' % (defect, 100 * frac))
  assert frac > 0.3


def _dgrad_f32(dy, w, H, W, stride, defect=None):
  """ConvDgradStridedOperand's product: dx[h, w, c] = sum over (dh, dw, n) in order of dy[(h - dh)/sh, ...] w."""
  kh, kw, C, N = w.shape
  n = dy.shape[0]
  Ho, Wo = dy.shape[1], dy.shape[2]
  terms = np.zeros((kh * kw * N, n, H, W, C))
  k = 0
  for dh in range(kh):
    for dw in range(kw):
      for o in range(N):
        for hh in range(H):
          y = hh - dh
          if y < 0 or y % stride[0]:
            continue
          y //= stride[0]
          if y >= Ho:
            continue
          for ww in range(W):
            xw = ww - dw + (1 if defect == 'tap_shift' and ww == W - 1 else 0)
            if xw < 0 or xw % stride[1]:
              continue
            xw //= stride[1]
            if xw >= Wo:
              continue
            terms[k, :, hh, ww, :] = dy[:, y, xw, o:o + 1].astype(np.float64) * w[dh, dw, :, o]
        k += 1
  out = _f32_chain(terms)
  if defect == 'unread_row':
    out[:, H - 1] = out[:, H - 2]
  if defect == 'drop_last_read':
    out[:, (Ho - 1) * stride[0] + kh - 1] = 0
  return out


@pytest.mark.parametrize('defect', [None, 'unread_row', 'drop_last_read', 'tap_shift', 'mask_ge'])
def test_strided_dgrad(defect):
  rng = _rng(1)
  H, W, stride = 8, 9, (2, 1)
  w = rng.standard_normal((3, 4, 2, 3)).astype(np.float32)
  Ho, Wo = (H - 3) // 2 + 1, W - 4 + 1
  dy = rng.standard_normal((2, Ho, Wo, 3)).astype(np.float32)
  x = np.maximum(rng.standard_normal((2, H, W, 2)), 0).astype(np.float32)
  x[:, :, 0] = 0.0                                        # exact zeros of the ReLU
  mask = torch.tensor(x > 0)
  model, bound = S.conv_dgrad(torch.tensor(dy, dtype=f64), torch.tensor(w, dtype=f64), (H, W), stride, 'fp32',
                              mask=mask)
  assert (Ho - 1) * stride[0] + 3 == H - 1               # row H - 1 is read by no output
  got = _dgrad_f32(dy, w, H, W, stride, None if defect == 'mask_ge' else defect)
  keep = (x >= 0) if defect == 'mask_ge' else (x > 0)
  got = torch.tensor(np.where(keep, got, 0), dtype=f64)
  if defect is None:
    print('dgrad: %.3f' % S.ratio(got, model, bound))
    assert S.ratio(got, model, bound) <= 1
    return
  frac = S.exceeded(got, model, bound)
  print('%s: %.1f %% of the elements outside their bound' % (defect, 100 * frac))
  assert frac > 0


@pytest.mark.parametrize('defect', [None, 'shift', 'half_up'])
def test_corr_backward(defect):
  rng = _rng(2)
  n, Wf, C = 2, 9, 128
  L = torch.tensor(np.abs(rng.standard_normal((n, Wf, C))).astype(np.float32), dtype=f64)
  R = torch.tensor(np.abs(rng.standard_normal((n, Wf, C))).astype(np.float32), dtype=f64)
  dc = torch.tensor(rng.standard_normal((n, Wf)).astype(np.float32), dtype=f64)
  model, bound = S.corr_backward(dc, L, R)
  half = Wf // 2
  out = np.zeros((2, n, Wf, C), np.float32)
  for p in range(n):
    for side in range(2):
      X = (R if side == 0 else L)[p].numpy()
      for r in range(Wf):
        h = half + 1 if defect == 'half_up' else half
        sh = 1 if defect == 'shift' else 0
        idx = [((r - q - h + sh) if side == 0 else (q - r - h + sh)) % Wf for q in range(Wf)]
        out[side, p, r] = _f32_chain(dc[p].numpy()[idx][:, None] * X.astype(np.float64))
  got = torch.tensor(out, dtype=f64)
  if defect is None:
    print('corr backward: %.3f' % S.ratio(got, model, bound))
    assert S.ratio(got, model, bound) <= 1
    return
  frac = S.exceeded(got, model, bound)
  print('%s: %.1f %% of the elements outside their bound' % (defect, 100 * frac))
  assert frac > 0.5


@pytest.mark.parametrize('defect', [None, 'sign0'])
def test_delta_dgrad_partials(defect):
  rng = _rng(3)
  n, s, Wf, C, O = 1, 3, 12, 128, 64
  nb = Wf // s
  L = np.abs(rng.standard_normal((n, Wf, C))).astype(np.float32)
  R = L.copy()                                            # LEFT == RIGHT: every sign of the diagonal taps is 0
  R[:, 1::2] = np.abs(rng.standard_normal((n, Wf // 2, C)))
  d1 = rng.standard_normal((n, Wf // s, nb, s, O)).astype(np.float32)
  w1 = rng.standard_normal((1, s, C, O)).astype(np.float32)
  t = lambda a: torch.tensor(a, dtype=f64)
  (pl, bl), _ = S.delta_dgrad(t(d1), t(w1), t(L), t(R), 'fp32')
  d = d1.transpose(0, 1, 3, 2, 4).reshape(n, Wf, nb, O)
  out = np.zeros((n, nb, Wf, C), np.float32)
  for jb in range(nb):
    acc = np.zeros((Wf, C), np.float32)
    for dj in range(s):
      G = _f32_chain(np.einsum('io,co->oic', d[0, :, jb].astype(np.float64), w1[0, dj].astype(np.float64)))
      diff = L[0] - R[0, s * jb + dj][None]
      sg = np.sign(diff)
      if defect == 'sign0':
        sg = np.where(diff == 0, 1.0, sg)
      acc = (acc + sg * G).astype(np.float32)
    out[0, jb] = acc
  got = t(out)
  if defect is None:
    print('delta dgrad part_l: %.3f' % S.ratio(got, pl, bl))
    assert S.ratio(got, pl, bl) <= 1
    return
  frac = S.exceeded(got, pl, bl)
  print('sign(0) = +1: %.1f %% of the elements outside their bound' % (100 * frac))
  assert frac > 0.05


@pytest.mark.parametrize('defect', [None, 'swap'])
def test_volume_dy_in_chunk_order(defect):
  """LEFT and RIGHT swapped in one chunk of a chunked batch."""
  rng = _rng(4)
  off = [0, 2, 2, 5]
  n, Wf, C, nb, nit = 5, 8, 4, 3, 1
  t = lambda a: torch.tensor(np.asarray(a, np.float32), dtype=f64)
  dfc = t(rng.standard_normal((2, n, Wf, C)))
  pl, pr = t(rng.standard_normal((n, nb, Wf, C))), t(rng.standard_normal((n, nit, Wf, C)))
  fv = t(np.abs(rng.standard_normal((2 * n, Wf, C))))
  model, bound = S.volume_dy(dfc, pl, pr, fv, off)
  sides = [dfc[0].numpy().astype(np.float32), dfc[1].numpy().astype(np.float32)]
  for z in range(nb):
    sides[0] = (sides[0] + pl[:, z].numpy()).astype(np.float32)
  for z in range(nit):
    sides[1] = (sides[1] + pr[:, z].numpy()).astype(np.float32)
  chunks = []
  for c, (a, b) in enumerate(zip(off[:-1], off[1:])):
    first, second = (1, 0) if (defect == 'swap' and c == 2) else (0, 1)
    chunks += [sides[first][a:b], sides[second][a:b]]
  got = t(np.where(fv.numpy() > 0, np.concatenate(chunks), 0))
  if defect is None:
    assert S.ratio(got, model, bound) <= 1
    return
  frac = S.exceeded(got, model, bound)
  print('LEFT / RIGHT swapped in chunk 2: %.1f %% of the elements outside their bound' % (100 * frac))
  assert frac > 0.3


@pytest.mark.parametrize('gap', [0.05, 0.5, 0.8, 0.9, 0.95])
def test_dz_is_within_two_ulp_and_the_float32_form_is_not(gap):
  """k_train_loss's dz (double, rounded once) against the exact derivative, and the float32 expression the kernel
  had before, which cancels in 1 - sigmoid(u)."""
  yhat = np.float32(0.97)
  y = np.float32(yhat - gap)
  model, bound = S.dz(torch.tensor([float(yhat)], dtype=f64), torch.tensor([float(y)], dtype=f64))
  d = float(yhat) - float(y)
  u = (abs(d) + 0.25) * 24 - 12
  e = np.exp(-u)
  now = np.float32(120.0 * e / (1 + e) ** 2 * np.sign(d) * float(yhat) * (1 - float(yhat)))
  assert S.ratio(torch.tensor([float(now)], dtype=f64), model, bound) <= 1
  f = np.float32
  uf = (f(abs(f(yhat - y))) + f(0.25)) * f(24) - f(12)
  sg = f(1) / (f(1) + np.exp(-uf))
  old = f(5) * sg * (f(1) - sg) * f(24) * f(np.sign(d)) / f(1) * (yhat * (f(1) - yhat))
  r_old = S.ratio(torch.tensor([float(old)], dtype=f64), model, bound)
  print('|yhat - y| = %.2f: float32 form %.1f x its bound' % (gap, r_old))
  if gap >= 0.8:
    assert r_old > 1


def test_tf32x3_split_k_stays_within_the_bound():
  """k_tc_gemm's per-K16-tile arithmetic (tests/test_train_tf32x3.py's restatement) on a wgrad with slices."""
  from test_train_tf32x3 import gemm_3xtf32
  x, dy, k, stride = _wgrad_case(5)
  P = _patches(x, k, stride)
  A = np.concatenate([P, np.ones((P.shape[0], 1), np.float32)], 1)
  Dy = dy.reshape(-1, dy.shape[-1])
  nsplit, kchunk = S.split_plan(A.shape[0], A.shape[1], Dy.shape[1])
  tot = np.zeros((A.shape[1], Dy.shape[1]), np.float32)
  for z0 in range(0, A.shape[0], kchunk):
    a, b = A[z0:z0 + kchunk], Dy[z0:z0 + kchunk]
    pad = (-a.shape[0]) % 16
    a = np.concatenate([a, np.zeros((pad, a.shape[1]), np.float32)])
    b = np.concatenate([b, np.zeros((pad, b.shape[1]), np.float32)])
    tot = (tot + gemm_3xtf32(a.T.copy(), b)).astype(np.float32)
  (dW, bW), (db, bb) = S.conv_wgrad(torch.tensor(x, dtype=f64), torch.tensor(dy, dtype=f64), k, stride, 'tf32x3')
  r = max(S.ratio(torch.tensor(tot[:-1].reshape(dW.shape), dtype=f64), dW, bW),
          S.ratio(torch.tensor(tot[-1], dtype=f64), db, bb))
  print('tf32x3 wgrad: %.3f' % r)
  assert r <= 1
