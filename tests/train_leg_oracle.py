"""float64 oracle of whole-network training (test infrastructure, imported by the training tests only).

The network of ``oracle/network`` -- the leg (``leg_layers``), the |l - r| overlap head (``delta_layer``,
``head_layers``) and the correlation head (``range_padding``, restated here in torch because
``N.correlation_head`` returns NumPy) -- with every layer's kernel and bias a float64 torch leaf tensor, the
losses of the reference's training.py (:71-92, :255-257) and Keras 2.1.5's Adagrad.  Gradients come from
``torch.autograd``; nothing is derived by hand.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import network as N
import train_oracle as T


def layer_names(model_cfg=None):
  return tuple(n for n, *_ in N.leg_layers(model_cfg)) + T.HEAD


def leaf_weights(weights, model_cfg=None):
  return {n: tuple(torch.tensor(np.asarray(a), dtype=torch.float64, requires_grad=True) for a in weights[n])
          for n in layer_names(model_cfg)}


def leg(x_nhwc, lw, model_cfg=None):
  """The leg on (n, H, W, C) images -> feature volumes (n, Wf, 128), float64, differentiable in lw."""
  x = torch.as_tensor(np.asarray(x_nhwc), dtype=torch.float64).permute(0, 3, 1, 2)
  for name, _, stride, _ in N.leg_layers(model_cfg):
    k, b = lw[name]
    x = torch.relu(F.conv2d(x, k.permute(3, 2, 0, 1).contiguous(), b, stride=stride))
  return x.permute(0, 2, 3, 1)[:, 0]


def overlap_head(l, r, lw, model_cfg=None):
  """oracle/network.delta_head on (B, Wf, 128) tensors -> overlap (B,)."""
  B, W, C = l.shape
  x = N.delta_layer(l.reshape(B, 1, W, C), r.reshape(B, 1, W, C)).permute(0, 3, 1, 2)
  for name, _, stride, _, act in N.head_layers(model_cfg):
    k, b = lw[name]
    x = F.conv2d(x, k.permute(3, 2, 0, 1).contiguous(), b, stride=stride)
    if act == 'relu':
      x = torch.relu(x)
  flat = x.permute(0, 2, 3, 1).reshape(B, -1)
  kd, bd = lw['overlap_output']
  return torch.sigmoid(flat @ kd + bd)[:, 0]


def correlation_head(l, r):
  """oracle/network.correlation_head on (B, Wf, 128) tensors, differentiable: corr (B, Wf)."""
  B, W, C = l.shape
  pad = N.range_padding(l.reshape(B, 1, W, C), W // 2)
  out = []
  for b in range(B):
    disp = pad[b:b + 1].permute(0, 3, 1, 2).contiguous()                # (1, C, 1, 2W-1)
    ker = r[b].reshape(1, W, C).permute(2, 0, 1)[None].contiguous()      # (1, C, 1, W)
    out.append(F.conv2d(disp, ker).reshape(-1))
  return torch.stack(out)


def weighted_ce(t, x, pos_weight):
  """tf.nn.weighted_cross_entropy_with_logits (stable form) on tensors."""
  return (1 - t) * x + (1 + (pos_weight - 1) * t) * (torch.log1p(torch.exp(-x.abs())) + torch.relu(-x))


def losses_and_gradients(left_imgs, right_imgs, weights, gt_overlap, gt_orientation, min_overlap_for_angle=0.7,
                         model_cfg=None, fv=None, chunk=2):
  """Losses (total, overlap, orientation), {layer: (dL/dkernel, dL/dbias)} for every layer and dL/d(volumes)
  [2, B, Wf, 128] for one batch, float64.

  ``fv`` (optional, [2B, Wf, 128]): the volumes at which the heads are evaluated, LEFT then RIGHT, standing in
  for the leg's float64 output in the forward while the gradient still flows through the leg.  The sign of
  l - r is discontinuous, so a test that compares against a float32 device passes the device's own volumes:
  then both sides take the same signs and the same head ReLU masks.

  The heads are pushed through autograd ``chunk`` pairs at a time (the delta tensor is 132 MB per pair) with
  the volumes as leaves; their gradient is then pushed through the leg in one backward call."""
  B = len(gt_overlap)
  lw = leaf_weights(weights, model_cfg)
  vol = leg(np.concatenate([np.asarray(left_imgs), np.asarray(right_imgs)]), lw, model_cfg)
  if fv is not None:          # exactly fv in the forward (a - a is exactly 0), the leg's gradient in the backward
    vol = torch.as_tensor(np.asarray(fv), dtype=torch.float64).reshape(vol.shape) + (vol - vol.detach())
  v = vol.detach().requires_grad_(True)
  W = v.shape[1]
  y = torch.as_tensor(np.asarray(gt_overlap, np.float32), dtype=torch.float64)
  t = torch.as_tensor(T.orientation_targets(gt_overlap, gt_orientation, W, min_overlap_for_angle))
  l_ov = l_or = 0.0
  for s in range(0, B, chunk):
    e = min(B, s + chunk)
    l, r = v[s:e], v[B + s:B + e]
    ov = T.sigmoid_loss(overlap_head(l, r, lw, model_cfg), y[s:e]).sum() / B
    orr = weighted_ce(t[s:e], correlation_head(l, r), W).mean(dim=1).sum() / B
    (T.LOSS_WEIGHTS[0] * ov + T.LOSS_WEIGHTS[1] * orr).backward()
    l_ov += float(ov.detach())
    l_or += float(orr.detach())
  vol.backward(v.grad)
  grads = {n: (lw[n][0].grad.numpy(), lw[n][1].grad.numpy()) for n in lw}
  total = T.LOSS_WEIGHTS[0] * l_ov + T.LOSS_WEIGHTS[1] * l_or
  return (total, l_ov, l_or), grads, v.grad.numpy().reshape(2, B, W, -1)


def forward(left_imgs, right_imgs, weights, model_cfg=None):
  """(volumes [2B, Wf, 128], overlap [B], corr [B, Wf]) of the oracle's forward, float64 numpy."""
  lw = leaf_weights(weights, model_cfg)
  with torch.no_grad():
    vol = leg(np.concatenate([np.asarray(left_imgs), np.asarray(right_imgs)]), lw, model_cfg)
    B = len(left_imgs)
    ov = overlap_head(vol[:B], vol[B:], lw, model_cfg)
    corr = correlation_head(vol[:B], vol[B:])
  return vol.numpy(), ov.numpy(), corr.numpy()


def adagrad_step(weights, grads, accum, lr, eps=1e-7):
  """Keras 2.1.5 Adagrad on every layer in ``grads``: a += g^2; w -= lr g / (sqrt(a) + eps).  In place."""
  for n in grads:
    ws, accs = [], []
    for w, g, a in zip(weights[n], grads[n], accum.setdefault(n, [0.0, 0.0])):
      a = a + np.asarray(g, np.float64) ** 2
      ws.append(np.asarray(w, np.float64) - lr * np.asarray(g, np.float64) / (np.sqrt(a) + eps))
      accs.append(a)
    weights[n] = tuple(ws)
    accum[n] = accs
  return weights
