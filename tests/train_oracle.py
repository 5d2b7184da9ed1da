"""float64 oracle of overlap-head training (test infrastructure, imported by the training tests only).

The overlap head of ``oracle/network.delta_head`` restated layer for layer with the head weights as
float64 torch leaf tensors, the two losses of the reference's training.py (:71-92, :255-257) and Keras
2.1.5's Adagrad.  Gradients come from ``torch.autograd``; nothing is derived by hand.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import network as N

HEAD = ('c_conv1', 'c_conv2', 'c_conv3', 'overlap_output')
LOSS_WEIGHTS = (5.0, 1.0)        # training.py:257 overlap_output, orientation_output


def leaf_weights(weights):
  return {n: tuple(torch.tensor(np.asarray(a), dtype=torch.float64, requires_grad=True) for a in weights[n])
          for n in HEAD}


def overlap_forward(l_fv, r_fv, lw, model_cfg=None):
  """oracle/network.delta_head on (B, 360, 128) volumes with leaf weights -> overlap (B,) float64 tensor."""
  l = torch.as_tensor(np.asarray(l_fv), dtype=torch.float64)
  r = torch.as_tensor(np.asarray(r_fv), dtype=torch.float64)
  B, W, C = l.shape
  x = N.delta_layer(l.reshape(B, 1, W, C), r.reshape(B, 1, W, C)).permute(0, 3, 1, 2)
  for name, _, stride, _, act in N.head_layers(model_cfg):
    k, b = lw[name]
    x = F.conv2d(x, k.permute(3, 2, 0, 1), b, stride=stride)
    if act == 'relu':
      x = torch.relu(x)
  flat = x.permute(0, 2, 3, 1).reshape(B, -1)                   # Flatten over (H, W, C)
  kd, bd = lw['overlap_output']
  return torch.sigmoid(flat @ kd + bd)[:, 0]


def sigmoid_loss(y_pred, y_true):
  """my_sigmoid_loss (training.py:71-83) per pair."""
  diff = (y_pred - y_true).abs()
  return torch.sigmoid((diff + 0.25) * 24 - 12)


def weighted_ce(targets, logits, pos_weight):
  """tf.nn.weighted_cross_entropy_with_logits, its numerically stable form."""
  t = np.asarray(targets, np.float64)
  x = np.asarray(logits, np.float64)
  return (1 - t) * x + (1 + (pos_weight - 1) * t) * (np.log1p(np.exp(-np.abs(x))) + np.maximum(-x, 0))


def orientation_targets(gt_overlap, gt_orientation, width, min_overlap_for_angle=0.7):
  """ImagePairOverlapOrientationSequence.py:118-121 followed by my_entropy's K.greater (training.py:90)."""
  y = np.zeros((len(gt_overlap), width))
  y[np.arange(len(gt_overlap)), np.asarray(gt_orientation, int)] = np.asarray(gt_overlap, np.float32)
  return (y > np.float32(min_overlap_for_angle)).astype(np.float64)


def losses_and_gradients(l_fv, r_fv, weights, gt_overlap, gt_orientation, min_overlap_for_angle=0.7,
                         model_cfg=None, chunk=2):
  """Losses (total, overlap, orientation) and {layer: (dL/dkernel, dL/dbias)} for one batch, float64.
  The batch is pushed through autograd ``chunk`` pairs at a time (the delta tensor is 132 MB per pair)."""
  l_fv = np.asarray(l_fv, np.float32).reshape(len(gt_overlap), -1, 128)
  r_fv = np.asarray(r_fv, np.float32).reshape(len(gt_overlap), -1, 128)
  B, W = l_fv.shape[0], l_fv.shape[1]
  y = torch.as_tensor(np.asarray(gt_overlap, np.float32), dtype=torch.float64)
  lw = leaf_weights(weights)
  l_ov = 0.0
  for s in range(0, B, chunk):
    per_pair = sigmoid_loss(overlap_forward(l_fv[s:s + chunk], r_fv[s:s + chunk], lw, model_cfg), y[s:s + chunk])
    (LOSS_WEIGHTS[0] * per_pair.sum() / B).backward()
    l_ov += float(per_pair.detach().sum())
  l_ov /= B
  corr = N.correlation_head(l_fv[:, None], r_fv[:, None])
  t = orientation_targets(gt_overlap, gt_orientation, W, min_overlap_for_angle)
  l_or = float(np.mean(np.mean(weighted_ce(t, corr, W), axis=1)))
  grads = {n: (lw[n][0].grad.numpy(), lw[n][1].grad.numpy()) for n in HEAD}
  return (LOSS_WEIGHTS[0] * l_ov + LOSS_WEIGHTS[1] * l_or, l_ov, l_or), grads


def adagrad_step(weights, grads, accum, lr, eps=1e-7):
  """Keras 2.1.5 Adagrad on the head layers: a += g^2; w -= lr g / (sqrt(a) + eps).  In place, float64."""
  for n in HEAD:
    ws, accs = [], []
    for w, g, a in zip(weights[n], grads[n], accum.setdefault(n, [0.0, 0.0])):
      a = a + np.asarray(g, np.float64) ** 2
      ws.append(np.asarray(w, np.float64) - lr * np.asarray(g, np.float64) / (np.sqrt(a) + eps))
      accs.append(a)
    weights[n] = tuple(ws)
    accum[n] = accs
  return weights
