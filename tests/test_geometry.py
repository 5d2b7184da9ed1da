"""The oracles and the host-side yaw arithmetic at image and head geometries other than the default
64 x 900 image, strides [2, 2], leg_output_width (Wf) 360 and conv1size (s) 15.  Every geometry test on
the GPU (tests/test_gpu_geometry.py) compares against these oracles, so they are pinned here first:
the overlap head against its loop restatement at s = 12 and s = 27, the correlation head at an odd
width, the circular padding at odd widths, and the argmax inversion of the evaluation flow."""
import numpy as np
import pytest
import torch

from oracle import network as N
from overlapnet_b200 import evaluate
from overlapnet_b200 import weights as Wt

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}

# (Wf, s) of the head geometries tested on the GPU: s = 12 and 24 change the tap count and the number of
# column blocks (nb = Wf / s), 225 is odd and not a multiple of 8 or 64, 405 is wider than a 384-thread block
HEAD_GEOMETRIES = [(360, 12), (360, 24), (225, 15), (405, 27)]


def head_model(wf, s, **extra):
  return dict(MODEL, leg_output_width=wf, conv1NetworkHead_conv1size=s, **extra)


def image_size(model, wf):
  """(H, W) of the images the leg reduces to 1 x wf: 64 rows and W = 2 wf + 180 with strides [2, 2] and
  s_conv3a, 32 rows and W = 2 wf + 158 without s_conv3a, W = wf + 97 with width stride 1, 32 rows with
  height stride 1."""
  sh, sw = model.get('strides_layer1', (2, 2))
  use3a = model.get('additional_unsymmetric_layer3a', False)
  H = 64 if (sh == 2 and use3a) else 32
  if sw == 2:
    W = 2 * wf + (180 if use3a else 158)
  else:
    W = wf + 97 if use3a else wf + 86
  return H, W


def leg_output(model, H, W):
  """(h, w, c) of the leg's output by the layer table of overlapnet_b200.weights."""
  h, w = H, W
  c = 4
  for name, kh, kw, sh, sw, cout, opt in Wt.LEG_TABLE:
    if opt and not model.get('additional_unsymmetric_layer3a', False):
      continue
    if sh is None:
      sh, sw = model.get('strides_layer1', (2, 2))
    h, w, c = (h - kh) // sh + 1, (w - kw) // sw + 1, cout
  return h, w, c


@pytest.mark.parametrize('model,wf,want', [
    (MODEL, 360, (64, 900)), (MODEL, 225, (64, 630)), (MODEL, 405, (64, 990)),
    (dict(MODEL, additional_unsymmetric_layer3a=False), 360, (32, 878)),
    (dict(MODEL, strides_layer1=[1, 1]), 360, (32, 457)),
    (dict(MODEL, strides_layer1=[1, 2]), 360, (32, 900)),
    (dict(MODEL, strides_layer1=[2, 1]), 360, (64, 457))])
def test_image_sizes_reduce_to_the_feature_width(model, wf, want):
  assert image_size(model, wf) == want
  assert leg_output(model, *want) == (1, wf, 128)
  shapes = Wt.layer_shapes(4, dict(model, leg_output_width=wf), *want)
  n = wf // 15
  assert shapes['overlap_output'][0] == ((n - 2) * (n - 2) * 256, 1)
  # the oracle's Glorot weights have the same shapes at that width
  w = N.glorot_weights(4, model, seed=0, leg_out_width=wf)
  assert {k: (v[0].shape, v[1].shape) for k, v in w.items()} == shapes


@pytest.mark.parametrize('wf,s', [(36, 12), (81, 27), (45, 15)])
def test_delta_head_against_naive_at_other_tap_counts(wf, s):
  """c_conv1 (1 x s, stride s), c_conv2 (s x 1, stride s), c_conv3 and Dense of the library-op oracle
  against the loop restatement, at tap counts other than 15 and an odd width."""
  rng = np.random.default_rng(wf + s)
  model = head_model(wf, s)
  w = N.glorot_weights(4, model, seed=4, leg_out_width=wf)
  n = wf // s
  assert w['overlap_output'][0].shape == ((n - 2) * (n - 2) * 256, 1)
  L = np.abs(rng.standard_normal((2, 1, wf, 128))).astype(np.float32)
  R = np.abs(rng.standard_normal((2, 1, wf, 128))).astype(np.float32)
  acts, z, o = N.delta_head(L, R, w, model, return_all=True)
  for b in range(2):
    o1 = N.delta_conv1_naive(L[b, 0], R[b, 0], w['c_conv1'][0], w['c_conv1'][1], s)
    assert o1.shape == (wf, n, 64)
    assert np.allclose(acts[0][b], o1, atol=1e-10)
    o2 = N.conv2d_valid_naive(o1, w['c_conv2'][0], w['c_conv2'][1], (s, 1), True)
    assert o2.shape == (n, n, 128)
    assert np.allclose(acts[1][b], o2, atol=1e-10)
    o3 = N.conv2d_valid_naive(o2, w['c_conv3'][0], w['c_conv3'][1], (1, 1), True)
    zz = o3.reshape(-1) @ w['overlap_output'][0].astype(np.float64)[:, 0] + w['overlap_output'][1][0]
    assert np.allclose(z[b, 0], zz, atol=1e-10)
    assert np.allclose(o[b, 0], 1 / (1 + np.exp(-zz)), atol=1e-12)


@pytest.mark.parametrize('wf', [225, 45, 7])
def test_correlation_head_against_naive_at_odd_width(wf):
  rng = np.random.default_rng(wf)
  L = np.abs(rng.standard_normal((2, 1, wf, 16))).astype(np.float32)
  R = np.abs(rng.standard_normal((2, 1, wf, 16))).astype(np.float32)
  c = N.correlation_head(L, R)
  assert c.shape == (2, wf)
  for b in range(2):
    assert np.allclose(c[b], N.correlation_naive(L[b, 0], R[b, 0]), rtol=1e-12, atol=1e-9)
  # shift property: R = roll(L, s) => argmax = (-s - W//2) mod W, which is (W//2 - s) mod W only for even W
  for s in (0, 1, -1, wf // 2, -(wf // 2), wf // 2 + 1, 37 % wf):
    k = int(np.argmax(N.correlation_head(L[:1], np.roll(L[:1], s, axis=2))[0]))
    assert k == (-s - wf // 2) % wf


@pytest.mark.parametrize('W', [5, 7, 225])
def test_range_padding_at_odd_width(W):
  """[x[W//2:], x, x[:W//2 - 1]]: width 2W - 1 for every W (RangePadding2D.py:31-38); entry k + j + W//2 of
  the padded row is x[(k + j + W//2) mod W] for every valid window position k, which is what the
  correlation head's circular sum relies on."""
  x = torch.arange(1., W + 1.).reshape(1, 1, W, 1)
  p = N.range_padding(x, W // 2).reshape(-1).numpy()
  assert p.shape == (2 * W - 1,)
  for k in range(W):
    for j in range(W):
      assert p[k + j] == x.reshape(-1)[(k + j + W // 2) % W]
  if W == 5:
    assert p.tolist() == [3, 4, 5, 1, 2, 3, 4, 5, 1]


@pytest.mark.parametrize('wf', [360, 225, 405, 24])
def test_readout_and_argmax_inversion_at_any_width(wf):
  """Infer returns 180 - argmax whatever the width (infer.py:158, :198, :233); the evaluation flow gets the
  argmax back as 180 - yaw, which lies in [0, wf)."""
  rng = np.random.default_rng(wf)
  argmax = np.concatenate([[0, wf - 1, wf // 2], rng.integers(0, wf, 20)])
  corr = rng.uniform(0, 1, (len(argmax), wf))
  corr[np.arange(len(argmax)), argmax] = 2.0
  _, yaw = N.readout(np.zeros(len(argmax)), corr)
  assert yaw.tolist() == (180 - argmax).tolist()
  back = evaluate.yaw_to_argmax(yaw)
  assert back.tolist() == argmax.tolist()
  assert back.min() >= 0 and back.max() < wf


def test_error_statistics_at_feature_width_225():
  """The circular yaw-bin error of testing.py:274-323 wraps at the network's output width."""
  wf = 225
  gt_ov = np.array([0.9, 0.8, 0.95, 0.5, 0.71])
  gt_or = np.array([0, 224, 100, 10, 3], float)
  model_argmax = evaluate.yaw_to_argmax(np.array([180 - 224, 180 - 1, 180 - 103, 180 - 150, 180 - 3]))
  assert model_argmax.tolist() == [224, 1, 103, 150, 3]
  model_ov = np.array([0.85, 0.8, 0.9, 0.1, 0.7])
  st = evaluate.error_statistics(model_ov, model_argmax, gt_ov, gt_or, wf)
  d_ov = np.abs(model_ov - gt_ov)
  assert st['overlap_mean'] == pytest.approx(d_ov.mean()) and st['overlap_max'] == pytest.approx(d_ov.max())
  d_yaw = np.array([1, 2, 3, 0])           # 0 vs 224 and 224 vs 1 wrap at 225; pair 3 has overlap <= 0.7
  assert st['yaw_pairs'] == 4
  assert st['yaw_mean'] == pytest.approx(d_yaw.mean()) and st['yaw_max'] == 3
  assert st['yaw_rms'] == pytest.approx(np.sqrt((d_yaw ** 2).mean()))
  # at 360 the same bins do not wrap
  st360 = evaluate.error_statistics(model_ov, model_argmax, gt_ov, gt_or, 360)
  assert st360['yaw_max'] == 137
