"""Every layer of the tensor-core leg against the float64 layer model (oracle/tc_leg.py), each from the GPU's own
input to that layer.

Engine.leg_stage runs the leg's own launches up to a layer and returns that layer's hi / lo planes.  For each case
every layer is compared with the model of that layer applied to the planes the GPU produced for the layer before
(the input image for s_conv1; the fp32 volume of Engine.leg for the last layer): |hi + lo - model| / bound <= 1 per
element, plus the exact relations the planes satisfy whatever their value (oracle.tc_leg.check_planes).  The cases
cover both layer-1 kernels and both channel paths, the K-sliced single-scan path (the slice counts follow the
device's SM count and are restated here) and the one-slice batched path, a lone last pixel, every layer-1 stride,
s_conv3a on and off, and activations at both ends of fp16's range.  `pytest -s` prints, per case and layer, the
slice count, the largest error / bound and the number of elements within the bound of the ReLU kink."""
import numpy as np
import pytest
import torch

from oracle import network as N
from oracle import tc_leg as T
from overlapnet_b200 import synth
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
USE = {4: {}, 5: {'use_intensity': True}, 25: {'use_intensity': True, 'use_class_probabilities': True}}
# image sizes that reduce to 1 x 360 (tests/test_geometry.py), by (s_conv3a, layer-1 strides)
SIZES = {(True, 2, 2): (64, 900), (True, 1, 1): (32, 457), (True, 1, 2): (32, 900), (True, 2, 1): (64, 457),
         (False, 2, 2): (32, 878)}


def size(model):
  return SIZES[(bool(model['additional_unsymmetric_layer3a']),) + tuple(model['strides_layer1'])]


def sm_count():
  return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def engine(model, C, n, w):
  H, W = size(model)
  eng = Engine(use=USE[C], model=model, precision='f16_tc', max_batch_scans=n, max_batch_pairs=1, proj_H=H, proj_W=W)
  assert eng.C == C
  eng.load_weights(w)
  return eng


def stages(eng, xt, n_layers):
  """[(hi, lo)] of layers 0 .. n_layers - 2 as float64 numpy, and the fp32 volume [n, 1, 360, 128]."""
  out = []
  for l in range(n_layers - 1):
    hi, lo = eng.leg_stage(xt, l)
    out.append((hi.cpu().numpy().astype(np.float64), lo.cpu().numpy().astype(np.float64)))
  fv = eng.leg(xt)
  eng.check()
  return out, fv.cpu().numpy().astype(np.float64)[:, None]


def check_case(label, model, C, x, w, scans=None):
  """Runs the scans x (n, H, W, C) in one call and checks every layer of the scans listed (default: all)."""
  n = len(x)
  H, W = size(model)
  specs = T.layer_specs(C, model, H, W)
  assert specs[-1]['h_out'] == 1 and specs[-1]['w_out'] == 360
  if n > 2 and model['additional_unsymmetric_layer3a']:
    assert specs[0]['w_out'] % 2 == 1                  # k_leg_layer1_direct's lone last pixel (even width without s_conv3a)
  splits = [1] + [T.leg_split(s, n, sm_count()) for s in specs[1:]]
  eng = engine(model, C, n, w)
  st, fv = stages(eng, torch.from_numpy(x).to(eng.device), len(specs))
  eng.close()
  ratios, kinks = np.zeros(len(specs)), np.zeros(len(specs), int)
  for i in (range(n) if scans is None else scans):
    for l, spec in enumerate(specs):
      k, b = w[spec['name']]
      last = l == len(specs) - 1
      if l == 0:
        m, tol, kink = T.layer1(x[i], k, b, spec)
      else:
        m, tol, kink = T.mma_layer(st[l - 1][0][i], st[l - 1][1][i], k, b, spec, splits[l], last)
      if last:
        got = fv[i]
        assert (got >= 0).all() and np.isfinite(got).all(), (label, i)
      else:
        hi, lo = st[l][0][i], st[l][1][i]
        assert T.check_planes(hi, lo) == [], (label, i, spec['name'], T.check_planes(hi, lo))
        got = hi + lo
      assert got.shape == m.shape, (label, spec['name'], got.shape, m.shape)
      ratios[l] = max(ratios[l], float((np.abs(got - m) / tol).max()))
      kinks[l] += kink
  print('\n[leg stages] %s (%d SMs): layer slices error/bound kink' % (label, sm_count()))
  for l, spec in enumerate(specs):
    print('[leg stages]   %-9s %3d %.3f %d' % (spec['name'], splits[l], ratios[l], kinks[l]))
  bad = [(specs[l]['name'], float(ratios[l])) for l in range(len(specs)) if not ratios[l] <= 1.0]
  assert not bad, (label, bad)
  return ratios


def scaled(w, names, factor, biases_of=()):
  """w with the kernels and biases of `names`, and the biases of `biases_of`, times a power of two (exact)."""
  f = np.float32(factor)
  out = dict(w)
  for name in names:
    out[name] = (w[name][0] * f, w[name][1] * f)
  for name in biases_of:
    out[name] = (out[name][0], out[name][1] * f)
  return out


@pytest.mark.parametrize('n', [1, 2, 3, 5])
def test_every_layer_within_its_bound(n):
  """n = 1, 2: k_leg_layer1_small and the K-sliced layers; n = 3, 5: k_leg_layer1_direct and one slice."""
  w = N.glorot_weights(4, MODEL, seed=0)
  x = synth.range_like_images(1234, n, 4)
  check_case('C=4 s_conv3a n=%d' % n, MODEL, 4, x, w, None if n <= 3 else (0, n - 1))


@pytest.mark.parametrize('C', [5, 25])
@pytest.mark.parametrize('n', [1, 3])
def test_generic_channel_path(C, n):
  w = N.glorot_weights(C, MODEL, seed=2)
  x = synth.range_like_images(7, n, C)
  check_case('C=%d s_conv3a n=%d' % (C, n), MODEL, C, x, w, (0, n - 1))


@pytest.mark.parametrize('n', [1, 3])
def test_without_s_conv3a(n):
  model = dict(MODEL, additional_unsymmetric_layer3a=False)
  w = N.glorot_weights(4, model, seed=4)
  H, W = size(model)
  x = synth.range_like_images(21, n, 4, H=H, W=W)
  check_case('C=4 no s_conv3a n=%d' % n, model, 4, x, w, (0, n - 1))


@pytest.mark.parametrize('strides', [[1, 1], [1, 2], [2, 1]])
@pytest.mark.parametrize('n', [1, 5])
def test_layer1_strides(strides, n):
  model = dict(MODEL, strides_layer1=strides)
  H, W = size(model)
  w = N.glorot_weights(4, model, seed=6)
  x = synth.range_like_images(31 + strides[0] + 2 * strides[1], n, 4, H=H, W=W)
  check_case('C=4 strides %s n=%d' % (strides, n), model, 4, x, w, (0, n - 1))


@pytest.mark.parametrize('log2_scale', [-12, 6])
@pytest.mark.parametrize('n', [1, 3])
def test_fp16_range_edges(log2_scale, n):
  """s_conv1's kernel and every bias of the leg times 2^-12 or 2^6: the leg is positively homogeneous in them, so
  every layer's activations are scaled by that power of two exactly.  At 2^-12 every lo plane and part of every hi
  plane is subnormal in fp16; the per-layer bounds hold all the same."""
  w0 = N.glorot_weights(4, MODEL, seed=0)
  leg = [s['name'] for s in T.layer_specs(4, MODEL)]
  w = scaled(w0, ['s_conv1'], 2.0 ** log2_scale, biases_of=leg[1:])
  x = synth.range_like_images(1234, n, 4)
  check_case('C=4 scale 2^%d n=%d' % (log2_scale, n), MODEL, 4, x, w, (0, n - 1))


def test_bits_do_not_depend_on_kernel_choice_position_or_call():
  """Statements that hold bit for bit: s_conv1 of a scan from k_leg_layer1_small (alone) and from
  k_leg_layer1_direct (inside a batch of 3): both are the same fmaf chain over (dh, dw, c) from the bias; every
  layer of a scan at any position of a batch of 3 and of 5; leg_stage twice; and Engine.leg after leg_stage on a
  handle against Engine.leg on a fresh one."""
  w = N.glorot_weights(4, MODEL, seed=0)
  x = synth.range_like_images(77, 5, 4)
  n_layers = len(T.layer_specs(4, MODEL))
  e1, e3, e5 = (engine(MODEL, 4, n, w) for n in (1, 3, 5))
  xt = torch.from_numpy(x).to(e1.device)

  def bits(t):
    return t.half().view(torch.int16)

  hi1, lo1 = e1.leg_stage(xt[2:3], 0)
  hi3, lo3 = e3.leg_stage(xt[:3], 0)
  assert torch.equal(bits(hi1[0]), bits(hi3[2])) and torch.equal(bits(lo1[0]), bits(lo3[2]))
  for l in range(n_layers - 1):
    a = e3.leg_stage(xt[[0, 1, 2]], l)
    b = e3.leg_stage(xt[[2, 0, 1]], l)
    c = e5.leg_stage(xt[[4, 3, 2, 1, 0]], l)
    again = e3.leg_stage(xt[[0, 1, 2]], l)
    for k in range(2):
      assert torch.equal(bits(a[k]), bits(again[k])), l
      assert torch.equal(bits(a[k][[2, 0, 1]]), bits(b[k])), l
      assert torch.equal(bits(a[k]), bits(c[k][[4, 3, 2]])), l
  fresh = engine(MODEL, 4, 3, w)
  assert torch.equal(e3.leg(xt[:3]).view(torch.int32), fresh.leg(xt[:3]).view(torch.int32))
  e1.leg_stage(xt[:1], 3)
  fresh1 = engine(MODEL, 4, 1, w)
  assert torch.equal(e1.leg(xt[:1]).view(torch.int32), fresh1.leg(xt[:1]).view(torch.int32))
  for e in (e1, e3, e5, fresh, fresh1):
    e.check()
    e.close()


def test_leg_stage_launches_the_leg_and_refuses_bad_arguments():
  """A plain Engine.leg launches what it did before leg_stage existed (one layer-1 kernel and one k_leg_mma per
  layer, plus a reduce per K-sliced layer); leg_stage of layer l launches the first l + 1 layers of that sequence
  and one copy kernel."""
  w = N.glorot_weights(4, MODEL, seed=0)
  specs = T.layer_specs(4, MODEL)
  x = torch.from_numpy(synth.range_like_images(5, 3, 4))
  for n in (1, 3):
    eng = engine(MODEL, 4, 3, w)
    xt = x[:n].to(eng.device)
    per_layer = [1] + [2 if T.leg_split(s, n, sm_count()) > 1 else 1 for s in specs[1:]]
    c0 = eng.launch_count()
    eng.leg(xt)
    assert eng.launch_count() - c0 == sum(per_layer)
    for l in (0, 4, len(specs) - 2):
      c0 = eng.launch_count()
      eng.leg_stage(xt, l)
      assert eng.launch_count() - c0 == sum(per_layer[:l + 1]) + 1
    eng.close()
  eng = engine(MODEL, 4, 2, w)
  xt = x.to(eng.device)
  for layer in (-1, len(specs) - 1):
    with pytest.raises(Exception, match='OVN_ERR_INVALID_ARG.*layer'):
      eng.leg_stage(xt[:1], layer)
  with pytest.raises(Exception, match='OVN_ERR_INVALID_ARG.*max_batch_scans'):
    eng.leg_stage(xt, 0)
  eng.close()
  eng = Engine(model=MODEL, precision='fp32', max_batch_scans=1, max_batch_pairs=1)
  eng.load_weights(w)
  with pytest.raises(Exception, match='OVN_ERR_BAD_CONFIG.*f16_tc'):
    eng.leg_stage(xt[:1], 0)
  eng.close()
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=1)
  with pytest.raises(Exception, match='OVN_ERR_WEIGHTS'):
    eng.leg_stage(xt[:1], 0)
  eng.close()
