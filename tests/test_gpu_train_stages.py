"""Every stage of a training step on the GPU against the float64 model of oracle/train_stages.py, element by element:
each stage from the GPU's own inputs to it (read back with Engine.set_train_stop / Engine.train_stage), error /
bound <= 1, at training precisions fp32 and tf32x3.  Head-only and whole-network flows, head geometries, leg
shapes (image heights, widths, layer-1 strides, input channels), a batch whose leg launches split over images, a
chunked call, edge values (LEFT == RIGHT, |yhat - y| up to 0.95, gt orientations at bins 0 and Wf - 1), and the
handle's behaviour after a stopped call."""
import functools
import time

import numpy as np
import pytest
import torch

from oracle import network as N
from oracle import train_stages as S
from overlapnet_b200 import synth
from overlapnet_b200._cabi import OvnError
from overlapnet_b200.engine import HEAD_LAYERS, Engine
from test_geometry import image_size

pytestmark = pytest.mark.gpu

USE = {4: {}, 5: {'use_intensity': True}, 25: {'use_intensity': True, 'use_class_probabilities': True}}
MIN_OV = 0.5
WORST = {}
T0 = time.time()


def _model(wf=360, s=15, use3a=True, strides=(2, 2)):
  return {'additional_unsymmetric_layer3a': use3a, 'strides_layer1': list(strides), 'leg_output_width': wf,
          'conv1NetworkHead_conv1size': s}


def _t(a, dev):
  return torch.as_tensor(np.asarray(a)).to(device=dev, dtype=torch.float64)


def _targets(ov, rng, wf):
  """gt overlaps |yhat - y| from 0.05 to 0.95 (as far as yhat allows), orientations at bins 0 and Wf - 1 first."""
  n = len(ov)
  d = np.linspace(0.05, 0.95, n) if n > 1 else np.array([0.3])
  y = np.where(ov - d >= 0, ov - d, np.where(ov + d <= 1, ov + d, np.clip(1 - ov, 0, 1)))
  gt_or = rng.integers(0, wf, n).astype(np.int32)
  gt_or[:2] = [0, wf - 1][:min(2, n)]
  return y.astype(np.float32), gt_or


def _spread(eng, w, bank, left, right, std):
  """Dense rescaled to a logit spread ``std`` over these pairs, so that yhat reaches both ends of (0, 1)."""
  dev = eng.device
  ov, _, _ = eng.heads(bank, torch.as_tensor(left).to(dev), torch.as_tensor(right).to(dev))
  ov = ov.double().cpu().numpy().clip(1e-6, 1 - 1e-6)
  return N.spread_dense(w, np.log(ov / (1 - ov)) + float(w['overlap_output'][1][0]), target_std=std)


def _grad_views(w, names, flat):
  """The flat gradient vector (c_conv1..3, overlap_output, then the leg input to output) as {layer: (k, b)}."""
  out, o = {}, 0
  for name in names:
    k, b = w[name]
    out[name] = (flat[o:o + k.size].reshape(k.shape), flat[o + k.size:o + k.size + b.size])
    o += k.size + b.size
  return out


class Step:
  """One batch through one handle: every stop stage from its own stopped call, then one whole call."""

  def __init__(self, eng, net, rows, left, right, gt_ov, gt_or, offsets=None):
    self.eng, self.net = eng, net
    self.n = len(left)
    self.off = list(offsets) if offsets is not None else [0, self.n]
    dev = eng.device
    self.args = (rows, torch.as_tensor(left).to(dev), torch.as_tensor(right).to(dev), gt_ov, gt_or, MIN_OV)
    self.stops = {}
    for stage in ('o1', 'x4') + (('dfv_corr',) if net else ()):
      self.stops[stage] = self._stopped(stage, 0)
    if net:
      for l in range(len(eng.leg_layers)):
        self.stops[('leg_dy', l)] = self._stopped('leg_dy', l)
    self.loss, self.parts = self._call()
    self.eng.check()

  def _call(self, copy=True):
    chunked = len(self.off) > 2 or self.off != [0, self.n]
    if chunked:
      fn = self.eng.net_gradients_chunks if self.net else self.eng.head_gradients_chunks
      rows, li, ri, gov, gor, mo = self.args
      loss, parts = fn(rows, li, ri, self.off, gov, gor, mo)
      return loss, parts
    fn = self.eng.net_gradients if self.net else self.eng.head_gradients
    loss = fn(*self.args)
    return [loss], self.eng.copy_gradients(self.net)[None] if copy else None

  def _stopped(self, stage, layer):
    self.eng.set_train_stop(stage, layer)
    self._call(copy=False)
    return self.eng.train_stage(stage, layer).double()

  def stage(self, name, layer=0):
    return self.eng.train_stage(name, layer).double()


def check_step(st, w, bank, left, right, gt_ov, gt_or, prec, tag):
  """Every stage of the Step against the model; returns {stage: error / bound}."""
  eng, dev = st.eng, st.eng.device
  n, Wf = st.n, eng.Wf
  s = eng.model.get('conv1NetworkHead_conv1size', 15)
  nb, nho = Wf // s, Wf // s
  W = {k: (_t(v[0], dev), _t(v[1], dev)) for k, v in w.items()}
  res = {}

  def put(key, gpu, model_bound):
    model, bound = model_bound
    gpu = gpu.reshape(model.shape)
    r = S.ratio(gpu, model, bound)
    if not r <= 1:
      e = int(((gpu - model).abs() / bound).reshape(-1).argmax())
      print('%s %s: element %d gpu %.9g model %.9g bound %.3g, %.2f %% of the elements outside' % (
          tag, key, e, float(gpu.reshape(-1)[e]), float(model.reshape(-1)[e]), float(bound.reshape(-1)[e]),
          100 * S.exceeded(gpu, model, bound)))
    res[key] = max(res.get(key, 0.0), r)

  legs = list(eng.leg_layers)
  specs = {name: spec for name, spec in zip(legs, _leg_specs(eng))}
  if st.net:
    imgs = st.stage('images').reshape(2 * n, eng.H, eng.W, eng.C)
    acts, x = [], imgs
    for l, name in enumerate(legs):
      sp = specs[name]
      a = st.stage('act', l).reshape(2 * n, sp['h_out'], sp['w_out'], sp['cout'])
      put('leg fwd %s' % name, a, S.conv_forward(x, W[name][0], W[name][1], (sp['sh'], sp['sw']), True, prec))
      acts.append(a)
      x = a
    fv = acts[-1].reshape(2 * n, Wf, 128)
    L = torch.cat([fv[2 * a:2 * a + (b - a)] for a, b in zip(st.off[:-1], st.off[1:])])
    R = torch.cat([fv[2 * a + (b - a):2 * b] for a, b in zip(st.off[:-1], st.off[1:])])
  else:
    B = bank.double()
    L, R = B[torch.as_tensor(left).long().to(dev)], B[torch.as_tensor(right).long().to(dev)]
  o1 = st.stops['o1'].reshape(n, Wf, nb, 64)
  put('o1', o1, S.delta_forward(L, R, W['c_conv1'][0], W['c_conv1'][1], prec))
  x3 = st.stage('x3').reshape(n, nho, nb, 128)
  put('x3', x3, S.conv_forward(o1, W['c_conv2'][0], W['c_conv2'][1], (s, 1), True, prec))
  x4 = st.stops['x4'].reshape(n, nho - 2, nb - 2, 256)
  put('x4', x4, S.conv_forward(x3, W['c_conv3'][0], W['c_conv3'][1], 1, True, prec))
  ov = st.stage('overlap')
  put('overlap', ov, S.dense_forward(x4.reshape(n, -1), W['overlap_output'][0], W['overlap_output'][1]))
  put('corr', st.stage('corr').reshape(n, Wf), S.corr_forward(L, R, prec))
  dzg = st.stage('dz')
  dpre3 = st.stage('dpre3').reshape(x4.shape)
  dx3 = st.stage('dx3').reshape(x3.shape)
  do1g = st.stage('do1').reshape(n, nho, nb, s, 64)
  gy, gor = _t(gt_ov, dev), torch.as_tensor(gt_or).to(dev)
  corr = st.stage('corr').reshape(n, Wf)
  names = list(HEAD_LAYERS) + (legs if st.net else [])
  for c, (a, b) in enumerate(zip(st.off[:-1], st.off[1:])):
    if a == b:
      continue
    g = _grad_views(w, names, st.parts[c].double())
    put('dz', dzg[a:b], S.dz(ov[a:b], gy[a:b]))
    (gw, gb), (db, dbb), pre = S.dense_backward(x4[a:b].reshape(b - a, -1), dzg[a:b], W['overlap_output'][0])
    put('dense dW', g['overlap_output'][0].reshape(-1), (gw, gb))
    put('dense db', g['overlap_output'][1].reshape(()), (db, dbb))
    put('dpre3', dpre3[a:b].reshape(b - a, -1), pre)
    for name, xin, dy, k, stride in (('c_conv3', x3, dpre3, (3, 3), 1), ('c_conv2', o1, dx3, (s, 1), (s, 1))):
      dw, dbias = S.conv_wgrad(xin[a:b], dy[a:b], k, stride, prec)
      put('%s dW' % name, g[name][0], dw)
      put('%s db' % name, g[name][1], dbias)
    dw, dbias = S.delta_wgrad(L[a:b], R[a:b], do1g[a:b], s, prec)
    put('c_conv1 dW', g['c_conv1'][0], dw)
    put('c_conv1 db', g['c_conv1'][1], dbias)
    if st.net:
      put('dcorr', st.stage('dcorr').reshape(n, Wf)[a:b], S.corr_dlogit(corr[a:b], gor[a:b], gy[a:b], MIN_OV, Wf))
      for l, name in enumerate(legs):
        sp = specs[name]
        X = imgs if l == 0 else acts[l - 1]
        dy = st.stops[('leg_dy', l)].reshape(acts[l].shape)
        dw, dbias = S.conv_wgrad(X[2 * a:2 * b], dy[2 * a:2 * b], (sp['kh'], sp['kw']), (sp['sh'], sp['sw']), prec)
        put('leg dW %s' % name, g[name][0], dw)
        put('leg db %s' % name, g[name][1], dbias)
  put('dx3', dx3, S.conv_dgrad(dpre3, W['c_conv3'][0], (nho, nb), 1, prec, mask=x3 > 0))
  put('do1', do1g, S.do1(dx3, W['c_conv2'][0], prec))
  if st.net:
    dcorr = st.stage('dcorr').reshape(n, Wf)
    dfvc = st.stops['dfv_corr'].reshape(2, n, Wf, 128)
    put('dfv corr', dfvc, S.corr_backward(dcorr, L, R))
    pl_m, pr_m = S.delta_dgrad(do1g, W['c_conv1'][0], L, R, prec)
    pl = st.stage('part_l').reshape(pl_m[0].shape)
    pr = st.stage('part_r').reshape(pr_m[0].shape)
    put('part_l', pl, pl_m)
    put('part_r', pr, pr_m)
    put('dy %s' % legs[-1], st.stops[('leg_dy', len(legs) - 1)].reshape(2 * n, Wf, 128),
        S.volume_dy(dfvc, pl, pr, fv, st.off))
    for l in range(len(legs) - 1, 0, -1):
      sp = specs[legs[l]]
      dy = st.stops[('leg_dy', l)].reshape(acts[l].shape)
      put('dy %s' % legs[l - 1], st.stops[('leg_dy', l - 1)].reshape(acts[l - 1].shape),
          S.conv_dgrad(dy, W[legs[l]][0], (sp['h_in'], sp['w_in']), (sp['sh'], sp['sw']), prec, mask=acts[l - 1] > 0))
  worst = max(res, key=res.get)
  print('%s [%s]: worst %s %.3f; %s' % (tag, prec, worst, res[worst],
                                         ', '.join('%s %.2f' % kv for kv in sorted(res.items()))))
  for k, v in res.items():
    WORST[k] = max(WORST.get(k, 0.0), v)
  return res


def _leg_specs(eng):
  from oracle.tc_leg import layer_specs
  return layer_specs(eng.C, eng.model, eng.H, eng.W)


def _assert_within(res):
  bad = {k: v for k, v in res.items() if not v <= 1.0}
  assert not bad, bad


# ---- head-only flow ------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _bank(wf, seed=0):
  """Leg-like volumes: non-negative, a quarter exact zeros."""
  rng = np.random.default_rng(seed)
  v = rng.standard_normal((20, wf, 128)).astype(np.float32)
  return np.where(v > -0.7, np.abs(v) * 0.5, 0).astype(np.float32)


@pytest.mark.parametrize('prec', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('wf,s', [(360, 15), (225, 15), (405, 27), (360, 12)])
@pytest.mark.parametrize('n', [1, 5, 16])
def test_head_stages(n, wf, s, prec):
  model = _model(wf, s)
  w = N.glorot_weights(4, model, seed=1, leg_out_width=wf)
  H, W_ = image_size(model, wf)
  eng = Engine(model=model, precision='fp32', max_batch_scans=2, max_batch_pairs=16, proj_H=H, proj_W=W_)
  eng.load_weights(w)
  dev = eng.device
  bank = torch.from_numpy(_bank(wf)).to(dev)
  rng = np.random.default_rng(n * wf + s)
  left = rng.integers(0, 20, n).astype(np.int32)
  right = rng.integers(0, 20, n).astype(np.int32)
  right[0] = left[0]                                       # LEFT == RIGHT: every sign 0
  w = _spread(eng, w, bank, left, right, 4.0)
  eng.load_weights(w)
  eng.set_train_precision(prec)
  ov, _, _ = eng.heads(bank, torch.as_tensor(left).to(dev), torch.as_tensor(right).to(dev))
  gt_ov, gt_or = _targets(ov.cpu().numpy().astype(np.float64), rng, wf)
  st = Step(eng, False, bank, left, right, gt_ov, gt_or)
  res = check_step(st, w, bank, left, right, gt_ov, gt_or, prec, 'head n=%d (%d, %d)' % (n, wf, s))
  eng.close()
  _assert_within(res)


# ---- whole network -------------------------------------------------------------------------------------------
def _net_case(model, H, W, C, n, prec, offsets=None, maxp=None, seed=3):
  w = N.glorot_weights(C, model, seed=seed, leg_out_width=model['leg_output_width'])
  n_img = max(4, min(2 * n, 8))
  eng = Engine(use=USE[C], model=model, precision='fp32', max_batch_scans=n_img, max_batch_pairs=maxp or max(n, 4),
               proj_H=H, proj_W=W)
  eng.load_weights(w)
  dev = eng.device
  x = torch.from_numpy(synth.range_like_images(seed, n_img, C, H=H, W=W)).to(dev)
  rng = np.random.default_rng(seed + n)
  left = (np.arange(n) % n_img).astype(np.int32)
  right = rng.integers(0, n_img, n).astype(np.int32)
  right[0] = left[0]
  fv = eng.leg(x)
  w = _spread(eng, w, fv, left, right, 4.0)
  eng.load_weights(w)
  eng.set_train_precision(prec)
  ov, _, _ = eng.heads(eng.leg(x), torch.as_tensor(left).to(dev), torch.as_tensor(right).to(dev))
  gt_ov, gt_or = _targets(ov.cpu().numpy().astype(np.float64), rng, eng.Wf)
  st = Step(eng, True, x, left, right, gt_ov, gt_or, offsets)
  tag = 'net n=%d %dx%d C=%d %s 3a=%s%s' % (n, H, W, C, model['strides_layer1'],
                                             model['additional_unsymmetric_layer3a'],
                                             ' chunks %s' % (offsets,) if offsets else '')
  res = check_step(st, w, None, left, right, gt_ov, gt_or, prec, tag)
  eng.close()
  return res


NET_CASES = [  # (use3a, strides, H, W, C, n)
    (True, (2, 2), 64, 900, 4, 1), (True, (2, 2), 64, 900, 4, 3),
    (True, (2, 2), 49, 900, 4, 1), (True, (2, 2), 53, 900, 4, 1), (True, (2, 2), 57, 900, 4, 1),
    (True, (2, 2), 62, 900, 4, 1), (True, (2, 2), 80, 900, 4, 1), (True, (2, 2), 64, 899, 4, 1),
    (False, (2, 2), 32, 878, 4, 1), (False, (2, 2), 37, 878, 4, 1),
    (True, (1, 1), 32, 457, 4, 1), (True, (1, 2), 32, 900, 4, 1), (True, (2, 1), 64, 457, 4, 1),
    (True, (2, 2), 64, 900, 5, 1), (True, (2, 2), 64, 900, 25, 1),
]


@pytest.mark.parametrize('prec', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('use3a,strides,H,W,C,n', NET_CASES)
def test_net_stages(use3a, strides, H, W, C, n, prec):
  _assert_within(_net_case(_model(use3a=use3a, strides=strides), H, W, C, n, prec))


@pytest.mark.parametrize('prec', ['fp32', 'tf32x3'])
def test_chunked_net_stages(prec):
  """Uneven chunks and an empty one: each chunk's weight gradients from its own rows, the leg dy in chunk order."""
  _assert_within(_net_case(_model(), 64, 900, 4, 5, prec, offsets=[0, 2, 2, 5]))


def test_net_stages_leg_launches_split_over_images():
  """160 pairs: 320 images of 30 x 443 s_conv1 rows, more than one launch's grid holds (157 pairs)."""
  _assert_within(_net_case(_model(), 64, 900, 4, 160, 'fp32', maxp=160))


# ---- the handle after a stopped call -------------------------------------------------------------------------
def test_stopped_call_leaves_no_gradients_and_the_next_call_is_fresh():
  model = _model()
  w = N.glorot_weights(4, model, seed=2)
  x = synth.range_like_images(9, 4, 4)
  left, right = np.array([0, 1, 2], np.int32), np.array([1, 2, 2], np.int32)
  gt_ov, gt_or = np.array([0.2, 0.6, 0.9], np.float32), np.array([0, 359, 17], np.int32)

  def fresh(net):
    eng = Engine(model=model, precision='fp32', max_batch_scans=4, max_batch_pairs=4)
    eng.load_weights(w)
    return eng

  for net in (False, True):
    ref = fresh(net)
    dev = ref.device
    xs = torch.from_numpy(x).to(dev)
    rows = xs if net else ref.leg(xs)
    call = (lambda e: e.net_gradients if net else e.head_gradients)
    args = (rows, torch.as_tensor(left).to(dev), torch.as_tensor(right).to(dev), gt_ov, gt_or, 0.7)
    launches0 = ref.launch_count()
    loss_ref = call(ref)(*args)
    launches_ref = ref.launch_count() - launches0
    g_ref = ref.copy_gradients(net).cpu().numpy()
    ref.close()
    eng = fresh(net)
    stops = [('o1', 0), ('x4', 0)] + ([('dfv_corr', 0), ('leg_dy', 3)] if net else [])
    for stage, layer in stops:
      eng.set_train_stop(stage, layer)
      call(eng)(*args)
      assert eng.train_stage(stage, layer).numel() > 0
      for fn in (lambda: eng.copy_gradients(False), lambda: eng.get_gradients(['c_conv1']),
                 lambda: eng.adagrad_step(1e-3), lambda: eng.net_adagrad_step(1e-3), lambda: eng.net_volumes(),
                 lambda: eng.adagrad_step_sum(torch.zeros((1, eng.gradient_size(net)), device=dev), [1.0], 1e-3,
                                              net),
                 lambda: eng.train_stage('dz')):
        with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
          fn()
    with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
      eng.set_train_stop('dz')                               # read after a whole call, not a stop
    with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
      eng.set_train_stop('leg_dy', len(eng.leg_layers))
    launches0 = eng.launch_count()
    loss = call(eng)(*args)                                  # the stop was consumed: a whole call
    assert eng.launch_count() - launches0 == launches_ref
    assert loss == loss_ref
    assert np.array_equal(eng.copy_gradients(net).cpu().numpy().view(np.uint32), g_ref.view(np.uint32))
    with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
      eng.train_stage('o1')                                  # a stop stage is held only by the call that stopped
    if not net:
      with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
        eng.train_stage('part_l')                            # whole-network stages after a head-only call
    eng.close()


def test_zz_report():
  """The largest error / bound of each stage over the cases above, and the module's run time."""
  for k in sorted(WORST):
    print('%-24s %.3f' % (k, WORST[k]))
  print('test_gpu_train_stages: %.1f s' % (time.time() - T0))
