"""Training at training precision tf32x3 (ovn_set_train_precision: every product of ovn_head_gradients and
ovn_net_gradients on 3xTF32 mma.sync) against the float64 autograd oracles (tests/train_oracle.py,
tests/train_leg_oracle.py) and against the fp32 SIMT step on the same handle: gradients of both flows at three
head geometries, a batch whose leg launches split, the pair limit, Adagrad, determinism, isolation from every
other entry point, errors, and both drivers on two ranks."""
import copy
import os
import pickle

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import train_leg_oracle as TL
import train_oracle as T
import test_gpu_geometry as GEO
import test_gpu_train as HG
import test_gpu_train_dp as DP
import test_gpu_train_leg as LG
from overlapnet_b200 import weights as Wt
from overlapnet_b200._cabi import OvnError, lib
from overlapnet_b200.engine import HEAD_LAYERS
from test_gpu_train import setup  # noqa: F401  (the head-only fixture)
from test_gpu_train_dp import dataset  # noqa: F401  (the driver dataset fixture)

pytestmark = pytest.mark.gpu

OVN_ERR_INVALID_ARG = -1


def bits(a):
  return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _idx(a, dev):
  return torch.from_numpy(np.ascontiguousarray(a, np.int32)).to(dev)


def _rel(g, r):
  return float(np.abs(np.asarray(g, np.float64) - r).max()) / float(np.abs(r).max())


def _check_layers(got, ref, fp32, names, tol):
  """Every layer against the oracle (bounded by tol(name)) and, reported, against the fp32 SIMT step."""
  for name in names:
    for i, part in enumerate(('kernel', 'bias')):
      g, r = got[name][i], ref[name][i]
      assert g.shape == r.shape
      err, dev32, err32 = _rel(g, r), _rel(g, fp32[name][i]), _rel(fp32[name][i], r)
      print('%s %s: tf32x3 vs oracle %.2e (fp32 vs oracle %.2e), tf32x3 vs fp32 %.2e, bound %.0e'
            % (name, part, err, err32, dev32, tol(name)))
      assert np.abs(r).max() > 0 and err <= tol(name), (name, part, err)


# ---- overlap head with a frozen leg -------------------------------------------------------------------------
@pytest.mark.parametrize('n', [1, 4, 16])
def test_head_gradients_match_oracle_and_fp32(setup, n):  # noqa: F811
  w, bank, fv, left, right, gt_ov, gt_or = setup
  eng = HG._engine(w)
  li, ri = _idx(left[:n], eng.device), _idx(right[:n], eng.device)
  loss32 = eng.head_gradients(bank, li, ri, gt_ov[:n], gt_or[:n], 0.7)
  g32 = eng.get_gradients()
  eng.set_train_precision('tf32x3')
  loss = eng.head_gradients(bank, li, ri, gt_ov[:n], gt_or[:n], 0.7)
  grads = eng.get_gradients()
  eng.close()
  ref_loss, ref = T.losses_and_gradients(fv[left[:n]], fv[right[:n]], w, gt_ov[:n], gt_or[:n], 0.7, HG.MODEL)
  print('losses tf32x3 %s fp32 %s oracle %s' % (loss, loss32, ref_loss))
  for got, exp in zip(loss, ref_loss):
    assert abs(got - exp) <= 1e-5 * abs(exp), (loss, ref_loss)
  _check_layers(grads, ref, g32, HEAD_LAYERS, lambda name: 1e-5)


def test_head_three_adagrad_steps_match_oracle(setup):  # noqa: F811
  """test_gpu_train.py's three-step check (its lr and bound) at tf32x3."""
  w, bank, fv, left, right, gt_ov, gt_or = setup
  n, lr = 4, 5e-8
  eng = HG._engine(w)
  eng.set_train_precision('tf32x3')
  li, ri = _idx(left[:n], eng.device), _idx(right[:n], eng.device)
  ref_w = {k: tuple(np.asarray(a, np.float64) for a in v) for k, v in w.items()}
  acc = {}
  for _ in range(3):
    eng.head_gradients(bank, li, ri, gt_ov[:n], gt_or[:n], 0.7)
    eng.adagrad_step(lr)
    _, g = T.losses_and_gradients(fv[left[:n]], fv[right[:n]], ref_w, gt_ov[:n], gt_or[:n], 0.7, HG.MODEL)
    T.adagrad_step(ref_w, g, acc, lr)
  got = eng.get_weights()
  eng.close()
  for name in HEAD_LAYERS:
    for i in range(2):
      scale = float(np.abs(ref_w[name][i]).max())
      err = float(np.abs(got[name][i] - ref_w[name][i]).max())
      print('%s[%d]: max err %.2e, tol %.2e' % (name, i, err, 1e-5 * scale))
      assert err <= 1e-5 * scale, (name, i, err, scale)
      if i == 0:
        assert float(np.abs(got[name][i] - w[name][i]).max()) > 0, (name, i)


def test_head_training_is_bit_reproducible(setup):  # noqa: F811
  w, bank, fv, left, right, gt_ov, gt_or = setup
  out = []
  for _ in range(2):
    eng = HG._engine(w)
    eng.set_train_precision('tf32x3')
    li, ri = _idx(left, eng.device), _idx(right, eng.device)
    for _ in range(5):
      eng.head_gradients(bank, li, ri, gt_ov, gt_or, 0.7)
      eng.adagrad_step(1e-4)
    out.append(eng.get_weights(HEAD_LAYERS))
    eng.close()
  for name in HEAD_LAYERS:
    for i in range(2):
      assert np.array_equal(bits(out[0][name][i]), bits(out[1][name][i])), name


# ---- whole network ----------------------------------------------------------------------------------------
# A tf32x3 step computes its own volumes in its leg forward; they differ from the fp32 leg's at rounding level, and
# that alone flips sign(l - r) of |l - r| and head ReLU masks.  So, like the fp32 tests, the oracle's heads run at the
# device's volumes: those of the tf32x3 step itself (ovn_copy_net_volumes).
def _net_step(eng, xs, li, ri, gt_ov, gt_or):
  """losses, dL/d(volumes), every layer's gradients and the step's own volumes [2n, Wf, 128]"""
  loss, dfv = eng.net_gradients(xs, li, ri, gt_ov, gt_or, 0.7, fv_grad=True)
  vol = eng.net_volumes().cpu().numpy()
  return loss, dfv.cpu().numpy(), eng.get_gradients(eng.layers), vol.reshape((-1,) + vol.shape[2:])


def _check_net(model, x, l, r, w, gt_ov, gt_or, got, fp32, head_tol, leg_tol, dfv_tol):
  loss, dfv, grads, vol = got
  loss32, dfv32, g32, vol32 = fp32
  n = len(l)
  print('volumes: tf32x3 vs fp32 leg %.2e' % _rel(vol, vol32))
  print('head ReLU margins at the tf32x3 volumes', GEO._head_relu_margins(vol[:n], vol[n:], w, model))
  ref_loss, ref, ref_dfv = TL.losses_and_gradients(x[l], x[r], w, gt_ov, gt_or, 0.7, model, fv=vol)
  print('losses tf32x3 %s fp32 %s oracle %s' % (loss, loss32, ref_loss))
  for got_l, exp in zip(loss, ref_loss):
    assert abs(got_l - exp) <= 1e-5 * abs(exp), (loss, ref_loss)
  assert dfv.shape == ref_dfv.shape == (2, n, vol.shape[1], 128)
  err = _rel(dfv, ref_dfv)
  print('dL/d(volumes): tf32x3 vs oracle %.2e, tf32x3 vs fp32 %.2e, bound %.0e' % (err, _rel(dfv, dfv32), dfv_tol))
  assert err <= dfv_tol
  assert sorted(grads) == sorted(ref)
  _check_layers(grads, ref, g32, TL.layer_names(model), lambda name: head_tol if name in HEAD_LAYERS else leg_tol)


@pytest.mark.parametrize('use3a', [True, False])
@pytest.mark.parametrize('n', [1, 4])
def test_net_gradients_match_oracle_and_fp32(n, use3a):
  """dL/d(volumes) and the head gradients within 1e-5, the leg within 5e-5 with s_conv3a.  Without s_conv3a one
  s_conv7 pre-activation of images 0 / 1 is 2.1e-8 of its layer's largest (test_gpu_train_leg.py): its mask can
  flip between device arithmetic and float64, which moves the leg layers up to 4e-3 (the ReLU-margin rule)."""
  w, x, _, gt_ov, gt_or = LG._setup(use3a)
  model = LG._model(use3a)
  eng = LG._engine(w, use3a)
  dev = eng.device
  xs = torch.from_numpy(x).to(dev)
  l, r = LG.LEFT[:n], LG.RIGHT[:n]
  li, ri = _idx(l, dev), _idx(r, dev)
  fp32 = _net_step(eng, xs, li, ri, gt_ov[:n], gt_or[:n])
  eng.set_train_precision('tf32x3')
  got = _net_step(eng, xs, li, ri, gt_ov[:n], gt_or[:n])
  eng.close()
  _check_net(model, x, l, r, w, gt_ov[:n], gt_or[:n], got, fp32, 1e-5, 5e-5 if use3a else 4e-3, 1e-5)


@pytest.mark.parametrize('wf,s', GEO.TRAIN_GEOMETRIES)
def test_gradients_at_head_geometry(wf, s):
  """Tails of the 64 x 64 x 16 tile in M, N and K: both flows on four pairs chosen by their head ReLU margins, at
  the bounds of test_gpu_geometry.py (the whole network's oracle at the step's own volumes), and against the fp32
  step."""
  n = GEO.N_PAIRS
  model, w, x, fv, left, right, gt_ov, gt_or = GEO._train_setup(wf, s)
  eng = GEO._train_engine(wf, s, w)
  dev = eng.device
  bank, xs = torch.from_numpy(fv).to(dev), torch.from_numpy(x).to(dev)
  li, ri = _idx(left, dev), _idx(right, dev)
  out = {}
  for prec in ('fp32', 'tf32x3'):
    eng.set_train_precision(prec)
    head = (eng.head_gradients(bank, li, ri, gt_ov, gt_or, 0.7), eng.get_gradients())
    out[prec] = head, _net_step(eng, xs, li, ri, gt_ov, gt_or)
  eng.close()
  ref_loss, ref = T.losses_and_gradients(fv[left], fv[right], w, gt_ov[:n], gt_or[:n], 0.7, model)
  (loss, grads), (loss32, g32) = out['tf32x3'][0], out['fp32'][0]
  for got, exp in zip(loss, ref_loss):
    assert abs(got - exp) <= 1e-5 * abs(exp), (loss, ref_loss)
  _check_layers(grads, ref, g32, HEAD_LAYERS, lambda name: 1e-4)
  _check_net(model, x, left, right, w, gt_ov, gt_or, out['tf32x3'][1], out['fp32'][1], 1e-4, 1e-3, 1e-4)


def test_net_batch_split_over_leg_launches_matches_small_batch():
  """test_gpu_train_leg.py's 160-pair batch (pairs 0-3 repeated 40 times, leg launches split over images) at
  tf32x3 against the 4-pair batch."""
  w, x, _, gt_ov, gt_or = LG._setup(True)
  reps, n = 40, 4
  out = {}
  for k in (1, reps):
    eng = LG._engine(w, maxp=n * k)
    eng.set_train_precision('tf32x3')
    dev = eng.device
    sel = np.tile(np.arange(n), k)
    loss, dfv = eng.net_gradients(torch.from_numpy(x).to(dev), _idx(LG.LEFT[sel], dev), _idx(LG.RIGHT[sel], dev),
                                  gt_ov[sel], gt_or[sel], 0.7, fv_grad=True)
    out[k] = (loss, dfv.cpu().numpy(), eng.get_gradients(eng.layers))
    eng.close()
  (l1, f1, g1), (lk, fk, gk) = out[1], out[reps]
  for a, b in zip(l1, lk):
    assert abs(a - b) <= 1e-5 * abs(a), (l1, lk)
  err = _rel(fk.reshape(2, reps, n, 360, 128) * reps, f1[:, None])
  print('dL/d(volumes), 160 pairs vs 4: %.2e' % err)
  assert err <= 1e-5
  for name in g1:
    for i in range(2):
      err = _rel(gk[name][i], g1[name][i])
      print('%s[%d]: 160 pairs vs 4: %.2e' % (name, i, err))
      assert err <= 1e-4, (name, i, err)


def test_net_pair_limit_is_unchanged():
  """485 pairs at Wf = 360 fill grid.y of the heads' c_conv1 (485 * 360 * 24 rows, 64 per CTA): they train, and
  486 are refused."""
  w, x, _, gt_ov, gt_or = LG._setup(True)
  eng = LG._engine(w, maxp=486)
  eng.set_train_precision('tf32x3')
  dev = eng.device
  xs = torch.from_numpy(x).to(dev)
  big = np.arange(486, dtype=np.int32) % LG.N_IMAGES
  rev = big[::-1].copy()
  with pytest.raises(OvnError, match='OVN_ERR_CAPACITY.*485 pairs'):
    eng.net_gradients(xs, _idx(big, dev), _idx(rev, dev), np.full(486, 0.5, np.float32), np.zeros(486, np.int32), 0.7)
  loss = eng.net_gradients(xs, _idx(big[:485], dev), _idx(rev[:485], dev), np.full(485, 0.5, np.float32),
                           np.zeros(485, np.int32), 0.7)
  grads = eng.get_gradients(eng.layers)
  eng.check()
  eng.close()
  assert all(np.isfinite(v) for v in loss), loss
  for name, (k, b) in grads.items():
    assert np.isfinite(k).all() and np.isfinite(b).all() and np.abs(k).max() > 0, name


def test_net_three_adagrad_steps_match_oracle():
  """test_gpu_train_leg.py's three-step check at tf32x3: the first step's gradients against float64 autograd (at
  the step's own volumes) at this file's bounds, then the device's displacement against the oracle's Adagrad on the
  device's gradients."""
  w, x, _, gt_ov, gt_or = LG._setup(True)
  n, lr, steps = 2, 1e-5, 3
  eng = LG._engine(w)
  eng.set_train_precision('tf32x3')
  dev = eng.device
  xs = torch.from_numpy(x).to(dev)
  li, ri = _idx(LG.LEFT[:n], dev), _idx(LG.RIGHT[:n], dev)
  ref_w = {k: tuple(np.asarray(a, np.float64) for a in v) for k, v in w.items()}
  acc = {}
  for step in range(steps):
    w_now = eng.get_weights()
    eng.net_gradients(xs, li, ri, gt_ov[:n], gt_or[:n], 0.7)
    g_dev = eng.get_gradients(eng.layers)
    vol = eng.net_volumes().cpu().numpy()
    eng.net_adagrad_step(lr)
    if step == 0:
      _, g_ref, _ = TL.losses_and_gradients(x[LG.LEFT[:n]], x[LG.RIGHT[:n]], w_now, gt_ov[:n], gt_or[:n], 0.7,
                                            LG.MODEL, fv=vol.reshape((-1,) + vol.shape[2:]))
      for name in g_ref:
        for i in range(2):
          err = _rel(g_dev[name][i], g_ref[name][i])
          print('step 0 %s[%d]: %.2e' % (name, i, err))
          assert err <= (1e-5 if name in HEAD_LAYERS else 5e-5), (name, i, err)
    TL.adagrad_step(ref_w, g_dev, acc, lr)
  got = eng.get_weights()
  eng.close()
  for name in TL.layer_names(LG.MODEL):
    for i in range(2):
      w0 = np.asarray(w[name][i], np.float32)
      d_got = got[name][i].astype(np.float64) - w0
      d_ref = ref_w[name][i] - w0
      tol = 1e-4 * steps * lr + steps * np.spacing(np.abs(w0) + steps * lr)
      err = float((np.abs(d_got - d_ref) / tol).max())
      print('%s[%d]: max |d - d_ref| / tol = %.2e' % (name, i, err))
      assert err <= 1, (name, i, err)
      assert float(np.abs(d_got).max()) >= lr, name


def test_net_training_is_bit_reproducible():
  w, x, _, gt_ov, gt_or = LG._setup(True)
  out = []
  for _ in range(2):
    eng = LG._engine(w)
    eng.set_train_precision('tf32x3')
    dev = eng.device
    xs = torch.from_numpy(x).to(dev)
    li, ri = _idx(LG.LEFT, dev), _idx(LG.RIGHT, dev)
    for _ in range(5):
      eng.net_gradients(xs, li, ri, gt_ov, gt_or, 0.7)
      eng.net_adagrad_step(1e-4)
    out.append(eng.get_weights())
    eng.close()
  for name in out[0]:
    for i in range(2):
      assert np.array_equal(bits(out[0][name][i]), bits(out[1][name][i])), name


# ---- isolation and errors ------------------------------------------------------------------------------------
def test_other_entry_points_stay_fp32_simt():
  """ovn_leg_forward and ovn_heads_forward give the same bits before the mode is set and after tf32x3 gradient
  calls; after switching back to fp32, both gradient calls give the bits of a handle that never switched."""
  w, x, _, gt_ov, gt_or = LG._setup(True)
  n = 4
  eng = LG._engine(w)
  dev = eng.device
  xs = torch.from_numpy(x).to(dev)
  li, ri = _idx(LG.LEFT[:n], dev), _idx(LG.RIGHT[:n], dev)

  def forward():
    bank = eng.leg(xs)
    ov, yaw, corr = eng.heads(bank, li, ri, want_corr=True)
    return bank, [t.cpu().numpy() for t in (bank, ov, yaw, corr)]

  def gradients(e):
    bank = e.leg(xs)
    e.head_gradients(bank, li, ri, gt_ov[:n], gt_or[:n], 0.7)
    g_head = e.get_gradients(HEAD_LAYERS)
    e.net_gradients(xs, li, ri, gt_ov[:n], gt_or[:n], 0.7)
    return g_head, e.get_gradients(e.layers)

  _, before = forward()
  eng.set_train_precision('tf32x3')
  _, set_only = forward()
  tc = gradients(eng)
  _, after = forward()
  for a, b, c in zip(before, set_only, after):
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and np.array_equal(a.view(np.uint32),
                                                                                    c.view(np.uint32))
  eng.set_train_precision('fp32')
  back = gradients(eng)
  eng.close()
  fresh = LG._engine(w)
  never = gradients(fresh)
  fresh.close()
  for gb, gn, gt in zip(back, never, tc):
    differs = False
    for name in gn:
      for i in range(2):
        assert np.array_equal(bits(gb[name][i]), bits(gn[name][i])), name
        differs |= not np.array_equal(bits(gt[name][i]), bits(gn[name][i]))
    assert differs                       # the tf32x3 calls did take the other kernels


def test_net_volumes_are_the_steps_leg_output():
  """ovn_copy_net_volumes: at fp32 the last batch's volumes are ovn_leg_forward's bits for its LEFT, then RIGHT
  images; refused before any whole-network batch and after a head-only one."""
  w, x, _, gt_ov, gt_or = LG._setup(True)
  n = 4
  eng = LG._engine(w)
  dev = eng.device
  xs = torch.from_numpy(x).to(dev)
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.net_volumes()
  eng.net_gradients(xs, _idx(LG.LEFT[:n], dev), _idx(LG.RIGHT[:n], dev), gt_ov[:n], gt_or[:n], 0.7)
  vol = eng.net_volumes().cpu().numpy()
  fv = eng.leg(xs).cpu().numpy()
  assert np.array_equal(bits(vol[0]), bits(fv[LG.LEFT[:n]])) and np.array_equal(bits(vol[1]), bits(fv[LG.RIGHT[:n]]))
  eng.head_gradients(torch.from_numpy(fv).to(dev), _idx(LG.LEFT[:n], dev), _idx(LG.RIGHT[:n], dev), gt_ov[:n],
                     gt_or[:n], 0.7)
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.net_volumes()
  eng.close()


def test_train_precision_errors():
  w, *_ = LG._setup(True)
  eng = LG._engine(w)
  assert lib().ovn_set_train_precision(eng._h, 2) == OVN_ERR_INVALID_ARG
  assert lib().ovn_set_train_precision(eng._h, -1) == OVN_ERR_INVALID_ARG
  with pytest.raises(ValueError, match='fp32, tf32x3'):
    eng.set_train_precision('tf32')
  eng.set_train_precision('tf32x3')
  eng.set_train_precision('fp32')
  eng.close()
  tc = LG._engine(w, precision='f16_tc')
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG'):
    tc.set_train_precision('tf32x3')
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG'):
    tc.set_train_precision('fp32')
  tc.close()


# ---- both drivers on two ranks ---------------------------------------------------------------------------------
@pytest.mark.parametrize('yaw', [False, True])
@pytest.mark.parametrize('legs', sorted(DP.FLOWS))
def test_drivers_on_two_ranks_at_tf32x3(tmp_path, monkeypatch, dataset, legs, yaw):  # noqa: F811
  """Both training drivers with ``training_precision: tf32x3`` on two gloo ranks sharing one GPU: the ranks end
  with bit-identical weights, equal to a one-process emulation of the two ranks, and every trained layer moved."""
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  cfg = dict(DP._config(root, pretrained, exp, 'dp', legs, yaw), training_precision='tf32x3')
  out = str(tmp_path / 'rank%d.pkl')
  mp.spawn(DP._dp_worker, args=(2, DP._free_port(), 'gloo', copy.deepcopy(cfg), out), nprocs=2, join=True)
  ranks = []
  for r in range(2):
    with open(out % r, 'rb') as f:
      ranks.append(pickle.load(f))
  module, name, train = DP.FLOWS[legs]
  monkeypatch.setattr(module, name, DP._emulated(getattr(module, name)))
  np.random.seed(0)
  emu = train(dict(DP._config(root, pretrained, exp, 'emu', legs, yaw), training_precision='tf32x3'))
  start = Wt.load(pretrained)
  emu_w = Wt.load(emu['weights_filename'])
  for wname in start:
    for i in range(2):
      ref = bits(ranks[0]['weights'][wname][i])
      assert np.array_equal(bits(ranks[1]['weights'][wname][i]), ref), ('rank 1', wname, i)
      assert np.array_equal(bits(emu_w[wname][i]), ref), ('emulation', wname, i)
    trained = not np.array_equal(emu_w[wname][0], start[wname][0])
    assert trained == (legs == '360OutputkLegs' or wname in HEAD_LAYERS), wname
  assert ranks[0]['hist']['batch_losses'] == ranks[1]['hist']['batch_losses'] == emu['batch_losses']
  print(legs, 'yaw' if yaw else '', 'epoch losses', emu['epoch_loss'])
  for d in ('dp', 'emu'):
    log = open(os.path.join(exp, d, 'training.log')).read()
    assert 'Training precision: tf32x3' in log and 'iteration 2, batch/epoch loss' in log
