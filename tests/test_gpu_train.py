"""Overlap-head training on the GPU through the C ABI against the float64 autograd oracle
(tests/train_oracle.py): gradients, Adagrad steps, determinism, error paths, the weight round trip
into a tensor-core Infer and the training.py driver end to end."""
import os

import numpy as np
import pytest
import torch

import train_oracle as T
from oracle import network as N
from overlapnet_b200 import synth, training
from overlapnet_b200 import weights as W
from overlapnet_b200._cabi import OvnError
from overlapnet_b200.engine import HEAD_LAYERS, Engine
from test_gpu_network import check_yaw

pytestmark = pytest.mark.gpu

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
N_SCANS = 8
MAXP = 16


def _engine(w, precision='fp32', maxp=MAXP):
  eng = Engine(model=MODEL, precision=precision, max_batch_scans=N_SCANS, max_batch_pairs=maxp)
  eng.load_weights(w)
  return eng


@pytest.fixture(scope='module')
def setup():
  """Bank of 8 scans from the fp32 leg, 16 (LEFT, RIGHT) pairs, Glorot weights with the Dense layer
  rescaled to a logit spread of 1.5, and targets above every prediction (so no |yhat - y| is 0 and the
  Dense-bias gradient does not cancel over the batch)."""
  w = N.glorot_weights(4, MODEL, seed=0)
  x = synth.range_like_images(77, N_SCANS, 4)
  eng = _engine(w)
  bank = eng.leg(torch.from_numpy(x).to(eng.device))
  eng.close()
  rng = np.random.default_rng(5)
  left = np.array([i % N_SCANS for i in range(MAXP)], np.int32)
  right = np.array([(i + 1 + i // N_SCANS) % N_SCANS for i in range(MAXP)], np.int32)
  fv = bank.cpu().numpy()
  _, _, _, z = N.heads_forward(fv[left][:, None], fv[right][:, None], w, MODEL, return_logit=True)
  w = N.spread_dense(w, z, target_std=1.5)
  ov_ref, _, _ = N.heads_forward(fv[left][:, None], fv[right][:, None], w, MODEL)
  gt_ov = (ov_ref + rng.uniform(0.15, 0.35, MAXP)).astype(np.float32)
  gt_or = rng.integers(0, 360, MAXP).astype(np.int32)
  return w, bank, fv, left, right, gt_ov, gt_or


def _idx(a, dev):
  return torch.from_numpy(np.ascontiguousarray(a, np.int32)).to(dev)


@pytest.mark.parametrize('n', [1, 16])
def test_gradients_match_float64_autograd(setup, n):
  w, bank, fv, left, right, gt_ov, gt_or = setup
  eng = _engine(w)
  loss = eng.head_gradients(bank, _idx(left[:n], eng.device), _idx(right[:n], eng.device), gt_ov[:n], gt_or[:n], 0.7)
  grads = eng.get_gradients()
  eng.close()
  ref_loss, ref = T.losses_and_gradients(fv[left[:n]], fv[right[:n]], w, gt_ov[:n], gt_or[:n], 0.7, MODEL)
  print('losses gpu %s oracle %s' % (loss, ref_loss))
  for got, exp in zip(loss, ref_loss):
    assert abs(got - exp) <= 1e-5 * abs(exp), (loss, ref_loss)
  for name in HEAD_LAYERS:
    for i, part in enumerate(('kernel', 'bias')):
      g, r = grads[name][i], ref[name][i]
      assert g.shape == r.shape
      err = float(np.abs(g - r).max()) / float(np.abs(r).max())
      print('%s %s: max|g - g_ref| / max|g_ref| = %.2e (max|g_ref| %.3e)' % (name, part, err, np.abs(r).max()))
      assert np.abs(r).max() > 0 and err <= 1e-4, (name, part, err)


def test_three_adagrad_steps_match_oracle(setup):
  w, bank, fv, left, right, gt_ov, gt_or = setup
  # Adagrad divides each gradient by its own running norm, so an element whose gradient is near zero (a
  # ReLU mask that fp32 and float64 decide differently) can take a step of size lr in either direction:
  # lr is chosen so that even such an element stays inside the tolerance (an H100 run at lr = 2e-6 had a
  # c_conv3 element 1.9 lr away from the oracle)
  n, lr = 4, 5e-8
  eng = _engine(w)
  li, ri = _idx(left[:n], eng.device), _idx(right[:n], eng.device)
  ref_w = {k: tuple(np.asarray(a, np.float64) for a in v) for k, v in w.items()}
  acc = {}
  for _ in range(3):
    eng.head_gradients(bank, li, ri, gt_ov[:n], gt_or[:n], 0.7)
    eng.adagrad_step(lr)
    _, g = T.losses_and_gradients(fv[left[:n]], fv[right[:n]], ref_w, gt_ov[:n], gt_or[:n], 0.7, MODEL)
    T.adagrad_step(ref_w, g, acc, lr)
  got = eng.get_weights()
  eng.close()
  for name in HEAD_LAYERS:
    for i in range(2):
      scale = float(np.abs(ref_w[name][i]).max())
      err = float(np.abs(got[name][i] - ref_w[name][i]).max())
      moved = float(np.abs(got[name][i] - w[name][i]).max())
      print('%s[%d]: max err %.2e, moved %.2e, tol %.2e' % (name, i, err, moved, 1e-5 * scale))
      assert err <= 1e-5 * scale, (name, i, err, scale)
      if i == 0:        # a bias of order 1 (the rescaled Dense bias) cannot take steps this small in fp32
        assert moved > 0, (name, i)
  for name in w:
    if name not in HEAD_LAYERS:                       # the frozen leg is never touched
      assert np.array_equal(got[name][0], w[name][0]) and np.array_equal(got[name][1], w[name][1]), name


def test_training_is_bit_reproducible(setup):
  w, bank, fv, left, right, gt_ov, gt_or = setup
  out = []
  for _ in range(2):
    eng = _engine(w)
    li, ri = _idx(left, eng.device), _idx(right, eng.device)
    for _ in range(5):
      eng.head_gradients(bank, li, ri, gt_ov, gt_or, 0.7)
      eng.adagrad_step(1e-4)
    out.append(eng.get_weights(HEAD_LAYERS))
    eng.close()
  for name in HEAD_LAYERS:
    for i in range(2):
      assert np.array_equal(out[0][name][i].view(np.uint32), out[1][name][i].view(np.uint32)), name


def test_training_errors(setup):
  w, bank, fv, left, right, gt_ov, gt_or = setup
  eng = _engine(w)
  dev = eng.device
  before = eng.get_weights(HEAD_LAYERS)
  bad = left[:4].copy()
  bad[2] = N_SCANS                                   # one past the bank
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.head_gradients(bank, _idx(bad, dev), _idx(right[:4], dev), gt_ov[:4], gt_or[:4], 0.7)
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.adagrad_step(1e-3)
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.get_gradients()
  after = eng.get_weights(HEAD_LAYERS)
  for name in HEAD_LAYERS:
    assert np.array_equal(before[name][0], after[name][0]) and np.array_equal(before[name][1], after[name][1])
  big = np.arange(MAXP + 1, dtype=np.int32) % N_SCANS
  with pytest.raises(OvnError, match='OVN_ERR_CAPACITY'):
    eng.head_gradients(bank, _idx(big, dev), _idx(big[::-1].copy(), dev), np.full(MAXP + 1, 0.5, np.float32),
                       np.zeros(MAXP + 1, np.int32), 0.7)
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.get_gradients(['s_conv1'])                   # gradients exist for the head layers only
  # the handle is still healthy: a valid batch trains, and no device fault happened
  eng.head_gradients(bank, _idx(left[:4], dev), _idx(right[:4], dev), gt_ov[:4], gt_or[:4], 0.7)
  eng.adagrad_step(1e-3)
  eng.check()
  torch.cuda.synchronize()
  eng.close()
  tc = _engine(w, precision='f16_tc')
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG'):
    tc.head_gradients(bank, _idx(left[:4], dev), _idx(right[:4], dev), gt_ov[:4], gt_or[:4], 0.7)
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG'):
    tc.adagrad_step(1e-3)
  tc.close()


def test_trained_weights_round_trip_into_tensor_core_infer(setup, tmp_path):
  from overlapnet_b200.infer import Infer
  w, bank, fv, left, right, gt_ov, gt_or = setup
  eng = _engine(w)
  dev = eng.device
  for _ in range(3):
    eng.head_gradients(bank, _idx(left[:8], dev), _idx(right[:8], dev), gt_ov[:8], gt_or[:8], 0.7)
    eng.adagrad_step(1e-5)
  path = os.path.join(str(tmp_path), 'SiameseNetworkTemplate_rt.weight')
  training.save_weights(path, eng.get_weights())
  hl, hr = left[8:], right[8:]                        # held-out pairs
  ov32, yaw32, corr32 = eng.heads(bank, _idx(hl, dev), _idx(hr, dev), want_corr=True)
  ov32, yaw32, corr32 = ov32.cpu().numpy(), yaw32.cpu().numpy(), corr32.cpu().numpy()
  eng.close()
  cfg = {'model': {'leg_output_width': 360, 'inputShape': [64, 900], 'legsType': '360OutputkLegsFixed',
                   'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                   **MODEL},
         'infer_seqs': '', 'data_root_folder': str(tmp_path), 'batch_size': 8, 'use_depth': True,
         'use_normals': True, 'use_class_probabilities': False, 'use_class_probabilities_pca': False,
         'use_intensity': False, 'pretrained_weightsfilename': path}
  inf = Infer(cfg, precision='f16_tc')
  ov16, corr16 = inf.head.predict([fv[hl][:, None], fv[hr][:, None]])
  yaw16 = 180 - np.argmax(corr16, axis=1)
  d = float(np.abs(ov16[:, 0] - ov32).max())
  print('held-out overlaps %s, max |f16_tc - fp32| = %.2e' % (np.round(ov32, 3).tolist(), d))
  assert d <= 1e-3
  check_yaw(yaw16, yaw32, corr32)


def _write_dataset(root, w, seed=11):
  """Two sequences of cue images (depth + normals) and GT npz files whose overlaps come from a seeded
  teacher head; returns the pretrained weight file (the teacher's leg, a fresh Glorot head)."""
  rng = np.random.default_rng(seed)
  seqs = {'00': 6, '01': 5}
  eng = _engine(w, maxp=64)
  for si, (seq, n) in enumerate(seqs.items()):
    x = synth.range_like_images(seed + si, n, 4)
    for sub in ('depth', 'normal'):
      os.makedirs(os.path.join(root, seq, sub), exist_ok=True)
    for i in range(n):
      np.save(os.path.join(root, seq, 'depth', '%06d.npy' % i), x[i, :, :, 0])
      np.save(os.path.join(root, seq, 'normal', '%06d.npy' % i), x[i, :, :, 1:4])
    bank = eng.leg(torch.from_numpy(x).to(eng.device))
    pairs = np.array([(i, j) for i in range(n) for j in range(n) if i != j])
    ov, _, _ = eng.heads(bank, _idx(pairs[:, 0], eng.device), _idx(pairs[:, 1], eng.device))
    table = np.zeros((len(pairs), 4))
    table[:, :2] = pairs
    table[:, 2] = ov.cpu().numpy()
    table[:, 3] = rng.integers(0, 360, len(pairs))
    perm = rng.permutation(len(pairs))
    n_val = len(pairs) // 4
    os.makedirs(os.path.join(root, seq, 'ground_truth'), exist_ok=True)
    for name, sel in (('validation_set', perm[:n_val]), ('train_set', perm[n_val:])):
      np.savez(os.path.join(root, seq, 'ground_truth', name + '.npz'), overlaps=table[sel],
               seq=np.array([[seq, seq]] * len(sel)))
  eng.close()
  student = dict(w)
  fresh = N.glorot_weights(4, MODEL, seed=1)
  for name in HEAD_LAYERS:
    student[name] = fresh[name]
  path = os.path.join(root, 'pretrained.weight')
  training.save_weights(path, student)
  return path


def test_training_driver_end_to_end(tmp_path):
  root = str(tmp_path / 'data')
  teacher = N.glorot_weights(4, MODEL, seed=0)
  eng = _engine(teacher, maxp=64)
  x = synth.range_like_images(11, 6, 4)
  fvh = eng.leg(torch.from_numpy(x).to(eng.device)).cpu().numpy()
  eng.close()
  _, _, _, z = N.heads_forward(fvh[:, None], np.roll(fvh, 1, 0)[:, None], teacher, MODEL, return_logit=True)
  teacher = N.spread_dense(teacher, z, target_std=1.5)
  pretrained = _write_dataset(root, teacher)
  cfg = {'experiments_path': str(tmp_path / 'exp'), 'testname': 'e2e', 'pretrained_weightsfilename': pretrained,
         'use_depth': True, 'use_normals': True, 'data_root_folder': root, 'training_seqs': '00 01',
         'batch_size': 8, 'no_batches_in_epoch': 1000, 'no_epochs': 3, 'no_test_pairs': 1000,
         'learning_rate': 1e-4, 'lr_alpha': 0.99, 'min_overlap_for_angle': 0.7,
         'model': {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegsFixed',
                   'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                   'inputShape': [64, 900], 'leg_output_width': 360, **MODEL}}
  np.random.seed(0)
  hist = training.train(cfg)
  print('epoch losses', hist['epoch_loss'], 'validation', [v['rms'] for v in hist['validation']])
  out = os.path.join(str(tmp_path / 'exp'), 'e2e')
  wfile = os.path.join(out, 'SiameseNetworkTemplate_e2e.weight')
  assert hist['weights_filename'] == wfile and os.path.isfile(wfile)
  log = open(os.path.join(out, 'training.log')).read()
  assert 'iteration 3, batch/epoch loss' in log and 'RMS  overlap error' in log
  assert len(hist['epoch_loss']) == 3 and hist['epoch_loss'][-1] < hist['epoch_loss'][0]
  back = W.load(wfile)
  start = W.load(pretrained)
  assert sorted(back) == sorted(start)
  for name in back:
    same = np.array_equal(back[name][0], start[name][0])
    assert same == (name not in HEAD_LAYERS), name      # head trained, leg frozen
