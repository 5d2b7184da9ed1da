"""CPU checks of overlap-head training: the losses of the float64 training oracle against independent
NumPy/SciPy values, the learning-rate schedule, the configurations the driver refuses and the weight
file it writes."""
import os

import numpy as np
import pytest
import torch
from scipy.special import expit

import train_oracle as T
from oracle import network as N
from overlapnet_b200 import training
from overlapnet_b200 import weights as W


@pytest.mark.parametrize('d,expected', [(0.0, expit(-6.0)), (0.25, 0.5), (0.5, expit(6.0))])
def test_sigmoid_loss_known_answers(d, expected):
  for y_true in (0.2, 0.7):
    for sgn in (1, -1):
      y = torch.tensor([y_true + sgn * d], dtype=torch.float64)
      got = float(T.sigmoid_loss(y, torch.tensor([y_true], dtype=torch.float64))[0])
      assert got == pytest.approx(expected, rel=1e-12)


def _wce_reference(t, x, q):
  # -(q t log sigmoid(x) + (1 - t) log(1 - sigmoid(x))) with log sigmoid(x) = -logaddexp(0, -x)
  return q * t * np.logaddexp(0.0, -x) + (1 - t) * np.logaddexp(0.0, x)


@pytest.mark.parametrize('x', [-1e4, -300.0, -30.0, -1.0, 0.0, 0.5, 30.0, 300.0, 1e4])
@pytest.mark.parametrize('t', [0.0, 1.0])
def test_weighted_cross_entropy_is_stable(x, t):
  got = T.weighted_ce(np.array([t]), np.array([x]), 360)[0]
  assert np.isfinite(got)
  # TF's form adds x and max(-x, 0): for x << 0 and t = 0 an exact 0 stands for exp(x)
  assert got == pytest.approx(_wce_reference(t, x, 360.0), rel=1e-12, abs=1e-12 * max(1.0, abs(x)))


def test_orientation_targets():
  t = T.orientation_targets(np.array([0.9, 0.5, 0.71, 0.7]), np.array([3, 4, 359, 0]), 360, 0.7)
  assert t.shape == (4, 360) and t.sum() == 2
  assert t[0, 3] == 1 and t[2, 359] == 1


def test_learning_rate_schedule():
  lrs = [training.learning_rate(e, 1e-3, 0.99) for e in range(3)]
  assert lrs == pytest.approx([1e-4, 1e-3, 0.99e-3], rel=1e-12)


def test_adagrad_oracle_first_step_is_sign_scaled():
  w = {n: (np.ones(3), np.zeros(1)) for n in T.HEAD}
  g = {n: (np.array([2.0, -0.5, 0.0]), np.array([1e-3])) for n in T.HEAD}
  acc = {}
  T.adagrad_step(w, g, acc, 0.1)
  k, b = w['c_conv1']
  assert k == pytest.approx([1 - 0.1 * 2 / (2 + 1e-7), 1 + 0.1 * 0.5 / (0.5 + 1e-7), 1.0])
  assert b == pytest.approx([-0.1 * 1e-3 / (1e-3 + 1e-7)])
  assert acc['c_conv1'][0] == pytest.approx([4.0, 0.25, 0.0])


def _config(tmp_path, **kw):
  cfg = {'experiments_path': str(tmp_path), 'testname': 't', 'pretrained_weightsfilename': '',
         'traindata_npzfile': 'x', 'validationdata_npzfile': 'y', 'batch_size': 2, 'no_batches_in_epoch': 1,
         'no_epochs': 1, 'no_test_pairs': 1, 'learning_rate': 1e-3,
         'model': {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegsFixed',
                   'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                   'inputShape': [64, 900], 'leg_output_width': 360}}
  cfg.update(kw)
  return cfg


@pytest.mark.parametrize('change,match', [
    ({'model': {'legsType': '360OutputkLegs'}}, '360OutputkLegsFixed'),
    ({'model': {'legsType': 'SomethingElse'}}, 'not supported'),
    ({'rotate_training_data': 1}, 'rotate_training_data'),
    ({'rotate_training_data': 2}, 'rotate_training_data'),
    ({'tensorboard': True}, 'TensorBoard'),
])
def test_driver_refuses_unsupported_configs(tmp_path, change, match):
  cfg = _config(tmp_path)
  if 'model' in change:
    cfg['model'].update(change['model'])
  else:
    cfg.update(change)
  with pytest.raises(Exception, match=match):
    training.check_config(cfg)
  with pytest.raises(Exception, match=match):      # refused before any file or device is touched
    training.train(cfg)
  assert not os.path.exists(os.path.join(str(tmp_path), 't'))


def test_driver_accepts_the_fixed_leg_config(tmp_path):
  training.check_config(_config(tmp_path, rotate_training_data=0))


def test_weight_file_round_trip(tmp_path):
  model = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
  w = N.glorot_weights(4, model, seed=3)
  path = os.path.join(str(tmp_path), 'SiameseNetworkTemplate_t.weight')
  training.save_weights(path, w)
  assert os.listdir(str(tmp_path)) == ['SiameseNetworkTemplate_t.weight']     # no '.npz' appended
  back = W.load(path)
  assert sorted(back) == sorted(w)
  for name, (k, b) in w.items():
    assert np.array_equal(back[name][0], k) and np.array_equal(back[name][1], b)


def test_orientation_rms_thresholds():
  ov = np.array([0.35, 0.95, 0.55])
  argmax = np.array([10, 355, 0])
  gt = np.array([13.0, 5.0, 0.0])
  r = training.orientation_rms(ov, argmax, gt, 360)
  assert r[0.3] == pytest.approx(np.sqrt((9 + 100 + 0) / 3))
  assert r[0.5] == pytest.approx(np.sqrt(100 / 2))
  assert r[0.9] == pytest.approx(10.0)
  assert r[0.6] == pytest.approx(10.0)
  assert np.isnan(training.orientation_rms(ov * 0.1, argmax, gt, 360)[0.3])      # no pair above: NaN
