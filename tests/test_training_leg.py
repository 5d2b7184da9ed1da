"""CPU checks of whole-network training (legsType 360OutputkLegs): the float64 oracle's forward against
oracle/network, the configurations the driver accepts and refuses, and the dispatch of
``python -m overlapnet_b200.training`` on legsType."""
import os

import numpy as np
import pytest
import yaml

import train_leg_oracle as TL
from oracle import network as N
from overlapnet_b200 import synth, training, training_leg
from overlapnet_b200.engine import HEAD_LAYERS, leg_layers

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}


@pytest.mark.parametrize('use3a', [True, False])
def test_oracle_forward_matches_oracle_network(use3a):
  model = dict(MODEL, additional_unsymmetric_layer3a=use3a)
  w = N.glorot_weights(4, model, seed=2)
  x = synth.range_like_images(3, 2, 4)
  vol, ov, corr = TL.forward(x[:1], x[1:], w, model)
  fv = N.leg_forward(x, w, model, return_all=True)[-1][:, 0]            # float64, not rounded
  assert np.abs(vol - fv).max() <= 1e-12 * np.abs(fv).max()
  ov_ref, _, corr_ref = N.heads_forward(fv[:1, None], fv[1:, None], w, model)
  _, _, _, z = N.heads_forward(fv[:1, None], fv[1:, None], w, model, return_logit=True)
  assert abs(ov[0] - 1 / (1 + np.exp(-z[0]))) <= 1e-12
  assert abs(ov[0] - ov_ref[0]) <= 1e-7                                   # heads_forward rounds to float32
  assert np.abs(corr - corr_ref).max() <= 1e-12 * np.abs(corr_ref).max()


def test_leg_layer_names_follow_the_config():
  assert leg_layers(MODEL) == tuple(n for n, *_ in N.leg_layers(MODEL))
  assert 's_conv3a' not in leg_layers({}) and len(leg_layers({})) == 10 and len(leg_layers(MODEL)) == 11
  assert TL.layer_names(MODEL) == leg_layers(MODEL) + HEAD_LAYERS


def _config(tmp_path, legs='360OutputkLegs', **kw):
  cfg = {'experiments_path': str(tmp_path), 'testname': 't', 'pretrained_weightsfilename': '',
         'traindata_npzfile': 'x', 'validationdata_npzfile': 'y', 'batch_size': 2, 'no_batches_in_epoch': 1,
         'no_epochs': 1, 'no_test_pairs': 1, 'learning_rate': 1e-3,
         'model': {'modelType': 'SiameseNetworkTemplate', 'legsType': legs,
                   'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                   'inputShape': [64, 900], 'leg_output_width': 360}}
  cfg.update(kw)
  return cfg


def test_leg_driver_accepts_the_reference_default(tmp_path):
  training_leg.check_config(_config(tmp_path, rotate_training_data=0))


@pytest.mark.parametrize('change,match', [
    ({'legs': '360OutputkLegsFixed'}, 'overlapnet_b200.training'),
    ({'legs': 'SomethingElse'}, 'not supported'),
    ({'rotate_training_data': 1}, 'rotate_training_data'),
    ({'tensorboard': True}, 'TensorBoard'),
])
def test_leg_driver_refuses_unsupported_configs(tmp_path, change, match):
  change = dict(change)
  cfg = _config(tmp_path, change.pop('legs', '360OutputkLegs'), **change)
  with pytest.raises(Exception, match=match):
    training_leg.check_config(cfg)
  with pytest.raises(Exception, match=match):      # refused before any file or device is touched
    training_leg.train(cfg)
  assert not os.path.exists(os.path.join(str(tmp_path), 't'))


def test_frozen_leg_driver_names_the_new_flow(tmp_path):
  with pytest.raises(Exception, match='training_leg'):
    training.check_config(_config(tmp_path))


@pytest.mark.parametrize('legs,which', [('360OutputkLegs', 'leg'), ('360OutputkLegsFixed', 'head')])
def test_main_dispatches_on_legs_type(tmp_path, monkeypatch, legs, which):
  calls = []
  monkeypatch.setattr(training, 'train', lambda cfg, device=None: calls.append(('head', cfg)))
  monkeypatch.setattr(training_leg, 'train', lambda cfg, device=None: calls.append(('leg', cfg)))
  path = os.path.join(str(tmp_path), 'network.yml')
  with open(path, 'w') as f:
    yaml.safe_dump(_config(tmp_path, legs), f)
  training.main([path])
  assert [c[0] for c in calls] == [which] and calls[0][1]['model']['legsType'] == legs
