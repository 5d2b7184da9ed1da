"""Yaw augmentation on the GPU: ovn_gather_images bit-exact against the NumPy oracle of tests/test_yaw_augmentation.py,
its error paths, the augmented steps of both training flows against the plain C-ABI calls on oracle-augmented
inputs (and the float64 autograd oracle), and both training drivers end to end with ``yaw_augmentation: True``."""
import functools
import os

import numpy as np
import pytest
import torch

import train_leg_oracle as TL
from oracle import network as N
from oracle import projection as P
from overlapnet_b200 import augment, synth, training, training_leg
from overlapnet_b200 import weights as Wt
from overlapnet_b200._cabi import OvnError
from overlapnet_b200.engine import HEAD_LAYERS, Engine
from test_gpu_train import _write_dataset
from test_gpu_train_leg import LEFT, MODEL, RIGHT, _engine, _idx, _setup
from test_yaw_augmentation import augment_oracle

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CASES = ['kitti_000000', 'kitti_000001', 'synth_3', 'synth_5']
# shifts 0, p, W/2, W - p, a non-multiple of the pitch and a negative one (taken mod W)
SHIFTS = np.array([0, 5, 450, 895, 7, -5], np.int32)
ROWS = np.array([0, 1, 2, 3, 0, 2], np.int32)


def bits(a):
  return np.ascontiguousarray(a, np.float32).view(np.uint32)


@functools.lru_cache(maxsize=None)
def _golden_images():
  """Depth, normals, 20 class probabilities and intensity of the golden clouds (C = 25), by the oracle: the
  normal maps hold the (-1, -1, -1) fill wherever a neighbour is empty."""
  out = []
  for i, case in enumerate(CASES):
    pts = np.load(os.path.join(GOLDEN, case + '.npz'))['points']
    rng, vert, inten, _ = P.range_projection(pts)
    prob = P.gen_semantic_image(pts, synth.random_probs(40 + i, pts.shape[0]))
    out.append(P.pack_input(rng, P.gen_normal_map(rng, vert), prob, inten))
  return np.stack(out)


# (use flags, channels of the 25-channel image, index of nx in the layout or None)
LAYOUTS = {
    'C4': ({}, slice(0, 4), 1),
    'C25': ({'use_class_probabilities': True, 'use_intensity': True}, slice(0, 25), 1),
    'depth_only': ({'use_normals': False}, slice(0, 1), None),
    'normals_only': ({'use_depth': False}, slice(1, 4), 0),
}


@pytest.mark.parametrize('precision', ['fp32', 'f16_tc'])
@pytest.mark.parametrize('layout', sorted(LAYOUTS))
def test_gather_images_is_bit_exact(layout, precision):
  use, chans, c_normal = LAYOUTS[layout]
  x = np.ascontiguousarray(_golden_images()[..., chans])
  if c_normal is not None:                           # every image has fill pixels, which stay (-1, -1, -1)
    assert np.all(np.all(x[..., c_normal:c_normal + 3] == -1, -1).sum((1, 2)) > 0)
  eng = Engine(use=use, model=MODEL, precision=precision, max_batch_scans=4, max_batch_pairs=1)
  assert eng.C == x.shape[-1]
  xs = torch.from_numpy(x).to(eng.device)
  rot = augment.rotation(SHIFTS, 900)
  got = eng.gather_images(xs, _idx(ROWS, eng.device), torch.from_numpy(SHIFTS), torch.from_numpy(rot))
  rolled = eng.gather_images(xs, _idx(ROWS, eng.device), torch.from_numpy(SHIFTS))
  copied = eng.gather_images(xs, _idx(ROWS, eng.device))
  eng.check()
  eng.close()
  assert np.array_equal(bits(got.cpu().numpy()), bits(augment_oracle(x, ROWS, SHIFTS, rot, c_normal)))
  assert np.array_equal(bits(rolled.cpu().numpy()), bits(augment_oracle(x, ROWS, SHIFTS, None, None)))
  assert np.array_equal(bits(copied.cpu().numpy()), bits(x[ROWS]))


def test_gather_images_errors():
  x = np.ascontiguousarray(_golden_images()[..., :4])
  eng = Engine(model=MODEL, precision='fp32', max_batch_scans=4, max_batch_pairs=1)
  dev = eng.device
  xs = torch.from_numpy(x).to(dev)
  bad = ROWS.copy()
  bad[3] = len(x)                                    # one past the image bank
  out = eng.gather_images(xs, _idx(bad, dev), torch.from_numpy(SHIFTS))
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.check()
  out = out.cpu().numpy()                            # clamped to the last row, no out-of-bounds read
  assert np.array_equal(bits(out[3]), bits(np.roll(x[-1], SHIFTS[3], axis=1)))
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.gather_images(xs, _idx(np.zeros(0, np.int32), dev))
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.gather_images(xs[:0], _idx(ROWS, dev))
  eng.gather_images(xs, _idx(ROWS, dev))             # the handle is still healthy
  eng.check()
  eng.close()


# ---- the training steps ----------------------------------------------------------------------------------
N_PAIRS = 4


def _whole_network(eng, images):
  flow = training_leg.WholeNetwork.__new__(training_leg.WholeNetwork)
  flow.eng, flow.images = eng, images
  return flow


def _frozen_leg(eng, images):
  """FrozenLeg with yaw augmentation on a bank encoded from ``images``: every image is also a RIGHT image."""
  flow = training.FrozenLeg.__new__(training.FrozenLeg)
  flow.eng, flow.images = eng, images
  bank = eng.leg(images)
  n, B = len(images), eng.max_batch_scans
  flow.rows = {i: i for i in range(n)}
  flow.bank = torch.cat([bank, bank.new_empty((B,) + tuple(bank.shape[1:]))])
  flow.scratch = torch.arange(n, n + B, dtype=torch.int32, device=eng.device)
  return flow


def _shifts(seed):
  return (np.random.default_rng(seed).integers(1, 180, N_PAIRS) * 5).astype(np.int32)


def _state(eng, loss, kind):
  return loss, eng.get_gradients(eng.layers if kind == 'whole' else HEAD_LAYERS), eng.get_weights()


def _assert_bit_identical(a, b):
  assert a[0] == b[0], (a[0], b[0])
  for part in (1, 2):
    assert sorted(a[part]) == sorted(b[part])
    for name in a[part]:
      for i in range(2):
        assert np.array_equal(bits(a[part][name][i]), bits(b[part][name][i])), (part, name, i)


def _run_step(kind, shifts, lr=1e-4):
  """One augmented step of the flow, and the same step by plain C-ABI calls on oracle-augmented inputs."""
  w, x, _, gt_ov, gt_or = _setup(True)
  n = N_PAIRS
  l, r = LEFT[:n], RIGHT[:n]
  rot = augment.rotation(shifts, 900)
  moved = augment.move_labels(gt_or[:n].astype(np.int64), shifts, 900, 360).astype(np.int32)
  aug = augment_oracle(x, r, shifts, rot, 1)
  out = []
  for plain in (False, True):
    eng = _engine(w)
    dev = eng.device
    xs = torch.from_numpy(x).to(dev)
    if plain:
      if kind == 'whole':
        batch = torch.from_numpy(np.concatenate([x[l], aug])).to(dev)
        pairs = _idx(np.arange(2 * n), dev)
        loss = eng.net_gradients(batch, pairs[:n], pairs[n:], gt_ov[:n], moved, 0.7)
        eng.net_adagrad_step(lr)
      else:
        bank = torch.cat([eng.leg(xs), eng.leg(torch.from_numpy(aug).to(dev))])
        loss = eng.head_gradients(bank, _idx(l, dev), _idx(len(x) + np.arange(n), dev), gt_ov[:n], moved, 0.7)
        eng.adagrad_step(lr)
    else:
      flow = (_whole_network if kind == 'whole' else _frozen_leg)(eng, xs)
      rotate = (_idx(r, dev), torch.from_numpy(shifts).to(dev), torch.from_numpy(rot).to(dev))
      loss = flow.step(_idx(l, dev), _idx(r, dev), torch.from_numpy(gt_ov[:n]).to(dev),
                       torch.from_numpy(moved).to(dev), 0.7, lr, rotate)
    eng.check()
    out.append(_state(eng, loss, kind))
    eng.close()
  return out


def _run_plain_step(kind, lr=1e-4):
  """Today's step without augmentation."""
  w, x, _, gt_ov, gt_or = _setup(True)
  n = N_PAIRS
  eng = _engine(w)
  dev = eng.device
  flow = (_whole_network if kind == 'whole' else _frozen_leg)(eng, torch.from_numpy(x).to(dev))
  loss = flow.step(_idx(LEFT[:n], dev), _idx(RIGHT[:n], dev), torch.from_numpy(gt_ov[:n]).to(dev),
                   torch.from_numpy(gt_or[:n]).to(dev), 0.7, lr)
  out = _state(eng, loss, kind)
  eng.close()
  return out


@pytest.mark.parametrize('kind', ['whole', 'frozen'])
def test_step_with_zero_shifts_equals_the_plain_step(kind):
  zero = np.zeros(N_PAIRS, np.int32)
  augmented, _ = _run_step(kind, zero)
  _assert_bit_identical(augmented, _run_plain_step(kind))


@pytest.mark.parametrize('kind', ['whole', 'frozen'])
def test_step_with_random_shifts_equals_the_step_on_oracle_augmented_inputs(kind):
  augmented, plain = _run_step(kind, _shifts(3))
  _assert_bit_identical(augmented, plain)


def test_augmented_whole_network_gradients_match_float64_autograd():
  """The augmented whole-network step's gradients against the float64 oracle on the oracle-augmented images with
  the moved labels, at the bounds of tests/test_gpu_train_leg.py."""
  w, x, _, gt_ov, gt_or = _setup(True)
  n = N_PAIRS
  l, r = LEFT[:n], RIGHT[:n]
  shifts = _shifts(3)
  rot = augment.rotation(shifts, 900)
  moved = augment.move_labels(gt_or[:n].astype(np.int64), shifts, 900, 360).astype(np.int32)
  aug = augment_oracle(x, r, shifts, rot, 1)
  eng = _engine(w)
  dev = eng.device
  xs = torch.from_numpy(x).to(dev)
  batch = torch.empty((2 * n,) + x.shape[1:], dtype=torch.float32, device=dev)
  eng.gather_images(xs, _idx(l, dev), out=batch[:n])
  eng.gather_images(xs, _idx(r, dev), torch.from_numpy(shifts), torch.from_numpy(rot), out=batch[n:])
  fv = eng.leg(batch).cpu().numpy()
  pairs = _idx(np.arange(2 * n), dev)
  loss = eng.net_gradients(batch, pairs[:n], pairs[n:], gt_ov[:n], moved, 0.7)
  grads = eng.get_gradients(eng.layers)
  eng.close()
  ref_loss, ref, _ = TL.losses_and_gradients(x[l], aug, w, gt_ov[:n], moved, 0.7, MODEL, fv=fv)
  print('losses gpu %s oracle %s' % (loss, ref_loss))
  for got, exp in zip(loss, ref_loss):
    assert abs(got - exp) <= 1e-5 * abs(exp), (loss, ref_loss)
  for name in TL.layer_names(MODEL):
    tol = 1e-4 if name in HEAD_LAYERS else 1e-3
    for i in range(2):
      g, rr = grads[name][i], ref[name][i]
      err = float(np.abs(g - rr).max()) / float(np.abs(rr).max())
      print('%s[%d]: max|g - g_ref| / max|g_ref| = %.2e' % (name, i, err))
      assert np.abs(rr).max() > 0 and err <= tol, (name, i, err)


# ---- the drivers ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('legs', ['360OutputkLegsFixed', '360OutputkLegs'])
def test_training_driver_with_yaw_augmentation(tmp_path, legs):
  root = str(tmp_path / 'data')
  teacher = N.glorot_weights(4, MODEL, seed=0)
  eng = _engine(teacher, maxp=64)
  xs = synth.range_like_images(11, 6, 4)
  fvh = eng.leg(torch.from_numpy(xs).to(eng.device)).cpu().numpy()
  eng.close()
  _, _, _, z = N.heads_forward(fvh[:, None], np.roll(fvh, 1, 0)[:, None], teacher, MODEL, return_logit=True)
  teacher = N.spread_dense(teacher, z, target_std=1.5)
  pretrained = _write_dataset(root, teacher)
  files = []
  for run in range(2):
    cfg = {'experiments_path': str(tmp_path / 'exp'), 'testname': 'run%d' % run,
           'pretrained_weightsfilename': pretrained, 'use_depth': True, 'use_normals': True, 'data_root_folder': root,
           'training_seqs': '00 01', 'batch_size': 8, 'no_batches_in_epoch': 1000, 'no_epochs': 2,
           'no_test_pairs': 1000, 'learning_rate': 1e-4, 'lr_alpha': 0.99, 'min_overlap_for_angle': 0.7,
           'yaw_augmentation': True,
           'model': {'modelType': 'SiameseNetworkTemplate', 'legsType': legs,
                     'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                     'inputShape': [64, 900], 'leg_output_width': 360, **MODEL}}
    np.random.seed(0)
    hist = (training_leg.train if legs == '360OutputkLegs' else training.train)(cfg)
    out = os.path.join(str(tmp_path / 'exp'), 'run%d' % run)
    log = open(os.path.join(out, 'training.log')).read()
    assert 'rotation of training data: RIGHT images by a random multiple of 5 columns (2 bins), labels moved' in log
    assert 'NO rotation' not in log and 'iteration 2, batch/epoch loss' in log
    print(legs, 'epoch losses', hist['epoch_loss'])
    files.append(hist['weights_filename'])
  a, b = Wt.load(files[0]), Wt.load(files[1])
  start = Wt.load(pretrained)
  assert sorted(a) == sorted(b) == sorted(start)
  for name in a:
    for i in range(2):
      assert np.array_equal(bits(a[name][i]), bits(b[name][i])), name
    trained = not np.array_equal(a[name][0], start[name][0])
    assert trained == (legs == '360OutputkLegs' or name in HEAD_LAYERS), name
