"""The 3xTF32 arithmetic of training precision tf32x3 restated in NumPy (the rounding of cvt.rna.tf32.f32, the
split, three products per step with fp32 accumulation) against float64, the ``training_precision`` config key of
both flows, and what the training loop calls with and without it (on fakes, one process and two gloo ranks)."""
import os
import pickle
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT  # noqa: F401
from overlapnet_b200 import data_parallel, training, training_leg


# ---- the arithmetic ------------------------------------------------------------------------------------------
def tf32_rna(x):
  """cvt.rna.tf32.f32: float32 rounded to a 10-bit mantissa, ties away from zero (the float32 bit pattern is
  sign-magnitude, so adding half a TF32 ulp to the magnitude bits and truncating rounds half away from zero)."""
  b = np.ascontiguousarray(x, np.float32).view(np.uint32)
  return ((b + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32)


def split(x):
  x = np.asarray(x, np.float32)
  hi = tf32_rna(x)
  return hi, tf32_rna(x - hi)


def _mma(acc, lhs, rhs):
  """One m16n8k8 per output element: the eight products (exact: two 11-bit significands) added to the float32
  accumulator and truncated to float32 (the tensor core rounds toward zero there)."""
  s = acc.astype(np.float64) + lhs.astype(np.float64) @ rhs.astype(np.float64)
  f = s.astype(np.float32)
  over = np.abs(f.astype(np.float64)) > np.abs(s)
  f[over] = np.nextafter(f[over], np.float32(0))
  return f


def gemm_3xtf32(a, b, per_tile=True):
  """C = A B as k_tc_gemm forms it: per K8 step three MMAs, lo_a hi_b, hi_a lo_b, then hi_a hi_b.  per_tile: the six
  MMAs of each K16 tile start from zero and their partial is added to the float32 sum with round-to-nearest (the
  kernel); else every MMA accumulates into the running sum."""
  ah, al = split(a)
  bh, bl = split(b)
  acc = np.zeros((a.shape[0], b.shape[1]), np.float32)
  for k0 in range(0, a.shape[1], 16):
    part = np.zeros_like(acc) if per_tile else acc
    for k8 in (k0, k0 + 8):
      ks = slice(k8, k8 + 8)
      for lhs, rhs in ((al, bh), (ah, bl), (ah, bh)):
        part = _mma(part, lhs[:, ks], rhs[ks])
    acc = acc + part if per_tile else part
  return acc


def gemm_tf32(a, b):
  """One-pass TF32, per K16 tile like gemm_3xtf32."""
  ah, bh = tf32_rna(a), tf32_rna(b)
  acc = np.zeros((a.shape[0], b.shape[1]), np.float32)
  for k0 in range(0, a.shape[1], 16):
    part = _mma(_mma(np.zeros_like(acc), ah[:, k0:k0 + 8], bh[k0:k0 + 8]), ah[:, k0 + 8:k0 + 16], bh[k0 + 8:k0 + 16])
    acc = acc + part
  return acc


def test_tf32_rounding_is_nearest_ties_away():
  one_ulp = np.float32(2.0 ** -10)
  x = np.array([1.0, 1.0 + one_ulp / 2, -(1.0 + one_ulp / 2), 1.0 + one_ulp / 2 - 2.0 ** -23, 3.0 + 2.0 ** -12],
               np.float32)
  assert tf32_rna(x).tolist() == [1.0, 1.0 + one_ulp, -(1.0 + one_ulp), 1.0, 3.0]
  r = np.random.default_rng(0).standard_normal(100000).astype(np.float32)
  assert not (tf32_rna(r).view(np.uint32) & np.uint32(0x1fff)).any()
  assert float(np.abs((tf32_rna(r) - r) / r).max()) <= 2.0 ** -11


def test_split_keeps_22_bits_and_products_are_exact():
  rng = np.random.default_rng(1)
  x = (rng.standard_normal(200000) * np.exp(rng.uniform(-20, 20, 200000))).astype(np.float32)
  hi, lo = split(x)
  assert not ((hi.view(np.uint32) | lo.view(np.uint32)) & np.uint32(0x1fff)).any()
  rel = np.abs(hi.astype(np.float64) + lo - x) / np.abs(x)
  print('max |x - hi - lo| / |x| = %.2e (2^-22 = %.2e)' % (rel.max(), 2.0 ** -22))
  assert rel.max() <= 2.0 ** -22
  y = np.roll(hi, 1)
  assert np.array_equal((hi * y).astype(np.float64), hi.astype(np.float64) * y.astype(np.float64))


@pytest.mark.parametrize('m,k,n', [(64, 256, 64), (37, 1920, 29), (64, 4096, 8)])
def test_3xtf32_product_is_fp32_grade(m, k, n):
  """Random normal matrices: 3xTF32 stays within 2e-6 of the float64 product (relative to its largest
  element), like plain fp32 accumulation; one-pass TF32 is about 1e-3 off."""
  rng = np.random.default_rng(m * k + n)
  a = rng.standard_normal((m, k)).astype(np.float32)
  b = rng.standard_normal((k, n)).astype(np.float32)
  ref = a.astype(np.float64) @ b.astype(np.float64)
  scale = float(np.abs(ref).max())
  fp32 = np.zeros((m, n), np.float32)
  for kk in range(k):
    fp32 = fp32 + np.outer(a[:, kk], b[kk]).astype(np.float32)
  e3 = float(np.abs(gemm_3xtf32(a, b) - ref).max()) / scale
  e32 = float(np.abs(fp32 - ref).max()) / scale
  e1 = float(np.abs(gemm_tf32(a, b) - ref).max()) / scale
  print('%d x %d x %d: 3xTF32 %.2e, fp32 %.2e, one-pass TF32 %.2e' % (m, k, n, e3, e32, e1))
  assert e3 <= 2e-6 and e3 <= 2 * e32
  assert 1e-4 <= e1 <= 3e-3


def test_per_tile_partials_stop_the_truncation_drift():
  """Non-negative operands (ReLU outputs, |l - r|) at c_conv1's K = 1920: one truncating accumulator over all 720
  MMAs drifts toward zero by far more than fp32's rounding; the kernel's per-K16 partials do not."""
  rng = np.random.default_rng(3)
  a = rng.uniform(0, 1, (16, 1920)).astype(np.float32)
  b = rng.uniform(0, 1, (1920, 8)).astype(np.float32)
  ref = a.astype(np.float64) @ b.astype(np.float64)
  tile = float(np.abs(gemm_3xtf32(a, b) - ref).max() / np.abs(ref).max())
  chain = float(np.abs(gemm_3xtf32(a, b, per_tile=False) - ref).max() / np.abs(ref).max())
  print('K = 1920, non-negative: per-tile partials %.2e, one accumulator %.2e' % (tile, chain))
  assert tile <= 1e-6 and chain >= 10 * tile


# ---- the config key ------------------------------------------------------------------------------------------
def _config(tmp_path, legs, **kw):
  cfg = {'experiments_path': str(tmp_path), 'testname': 't', 'pretrained_weightsfilename': '',
         'traindata_npzfile': 'x', 'validationdata_npzfile': 'y', 'batch_size': 2, 'no_batches_in_epoch': 1,
         'no_epochs': 1, 'no_test_pairs': 1, 'learning_rate': 1e-3,
         'model': {'modelType': 'SiameseNetworkTemplate', 'legsType': legs,
                   'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                   'inputShape': [64, 900], 'leg_output_width': 360}}
  cfg.update(kw)
  return cfg


FLOWS = [('360OutputkLegsFixed', training), ('360OutputkLegs', training_leg)]


@pytest.mark.parametrize('legs,module', FLOWS)
def test_both_flows_accept_the_key(tmp_path, legs, module):
  module.check_config(_config(tmp_path, legs))
  for p in ('fp32', 'tf32x3'):
    module.check_config(_config(tmp_path, legs, training_precision=p))
  module.check_config(_config(tmp_path, legs, training_precision='tf32x3', yaw_augmentation=True))


@pytest.mark.parametrize('legs,module', FLOWS)
@pytest.mark.parametrize('value', ['tf32', 'f16_tc', 'TF32X3', 1, None])
def test_other_values_are_refused(tmp_path, legs, module, value):
  cfg = _config(tmp_path, legs, training_precision=value)
  with pytest.raises(Exception, match='training_precision.*fp32, tf32x3'):
    module.check_config(cfg)
  with pytest.raises(Exception, match='training_precision'):
    module.train(cfg)                               # refused before any file or device is touched
  assert not os.path.exists(os.path.join(str(tmp_path), 't'))


# ---- the loop on fakes ---------------------------------------------------------------------------------------
class _Engine:
  device = torch.device('cpu')
  W = 900

  def __init__(self, events):
    self.events = events

  def set_train_precision(self, p):
    self.events.append(('set_train_precision', p))

  def get_weights(self):
    return {'w': (np.arange(3, dtype=np.float32), np.zeros(1, np.float32))}

  def load_weights(self, w):
    self.events.append(('load_weights',))

  def check(self):
    pass

  def gradient_size(self, whole_network=False):
    return 2

  def copy_gradients(self, whole_network=False, out=None):
    out.fill_(1.0)
    return out

  def adagrad_step_sum(self, parts, weights, lr, whole_network=False):
    self.events.append(('adagrad_step_sum', list(weights), lr))


class _Infer:
  events = None

  def __init__(self, cfg, precision, device, max_batch_pairs):
    self.events.append(('infer', precision, max_batch_pairs))
    self._engine = _Engine(self.events)
    self.network_output_size = cfg['model']['leg_output_width']


class _Flow:
  whole_network = True

  def __init__(self, infer, keys, rotate_keys=None):
    self.events = infer._engine.events
    self.rows = {k: i for i, k in enumerate(sorted(keys))}
    self.image_rows = {k: 100 + i for i, k in enumerate(sorted(rotate_keys or ()))}
    self.events.append(('flow', rotate_keys is not None))

  def gradients(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate=None):
    self.events.append(('gradients', left.tolist(), right.tolist(), gt_orientation.tolist(),
                        None if rotate is None else rotate[1].tolist()))
    return (1.0, 0.5, 0.5)

  def step(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, lr, rotate=None):
    loss = self.gradients(left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate)
    self.events.append(('step', lr))
    return loss

  def evaluate(self, left, right):
    self.events.append(('evaluate', left.tolist()))
    return torch.zeros(left.numel()), torch.full((left.numel(),), 180, dtype=torch.int32)


def _write_files(tmp):
  table = np.array([[i, (i + 1 + i // 6) % 7, 0.5, (37 * i) % 360] for i in range(11)], float)
  np.savez(os.path.join(tmp, 'train.npz'), overlaps=table, seq=np.array([['00', '00']] * 11))
  np.savez(os.path.join(tmp, 'val.npz'), overlaps=table[:3], seq=np.array([['00', '00']] * 3))


def _run(tmp, dp, **kw):
  """training._train on the fakes; returns the events and numpy's random state after the loop."""
  cfg = _config(tmp, '360OutputkLegs', traindata_npzfile=os.path.join(tmp, 'train.npz'),
                validationdata_npzfile=os.path.join(tmp, 'val.npz'), batch_size=5, no_batches_in_epoch=3,
                no_epochs=2, no_test_pairs=3, **kw)
  save = training.save_weights
  training.save_weights = lambda path, w: None
  _Infer.events = []
  try:
    np.random.seed(7)
    training._train(cfg, cfg['model'], '', tmp, None, _Infer, _Flow, dp=dp)
  finally:
    training.save_weights = save
  return _Infer.events, np.random.get_state()[1].copy()


def _without_precision(events):
  return [e for e in events if e[0] != 'set_train_precision']


@pytest.mark.parametrize('yaw', [False, True])
def test_loop_sets_the_precision_once_before_the_first_step(tmp_path, caplog, yaw):
  import logging
  caplog.set_level(logging.INFO, logger='overlapnet_b200.training')
  tmp = str(tmp_path)
  _write_files(tmp)
  base, state = _run(tmp, None, yaw_augmentation=yaw)
  assert 'Training precision' not in caplog.text
  assert not any(e[0] == 'set_train_precision' for e in base)      # no key: today's calls only
  caplog.clear()
  events, state_tc = _run(tmp, None, yaw_augmentation=yaw, training_precision='tf32x3')
  assert 'Training precision: tf32x3' in caplog.text
  sets = [i for i, e in enumerate(events) if e[0] == 'set_train_precision']
  assert [events[i] for i in sets] == [('set_train_precision', 'tf32x3')]
  assert events[sets[0] - 1][0] == 'infer' and events[sets[0] - 1][1] == 'fp32'
  assert sets[0] < min(i for i, e in enumerate(events) if e[0] in ('flow', 'gradients'))
  # the key adds that call and nothing else: the same steps, labels, rotations and random draws
  assert _without_precision(events) == base
  assert np.array_equal(state, state_tc)
  explicit, _ = _run(tmp, None, yaw_augmentation=yaw, training_precision='fp32')
  assert [e for e in explicit if e[0] == 'set_train_precision'] == [('set_train_precision', 'fp32')]


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _worker(rank, world, port, tmp, kw):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  try:
    res = _run(tmp, data_parallel.default_group(), **kw)
    with open(os.path.join(tmp, 'rank%d.pkl' % rank), 'wb') as f:
      pickle.dump(res, f)
  finally:
    dist.destroy_process_group()


@pytest.mark.parametrize('key', [False, True])
def test_every_rank_sets_the_precision_before_its_first_step(tmp_path, key):
  tmp = str(tmp_path)
  _write_files(tmp)
  kw = {'yaw_augmentation': True}
  if key:
    kw['training_precision'] = 'tf32x3'
  mp.spawn(_worker, args=(2, _free_port(), tmp, kw), nprocs=2, join=True)
  ranks = []
  for r in range(2):
    with open(os.path.join(tmp, 'rank%d.pkl' % r), 'rb') as f:
      ranks.append(pickle.load(f))
  for events, _ in ranks:
    sets = [i for i, e in enumerate(events) if e[0] == 'set_train_precision']
    assert [events[i] for i in sets] == ([('set_train_precision', 'tf32x3')] if key else [])
    if key:
      assert sets[0] < min(i for i, e in enumerate(events) if e[0] in ('load_weights', 'flow', 'gradients'))
  if key:             # the same calls and draws as without the key
    kw.pop('training_precision')
    mp.spawn(_worker, args=(2, _free_port(), tmp, kw), nprocs=2, join=True)
    for r in range(2):
      with open(os.path.join(tmp, 'rank%d.pkl' % r), 'rb') as f:
        events, state = pickle.load(f)
      assert _without_precision(ranks[r][0]) == events
      assert np.array_equal(ranks[r][1], state)
