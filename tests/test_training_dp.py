"""CPU checks of data-parallel training (overlapnet_b200.data_parallel): the shares of a batch, and the training
loop of overlapnet_b200.training on two gloo ranks with a fake handle and flow against the one-process loop."""
import os
import pickle
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT  # noqa: F401
from overlapnet_b200 import augment, data_parallel, training


def test_shares_partition_each_batch_in_rank_order():
  for n in range(1, 21):
    for world in range(1, 5):
      bounds, weights = data_parallel.shares(n, world)
      assert bounds[0][0] == 0 and bounds[-1][1] == n
      assert all(bounds[r][1] == bounds[r + 1][0] for r in range(world - 1))
      assert all(hi - lo <= -(-n // world) for lo, hi in bounds)                 # at most ceil(n / world)
      assert sum(weights) == pytest.approx(1.0, abs=1e-15)
      for (lo, hi), w in zip(bounds, weights):
        assert w == (hi - lo) / n and (w == 0) == (hi == lo)
  assert data_parallel.shares(1, 2) == ([(0, 1), (1, 1)], [1.0, 0.0])
  assert data_parallel.default_group() is None                                  # no process group here


# ---- the loop on fakes ---------------------------------------------------------------------------------------
class _Engine:
  device = torch.device('cpu')
  W = 900

  def __init__(self):
    self.loaded, self.sums, self.last = [], [], None

  def get_weights(self):
    return {'w': (np.arange(3, dtype=np.float32) + 7, np.zeros(1, np.float32))}

  def load_weights(self, w):
    self.loaded.append(w)

  def check(self):
    pass

  def gradient_size(self, whole_network=False):
    return 4

  def copy_gradients(self, whole_network=False, out=None):
    out.copy_(self.last)
    return out

  def adagrad_step_sum(self, parts, weights, lr, whole_network=False):
    self.sums.append((parts.numpy().copy(), list(weights), lr, whole_network))


class _Infer:
  def __init__(self, cfg, precision, device, max_batch_pairs):
    self._engine = _Engine()
    self.network_output_size = cfg['model']['leg_output_width']


class _Flow:
  """Records what the loop hands to each step; the 'gradients' of a share reveal its pairs and labels."""
  whole_network = True

  def __init__(self, infer, keys, rotate_keys=None):
    self.eng = infer._engine
    self.rows = {k: i for i, k in enumerate(sorted(keys))}
    self.image_rows = {k: 100 + i for i, k in enumerate(sorted(rotate_keys or ()))}
    self.calls = []
    _Flow.instance = self

  def gradients(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate=None):
    rot = None if rotate is None else tuple(t.numpy().copy() for t in rotate)
    self.calls.append((left.numpy().copy(), right.numpy().copy(), gt_orientation.numpy().copy(), rot))
    self.eng.last = torch.tensor([left.sum(), right.sum(), gt_orientation.sum(), left.numel()], dtype=torch.float32)
    return (float(left.sum()) + 0.5, float(right.sum()), float(left.numel()))

  def step(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, lr, rotate=None):
    return self.gradients(left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate)

  def evaluate(self, left, right):
    return 0.3 + left.float() / 20, (180 - right).to(torch.int32)


N_PAIRS = 11                 # batches of 5, 5 and 1 pairs: the last one leaves rank 1 an empty share


def _write_files(tmp):
  table = np.array([[i, (i + 1 + i // 6) % 7, 0.5, (37 * i) % 360] for i in range(N_PAIRS)], float)
  np.savez(os.path.join(tmp, 'train.npz'), overlaps=table, seq=np.array([['00', '00']] * N_PAIRS))
  np.savez(os.path.join(tmp, 'val.npz'), overlaps=table[:3], seq=np.array([['00', '00']] * 3))


def _run(tmp, on, dp):
  cfg = {'experiments_path': tmp, 'testname': 't', 'pretrained_weightsfilename': '',
         'traindata_npzfile': os.path.join(tmp, 'train.npz'), 'validationdata_npzfile': os.path.join(tmp, 'val.npz'),
         'batch_size': 5, 'no_batches_in_epoch': 3, 'no_epochs': 2, 'no_test_pairs': 3, 'learning_rate': 1e-3,
         'yaw_augmentation': on,
         'model': {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
                   'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                   'inputShape': [64, 900], 'leg_output_width': 360}}
  saves = []
  save = training.save_weights
  training.save_weights = lambda path, w: saves.append(path)
  try:
    np.random.seed(7)
    hist = training._train(cfg, cfg['model'], '', tmp, None, _Infer, _Flow, dp=dp)
  finally:
    training.save_weights = save
  flow = _Flow.instance
  return {'state': np.random.get_state()[1].copy(), 'calls': flow.calls, 'sums': flow.eng.sums,
          'loaded': flow.eng.loaded, 'hist': hist, 'saves': saves}


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _worker(rank, world, port, tmp, on):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  try:
    dp = data_parallel.default_group()
    assert dp is not None and (dp.rank, dp.world, dp.nccl) == (rank, world, False)
    res = _run(tmp, on, dp)
    with open(os.path.join(tmp, 'rank%d.pkl' % rank), 'wb') as f:
      pickle.dump(res, f)
  finally:
    dist.destroy_process_group()


@pytest.mark.parametrize('on', [False, True])
def test_two_rank_loop_makes_the_one_process_steps(tmp_path, on):
  tmp = str(tmp_path)
  _write_files(tmp)
  mp.spawn(_worker, args=(2, _free_port(), tmp, on), nprocs=2, join=True)
  ranks = []
  for r in range(2):
    with open(os.path.join(tmp, 'rank%d.pkl' % r), 'rb') as f:
      ranks.append(pickle.load(f))
  one = _run(tmp, on, None)

  # rank 0 makes exactly the draws of one process; the other ranks receive its results
  assert np.array_equal(ranks[0]['state'], one['state'])
  # one start: rank 1 takes rank 0's initial weights
  assert ranks[0]['loaded'] == [] and len(ranks[1]['loaded']) == 1
  assert np.array_equal(ranks[1]['loaded'][0]['w'][0], _Engine().get_weights()['w'][0])
  # only rank 0 writes the weight file, once per epoch like one process
  assert len(ranks[0]['saves']) == len(one['saves']) == 2 and ranks[1]['saves'] == []

  # per step: the ranks' shares, concatenated in rank order, are the one-process step (pairs, labels moved by the
  # same shifts, the same rotations)
  steps = one['calls']
  assert len(steps) == 6 and len(ranks[0]['sums']) == len(ranks[1]['sums']) == 6
  calls = [list(ranks[0]['calls']), list(ranks[1]['calls'])]
  batch_losses = []
  for i, (left, right, gt_or, rot) in enumerate(steps):
    m = len(left)
    bounds, weights = data_parallel.shares(m, 2)
    got = [calls[r].pop(0) if hi > lo else None for r, (lo, hi) in enumerate(bounds)]
    assert [c is not None for c in got] == [True, m > 1]
    got = [c for c in got if c is not None]
    for k in range(3):
      assert np.array_equal(np.concatenate([c[k] for c in got]), (left, right, gt_or)[k]), (i, k)
    assert (rot is None) == (not on)
    if on:
      for k in range(3):
        assert np.array_equal(np.concatenate([c[3][k] for c in got]), rot[k]), (i, k)
      assert np.array_equal(rot[2], augment.rotation(rot[1], 900))
    # both ranks apply the same sum: row r is rank r's gradients (zero for an empty share), weights n_r / n
    for r in range(2):
      parts, w, lr, whole = ranks[r]['sums'][i]
      assert w == weights and whole is True and lr == one['hist']['validation'][i // 3]['learning_rate']
      for rr, c in enumerate(got + [None] * (2 - len(got))):
        want = [0, 0, 0, 0] if c is None else [c[0].sum(), c[1].sum(), c[2].sum(), len(c[0])]
        assert np.array_equal(parts[rr], np.asarray(want, np.float32)), (i, r, rr)
    # the logged loss is sum_r w_r loss_r
    per_rank = [(float(c[0].sum()) + 0.5, float(c[1].sum()), float(len(c[0]))) for c in got] + [(0.0, 0.0, 0.0)]
    batch_losses.append(float(sum(w * l[0] for w, l in zip(weights, per_rank))))
  assert calls == [[], []]
  for r in range(2):
    assert ranks[r]['hist']['batch_losses'] == [batch_losses[:3], batch_losses[3:]]
    # validation: each rank scores a share, the results are gathered in rank order
    assert repr(ranks[r]['hist']['validation']) == repr(one['hist']['validation'])
    assert ranks[r]['hist']['epoch_loss'] == ranks[0]['hist']['epoch_loss']
