"""The calls each training step makes, per configuration: the loop of overlapnet_b200.training on a fake handle and
flow that record, in order, every flow, engine and gradient-gather call, on one process and on two gloo ranks, plain,
with yaw augmentation and with gradient chunks.

  one process, no chunks   flow.step
  ranks, no chunks         flow.gradients + eng.copy_gradients (nothing for an empty share), dp.gather_flat,
                           eng.adagrad_step_sum over the ranks' shares
  gradient_chunks K        flow.gradients(chunks=...) (nothing for an empty range), with ranks dp.gather_flat, then
                           eng.adagrad_step_sum over the K chunks in chunk order
"""
import os
import pickle
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT  # noqa: F401
from overlapnet_b200 import data_parallel, training

CALLS = []                   # what the fakes of this process were called with, in order
N_PAIRS = 11                 # batches of 5, 5 and 1 pairs: the last one leaves rank 1 no pairs, with or without chunks
CONFIGS = {'plain': {}, 'yaw': {'yaw_augmentation': True}, 'chunks': {'gradient_chunks': 3}}


class _Engine:
  device = torch.device('cpu')
  W = 900

  def get_weights(self):
    return {'w': (np.zeros(3, np.float32), np.zeros(1, np.float32))}

  def load_weights(self, w):
    pass

  def check(self):
    pass

  def gradient_size(self, whole_network=False):
    return 2

  def copy_gradients(self, whole_network=False, out=None):
    CALLS.append(('copy_gradients', whole_network))
    out.fill_(self.last)
    return out

  def adagrad_step_sum(self, parts, weights, lr, whole_network=False):
    CALLS.append(('adagrad_step_sum', list(weights), parts[:, 0].tolist(), whole_network))


class _Infer:
  def __init__(self, cfg, precision, device, max_batch_pairs):
    self._engine = _Engine()
    self.network_output_size = cfg['model']['leg_output_width']


class _Flow:
  """A part's gradient is its pair count, so that the parts the sum receives show which pairs each one covers."""
  whole_network = True

  def __init__(self, infer, keys, rotate_keys=None, gradient_chunks=None):
    self.eng = infer._engine
    self.rows = {k: i for i, k in enumerate(sorted(keys))}
    self.image_rows = {k: 100 + i for i, k in enumerate(sorted(rotate_keys or ()))}

  def step(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, lr, rotate=None):
    CALLS.append(('step', left.numel(), None if rotate is None else rotate[0].numel()))
    return (1.0, 0.5, 0.5)

  def gradients(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate=None, chunks=None):
    CALLS.append(('gradients', left.numel(), None if rotate is None else rotate[0].numel(),
                  None if chunks is None else list(chunks[0])))
    if chunks is None:
      self.eng.last = float(left.numel())
      return (1.0, 0.5, 0.5)
    offsets, parts = chunks
    for c in range(len(offsets) - 1):
      parts[c] = float(offsets[c + 1] - offsets[c])
    return [(1.0, 0.5, 0.5)] * (len(offsets) - 1)

  def evaluate(self, left, right):
    CALLS.append(('evaluate',))
    return 0.3 + left.float() / 20, (180 - right).to(torch.int32)


def _write_files(tmp):
  table = np.array([[i, (i + 1 + i // 6) % 7, 0.5, (37 * i) % 360] for i in range(N_PAIRS)], float)
  np.savez(os.path.join(tmp, 'train.npz'), overlaps=table, seq=np.array([['00', '00']] * N_PAIRS))
  np.savez(os.path.join(tmp, 'val.npz'), overlaps=table[:3], seq=np.array([['00', '00']] * 3))


def _run(tmp, dp, name):
  """training._train on the fakes after np.random.seed(7); the calls it made."""
  cfg = dict({'experiments_path': tmp, 'testname': name, 'pretrained_weightsfilename': '',
              'traindata_npzfile': os.path.join(tmp, 'train.npz'),
              'validationdata_npzfile': os.path.join(tmp, 'val.npz'), 'batch_size': 5, 'no_batches_in_epoch': 3,
              'no_epochs': 2, 'no_test_pairs': 3, 'learning_rate': 1e-3,
              'model': {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
                        'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                        'inputShape': [64, 900], 'leg_output_width': 360}}, **CONFIGS[name])
  save = training.save_weights
  training.save_weights = lambda path, w: None
  del CALLS[:]
  try:
    np.random.seed(7)
    training._train(cfg, cfg['model'], '', tmp, None, _Infer, _Flow, dp=dp)
  finally:
    training.save_weights = save
  return list(CALLS)


def _expected_step(n, world, rank, chunks, rotate):
  """The calls of one step of an n-pair batch on ``rank`` of ``world``."""
  if world == 1 and chunks is None:
    return [('step', n, n if rotate else None)]
  if chunks is None:
    bounds, weights = data_parallel.shares(n, world)
    lo, hi = bounds[rank]
    calls = [('gradients', hi - lo, hi - lo if rotate else None, None), ('copy_gradients', True)] if hi > lo else []
  else:
    bounds, weights, (c0, c1), (lo, hi) = data_parallel.chunk_plan(n, chunks, world, rank)
    offsets = [bounds[c][0] - lo for c in range(c0, c1)] + [hi - lo]
    calls = [('gradients', hi - lo, hi - lo if rotate else None, offsets)] if hi > lo else []
  if world > 1:
    calls.append(('gather_flat',))
  return calls + [('adagrad_step_sum', weights, [float(hi - lo) for lo, hi in bounds], True)]


def _check(calls, sizes, world, rank, name):
  chunks = CONFIGS[name].get('gradient_chunks')
  want = []
  for epoch in range(2):
    for n in sizes[3 * epoch:3 * epoch + 3]:
      want += _expected_step(n, world, rank, chunks, name == 'yaw')
    want.append(('evaluate',))
  assert calls == want, (name, world, rank)


def _batch_sizes(calls):
  """The batch size of each step of a one-process run without chunks: two epochs of 5, 5 and 1 pairs."""
  sizes = [c[1] for c in calls if c[0] == 'step']
  assert sorted(sizes[:3]) == sorted(sizes[3:]) == [1, 5, 5]
  return sizes


def test_one_process_step_calls(tmp_path):
  tmp = str(tmp_path)
  _write_files(tmp)
  for name in CONFIGS:
    calls = _run(tmp, None, name)
    sizes = _batch_sizes(calls if name != 'chunks' else _run(tmp, None, 'plain'))
    _check(calls, sizes, 1, 0, name)


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _worker(rank, world, port, tmp):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  try:
    dp = data_parallel.default_group()
    gather_flat = dp.gather_flat

    def recorded(flat, out):
      CALLS.append(('gather_flat',))
      return gather_flat(flat, out)

    dp.gather_flat = recorded
    res = {name: _run(tmp, dp, name) for name in CONFIGS}
    with open(os.path.join(tmp, 'rank%d.pkl' % rank), 'wb') as f:
      pickle.dump(res, f)
  finally:
    dist.destroy_process_group()


def test_two_rank_step_calls(tmp_path):
  tmp = str(tmp_path)
  _write_files(tmp)
  mp.spawn(_worker, args=(2, _free_port(), tmp), nprocs=2, join=True)
  # rank 0 makes the draws of one process, so the batches come in the one-process order
  sizes = {name: _batch_sizes(_run(tmp, None, 'yaw' if name == 'yaw' else 'plain')) for name in CONFIGS}
  for rank in range(2):
    with open(os.path.join(tmp, 'rank%d.pkl' % rank), 'rb') as f:
      res = pickle.load(f)
    for name in CONFIGS:
      _check(res[name], sizes[name], 2, rank, name)
  # the last batch's single pair leaves rank 1 nothing to compute, with and without chunks
  assert 1 in sizes['plain'] and data_parallel.shares(1, 2)[0][1] == (1, 1)
  assert data_parallel.chunk_plan(1, 3, 2, 1)[3] == (1, 1)
