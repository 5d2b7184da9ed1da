"""Gradients per chunk of a batch (``gradient_chunks``) on the GPU: ovn_head_gradients_chunks /
ovn_net_gradients_chunks against one-chunk calls, their errors and what the handle keeps after them; K = 1 against
the run without the key; and runs with K = 4 that give the same bits on one process, two and three ranks (gloo on
one GPU), also when resumed on another world size."""
import copy
import os
import pickle

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from overlapnet_b200 import training
from overlapnet_b200 import weights as Wt
from overlapnet_b200._cabi import OvnError
from test_gpu_train_dp import FLOWS, _config, _free_port, dataset  # noqa: F401  (dataset is a fixture)
from test_gpu_train_leg import LEFT, RIGHT, _engine, _idx, _setup

pytestmark = pytest.mark.gpu

OFFSETS = [0, 3, 3, 5, 7]            # 7 pairs in chunks of 3, 0, 2 and 2


def bits(a):
  return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _one_chunk(eng, whole, rows, li, ri, gt_ov, gt_or, a, b):
  if whole:
    loss = eng.net_gradients(rows, li[a:b], ri[a:b], gt_ov[a:b], gt_or[a:b], 0.7)
  else:
    loss = eng.head_gradients(rows, li[a:b], ri[a:b], gt_ov[a:b], gt_or[a:b], 0.7)
  return np.asarray(loss, np.float32), eng.copy_gradients(whole).cpu().numpy()


def _chunks(eng, whole, rows, li, ri, offsets, gt_ov, gt_or):
  fn = eng.net_gradients_chunks if whole else eng.head_gradients_chunks
  return fn(rows, li, ri, offsets, gt_ov, gt_or, 0.7)


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('kind', ['frozen', 'whole'])
def test_each_part_is_the_one_chunk_call(kind, precision):
  w, x, _, gt_ov, gt_or = _setup(True)
  whole = kind == 'whole'
  eng = _engine(w)
  eng.set_train_precision(precision)
  dev = eng.device
  xs = torch.from_numpy(x).to(dev)
  rows = xs if whole else eng.leg(xs)
  n = OFFSETS[-1]
  li, ri = _idx(LEFT[:n], dev), _idx(RIGHT[:n], dev)
  for offsets in (OFFSETS, [0, n]):
    losses, parts = _chunks(eng, whole, rows, li, ri, offsets, gt_ov[:n], gt_or[:n])
    parts = parts.cpu().numpy()
    assert parts.shape == (len(offsets) - 1, eng.gradient_size(whole)) and len(losses) == len(offsets) - 1
    for c in range(len(offsets) - 1):
      a, b = offsets[c], offsets[c + 1]
      if a == b:
        assert not parts[c].any() and losses[c] == (0.0, 0.0, 0.0), c
        continue
      loss, g = _one_chunk(eng, whole, rows, li, ri, gt_ov, gt_or, a, b)
      assert np.array_equal(bits(losses[c]), bits(loss)), (offsets, c)
      assert np.array_equal(bits(parts[c]), bits(g)), (offsets, c)
      assert g.any()
  eng.check()
  eng.close()


@pytest.mark.parametrize('kind', ['frozen', 'whole'])
def test_errors_and_what_the_handle_keeps(kind):
  """The refusals, and after a chunked call: no gradients and no batch in the handle, until a one-chunk call."""
  w, x, _, gt_ov, gt_or = _setup(True)
  whole = kind == 'whole'
  eng = _engine(w)
  dev = eng.device
  xs = torch.from_numpy(x).to(dev)
  rows = xs if whole else eng.leg(xs)
  n = 7
  li, ri = _idx(LEFT[:n], dev), _idx(RIGHT[:n], dev)
  args = (eng, whole, rows, li, ri)
  before = eng.get_weights()
  for offsets, status in (([0], 'OVN_ERR_INVALID_ARG.*n_chunks'),
                          ([0] * 59 + list(range(1, 8)), 'OVN_ERR_CAPACITY.*n_chunks'),
                          ([0, 3, 6], 'OVN_ERR_INVALID_ARG.*from 0 to n_pairs'),
                          ([1, 3, 7], 'OVN_ERR_INVALID_ARG.*from 0 to n_pairs'),
                          ([0, 4, 3, 7], 'OVN_ERR_INVALID_ARG.*below offset')):
    with pytest.raises(OvnError, match=status):
      _chunks(*args, offsets, gt_ov[:n], gt_or[:n])
  bad = _idx(np.where(np.arange(n) == 4, 99, LEFT[:n]), dev)         # the one-chunk calls' errors
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    _chunks(eng, whole, rows, bad, ri, OFFSETS, gt_ov[:n], gt_or[:n])
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG.*positive'):
    _chunks(eng, whole, rows, li[:0], ri[:0], [0, 0], gt_ov[:0], gt_or[:0])
  _one_chunk(eng, whole, rows, li, ri, gt_ov, gt_or, 0, 4)          # valid gradients and a batch ...
  _chunks(*args, OFFSETS, gt_ov[:n], gt_or[:n])                      # ... which a chunked call does not keep
  for call in ([lambda: eng.copy_gradients(False), lambda: eng.copy_gradients(True), lambda: eng.adagrad_step(1e-3),
                lambda: eng.net_adagrad_step(1e-3), lambda: eng.net_volumes(),
                lambda: eng.get_gradients(('c_conv1',))]):
    with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
      call()
  after = eng.get_weights()
  for name in before:
    for i in range(2):
      assert np.array_equal(bits(before[name][i]), bits(after[name][i])), name
  _one_chunk(eng, whole, rows, li, ri, gt_ov, gt_or, 0, 4)          # a one-chunk call works as before
  eng.check()
  eng.close()


# ---- the training loop ------------------------------------------------------------------------------------
def _cfg(root, pretrained, exp, name, legs, yaw, precision='fp32', **keys):
  cfg = _config(root, pretrained, exp, name, legs, yaw)
  # 38 training pairs in batches of 12: the last batch has 2 pairs, so with K = 4 its last two chunks are empty
  cfg.update(dict({'batch_size': 12, 'no_epochs': 3, 'training_precision': precision}, **keys))
  return cfg


def _train(cfg, image_bank=None, device=None):
  """One run: its history and the handle's weights and Adagrad state at the end."""
  module, name, train = FLOWS[cfg['model']['legsType']]
  base = getattr(module, name)
  kept = []

  class Keep(base):
    def __init__(self, *args, **kw):
      if image_bank is not None:
        kw['image_bank'] = image_bank
      super().__init__(*args, **kw)
      kept.append(self)

  setattr(module, name, Keep)
  try:
    hist = train(copy.deepcopy(cfg), device)
  finally:
    setattr(module, name, base)
  eng = kept[0].eng
  out = {'hist': hist, 'weights': eng.get_weights(), 'state': eng.train_state(base.whole_network).cpu().numpy()}
  eng.close()
  return out


def _worker(rank, world, port, cfg, image_bank, out):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(0)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  try:
    np.random.seed(0)
    run = _train(cfg, image_bank, 0)
    with open(out % rank, 'wb') as f:
      pickle.dump(run, f)
  finally:
    dist.destroy_process_group()


def _run(tmp_path, cfg, world, image_bank=None):
  """A run on one process (world 1) or on ``world`` gloo ranks sharing the GPU; rank 0's result, after checking
  that every rank ends with its weights and state."""
  if world == 1:
    np.random.seed(0)
    return _train(cfg, image_bank)
  out = str(tmp_path / ('%s_rank%%d.pkl' % cfg['testname']))
  mp.spawn(_worker, args=(world, _free_port(), cfg, image_bank, out), nprocs=world, join=True)
  ranks = []
  for r in range(world):
    with open(out % r, 'rb') as f:
      ranks.append(pickle.load(f))
  for other in ranks[1:]:
    _same(other, ranks[0], checkpoints=False)
  return ranks[0]


def _same(got, ref, checkpoints=True, exp=None, names=None):
  for key in ('epoch_loss', 'batch_losses', 'validation'):
    assert repr(got['hist'][key]) == repr(ref['hist'][key]), key
  assert np.array_equal(bits(got['state']), bits(ref['state'])) and ref['state'].any()
  files = [Wt.load(got['hist']['weights_filename']), Wt.load(ref['hist']['weights_filename'])]
  for name, (k, b) in ref['weights'].items():
    for i, r in enumerate((k, b)):
      assert np.array_equal(bits(got['weights'][name][i]), bits(r)), (name, i)
      assert np.array_equal(bits(files[0][name][i]), bits(files[1][name][i])), ('weight file', name, i)
  if checkpoints:
    ck = [np.load(os.path.join(exp, d, training.CHECKPOINT), allow_pickle=False) for d in names]
    assert sorted(ck[0].files) == sorted(ck[1].files)
    for key in ck[0].files:
      assert np.array_equal(ck[0][key], ck[1][key]), key


@pytest.mark.parametrize('legs', sorted(FLOWS))
def test_one_chunk_is_the_run_without_the_key(tmp_path, dataset, legs):
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  plain = _run(tmp_path, _cfg(root, pretrained, exp, 'plain', legs, False, no_epochs=2), 1)
  one = _run(tmp_path, _cfg(root, pretrained, exp, 'one', legs, False, no_epochs=2, gradient_chunks=1), 1)
  _same(one, plain, checkpoints=False)
  assert 'gradient chunks: 1 per batch' in open(os.path.join(exp, 'one', 'training.log')).read()


@pytest.mark.parametrize('legs,yaw,precision,image_bank', [('360OutputkLegs', False, 'fp32', None),
                                                           ('360OutputkLegsFixed', True, 'fp32', None),
                                                           ('360OutputkLegs', True, 'tf32x3', 'host')])
def test_four_chunks_give_the_same_run_on_one_two_and_three_ranks(tmp_path, dataset, legs, yaw, precision,
                                                                   image_bank):
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  runs = {}
  for world in (1, 2, 3):
    cfg = _cfg(root, pretrained, exp, 'w%d' % world, legs, yaw, precision, gradient_chunks=4, checkpoint=True)
    runs[world] = _run(tmp_path, cfg, world, image_bank)
  for world in (2, 3):
    _same(runs[world], runs[1], exp=exp, names=('w%d' % world, 'w1'))
  log = open(os.path.join(exp, 'w3', 'training.log')).read()
  assert 'chunk ranges by rank: 0: [0, 2), 1: [2, 3), 2: [3, 4)' in log
  print(legs, yaw, precision, image_bank, 'epoch losses', runs[1]['hist']['epoch_loss'])


@pytest.mark.parametrize('legs', sorted(FLOWS))
def test_a_resume_on_another_world_size_continues_the_run(tmp_path, dataset, legs):
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  cfg = lambda name, **keys: _cfg(root, pretrained, exp, name, legs, True, gradient_chunks=4, **keys)
  straight = _run(tmp_path, cfg('straight', checkpoint=True), 1)
  for name, first, then in (('two_then_one', 2, 1), ('one_then_three', 1, 3)):
    _run(tmp_path, cfg(name, checkpoint=True, no_epochs=1), first)
    resumed = _run(tmp_path, cfg(name, resume=True), then)
    _same(resumed, straight, exp=exp, names=(name, 'straight'))
    assert 'after epoch 1 of 3' in open(os.path.join(exp, name, 'training.log')).read()
