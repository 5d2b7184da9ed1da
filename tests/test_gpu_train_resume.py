"""Resumable training on the GPU: ovn_copy_train_state / ovn_set_train_state (round trip, reset by
ovn_finalize_weights, an Adagrad step from a set state against the NumPy float32 oracle, the error paths), and both
training drivers stopped after one epoch and resumed to three against the straight three-epoch run, bit for bit:
weight files, Engine.train_state, histories and checkpoints; in one process and on two gloo ranks sharing one
GPU."""
import copy
import ctypes as C
import os
import pickle

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from overlapnet_b200 import training
from overlapnet_b200 import weights as Wt
from overlapnet_b200._cabi import OvnError, lib
from overlapnet_b200.engine import Engine
from test_gpu_train_dp import FLOWS, _config, _flatten, _free_port, adagrad_sum_oracle, bits, dataset  # noqa: F401
from test_gpu_train_leg import MAXP, MODEL, N_IMAGES, _engine, _setup

pytestmark = pytest.mark.gpu


def _positive(rng, n):
  return (rng.random(n) * 10.0 ** rng.integers(-8, -2, n)).astype(np.float32)


def test_state_round_trips_and_is_reset_by_new_weights():
  w, _, _, _, _ = _setup(True)
  eng = _engine(w)
  n_head, n_all = eng.gradient_size(False), eng.gradient_size(True)
  for whole, n in ((False, n_head), (True, n_all)):           # a handle that never trained
    z = eng.train_state(whole).cpu().numpy()
    assert z.shape == (n,) and not z.any()
  rng = np.random.default_rng(3)
  a = _positive(rng, n_all)
  eng.set_train_state(a, True)
  assert np.array_equal(bits(eng.train_state(True).cpu().numpy()), bits(a))
  assert np.array_equal(bits(eng.train_state(False).cpu().numpy()), bits(a[:n_head]))
  b = _positive(rng, n_head)
  eng.set_train_state(torch.from_numpy(b).to(eng.device), False)      # the heads' prefix only
  got = eng.train_state(True).cpu().numpy()
  assert np.array_equal(bits(got[:n_head]), bits(b)) and np.array_equal(bits(got[n_head:]), bits(a[n_head:]))
  eng.load_weights(w)                                            # ovn_finalize_weights: Adagrad starts over
  assert not eng.train_state(True).cpu().numpy().any()
  eng.check()
  eng.close()


@pytest.mark.parametrize('whole', [False, True])
def test_step_from_a_set_state_matches_numpy_oracle(whole):
  """On a handle that never trained: set a known state, then one adagrad_step_sum of one part, bit for bit
  against the oracle started from that state; the new state too."""
  w, _, _, _, _ = _setup(True)
  eng = _engine(w)
  n = eng.gradient_size(whole)
  rng = np.random.default_rng(5)
  a0 = _positive(rng, n)
  g = (rng.standard_normal(n) * 10.0 ** rng.integers(-5, -1, n)).astype(np.float32)
  eng.set_train_state(a0, whole)
  eng.adagrad_step_sum(torch.from_numpy(g[None]).to(eng.device), [1.0], 2e-3, whole)
  ref_w, ref_a = adagrad_sum_oracle(_flatten(eng, w, whole), a0, g[None], [1.0], 2e-3)
  assert np.array_equal(bits(_flatten(eng, eng.get_weights(), whole)), bits(ref_w))
  assert np.array_equal(bits(eng.train_state(whole).cpu().numpy()), bits(ref_a))
  eng.check()
  eng.close()


def test_train_state_errors():
  w, _, _, _, _ = _setup(True)
  L = lib()
  eng = _engine(w)
  s = eng._stream()
  for whole in (0, 1):                                           # NULL pointers
    assert L.ovn_copy_train_state(eng._h, whole, None, s) == -1     # OVN_ERR_INVALID_ARG
    assert L.ovn_set_train_state(eng._h, whole, None, s) == -1
  assert not eng.train_state(True).cpu().numpy().any()           # the refused calls changed nothing
  eng.close()
  bare = Engine(model=MODEL, precision='fp32', max_batch_scans=N_IMAGES, max_batch_pairs=MAXP)   # no weights yet
  for whole in (False, True):
    with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG.*weights not finalised'):
      bare.train_state(whole)
    with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG.*weights not finalised'):
      bare.set_train_state(np.zeros(bare.gradient_size(whole), np.float32), whole)
  bare.close()
  tc = _engine(w, precision='f16_tc')
  buf = torch.zeros(tc.gradient_size(True), dtype=torch.float32, device=tc.device)
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG'):
    tc.train_state(True)
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG'):
    tc.set_train_state(buf, True)
  assert L.ovn_copy_train_state(tc._h, 1, C.c_void_p(buf.data_ptr()), tc._stream()) == -2   # OVN_ERR_BAD_CONFIG
  tc.close()


# ---- the drivers, stopped and resumed ------------------------------------------------------------------------
def _train(cfg, device=None):
  """One training run; its history and the handle's weights and Adagrad state at the end."""
  module, name, train = FLOWS[cfg['model']['legsType']]
  base = getattr(module, name)
  kept = []

  class Keep(base):
    def __init__(self, *args, **kw):
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


def _straight_and_resumed(root, pretrained, exp, legs, yaw, precision, device=None):
  runs = {}
  for name, epochs, keys, seed in (('straight', 3, {'checkpoint': True}, 0), ('stopped', 1, {'checkpoint': True}, 0),
                                   ('resumed', 3, {'resume': True}, 99)):
    cfg = _config(root, pretrained, exp, 'straight' if name == 'straight' else 'split', legs, yaw)
    cfg.update(no_epochs=epochs, training_precision=precision, **keys)
    np.random.seed(seed)                                         # the resumed run restores the saved state
    runs[name] = _train(cfg, device)
  return runs


def _check(runs, exp):
  straight, resumed = runs['straight'], runs['resumed']
  for key in ('epoch_loss', 'batch_losses', 'validation'):
    assert repr(resumed['hist'][key]) == repr(straight['hist'][key]), key
  assert len(resumed['hist']['epoch_loss']) == 3 and runs['stopped']['hist']['epoch_loss'] == \
      straight['hist']['epoch_loss'][:1]
  files = [Wt.load(straight['hist']['weights_filename']), Wt.load(resumed['hist']['weights_filename'])]
  for name, (k, b) in straight['weights'].items():
    for i, ref in enumerate((k, b)):
      assert np.array_equal(bits(resumed['weights'][name][i]), bits(ref)), (name, i)
      assert np.array_equal(bits(files[0][name][i]), bits(ref)), ('weight file', name, i)
      assert np.array_equal(bits(files[1][name][i]), bits(ref)), ('resumed weight file', name, i)
  assert np.array_equal(bits(resumed['state']), bits(straight['state'])) and straight['state'].any()
  ck = [np.load(os.path.join(exp, d, training.CHECKPOINT), allow_pickle=False) for d in ('straight', 'split')]
  assert sorted(ck[0].files) == sorted(ck[1].files) and int(ck[1]['epochs']) == 3
  for key in ck[0].files:
    assert np.array_equal(ck[0][key], ck[1][key]), key
  log = open(os.path.join(exp, 'split', 'training.log')).read()
  assert 'Resuming from' in log and 'after epoch 1 of 3' in log and 'iteration 3, batch/epoch loss' in log
  for line in log.splitlines():                                  # the cost of a checkpoint, as logged
    if 'checkpoint after epoch' in line:
      print(line.replace(exp, '<exp>'))


@pytest.mark.parametrize('precision,yaw', [('fp32', False), ('fp32', True), ('tf32x3', True)])
@pytest.mark.parametrize('legs', sorted(FLOWS))
def test_resumed_run_matches_the_straight_run(tmp_path, dataset, legs, precision, yaw):
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  _check(_straight_and_resumed(root, pretrained, exp, legs, yaw, precision), exp)


def _worker(rank, world, port, root, pretrained, exp, legs, out):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(0)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  try:
    runs = _straight_and_resumed(root, pretrained, exp, legs, True, 'fp32', 0)
    with open(out % rank, 'wb') as f:
      pickle.dump(runs, f)
  finally:
    dist.destroy_process_group()


@pytest.mark.parametrize('legs', sorted(FLOWS))
def test_two_ranks_on_one_gpu_resume_the_straight_run(tmp_path, dataset, legs):
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  out = str(tmp_path / 'rank%d.pkl')
  mp.spawn(_worker, args=(2, _free_port(), root, pretrained, exp, legs, out), nprocs=2, join=True)
  ranks = []
  for r in range(2):
    with open(out % r, 'rb') as f:
      ranks.append(pickle.load(f))
  _check(ranks[0], exp)
  for name in ('straight', 'resumed'):                           # rank 1 keeps rank 0's weights and state
    assert np.array_equal(bits(ranks[1][name]['state']), bits(ranks[0][name]['state'])), name
    for layer, (k, b) in ranks[0][name]['weights'].items():
      assert np.array_equal(bits(ranks[1][name]['weights'][layer][0]), bits(k)), (name, layer)
      assert np.array_equal(bits(ranks[1][name]['weights'][layer][1]), bits(b)), (name, layer)
    assert repr(ranks[1][name]['hist']['validation']) == repr(ranks[0][name]['hist']['validation'])
  assert 'data-parallel over 2 ranks' in open(os.path.join(exp, 'split', 'training.log')).read()
