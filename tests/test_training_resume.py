"""CPU checks of resumable training (overlapnet_b200.training, ``checkpoint`` / ``resume``) on a fake handle and
flow: a run stopped after 2 of 4 epochs and resumed makes the steps, history and state of the straight run, in one
process and on two gloo ranks; every refusal of a checkpoint; and a run without the keys writes no checkpoint and
records what a checkpointing run records."""
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
from overlapnet_b200 import infer as _infer
from overlapnet_b200 import weights as Wt


class _Engine:
  """Weights w (3 kernel + 1 bias floats) and their accumulators in the flat order: the 'heads' are the first 2."""
  device = torch.device('cpu')
  W = 900

  def __init__(self):
    self.w = {'w': (np.arange(3, dtype=np.float32) + 7, np.zeros(1, np.float32))}
    self.accum = np.zeros(4, np.float32)
    self.last = None
    self.loaded, self.set_states, self.read_states = [], [], []

  def get_weights(self):
    return {k: (a.copy(), b.copy()) for k, (a, b) in self.w.items()}

  def load_weights(self, w):
    self.w = {k: (np.array(a, np.float32), np.array(b, np.float32)) for k, (a, b) in w.items()}
    self.accum[:] = 0                                  # like ovn_finalize_weights
    self.loaded.append(self.get_weights())

  def check(self):
    pass

  def gradient_size(self, whole_network=False):
    return 4 if whole_network else 2

  def train_state(self, whole_network=False, out=None):
    v = self.accum[:self.gradient_size(whole_network)].copy()
    self.read_states.append(v)
    return torch.from_numpy(v.copy())

  def set_train_state(self, vec, whole_network=False):
    v = np.asarray(vec, np.float32)
    assert v.shape == (self.gradient_size(whole_network),)
    self.set_states.append(v.copy())
    self.accum[:v.size] = v

  def copy_gradients(self, whole_network=False, out=None):
    out.copy_(self.last[:self.gradient_size(whole_network)])
    return out

  def adagrad_step_sum(self, parts, weights, lr, whole_network=False):
    g = None
    for p, wk in zip(parts.numpy(), np.asarray(weights, np.float32)):
      g = wk * p if g is None else g + wk * p
    self.adagrad(g, lr)

  def adagrad(self, g, lr):
    n = g.size
    self.accum[:n] += g * g
    flat = np.concatenate([self.w['w'][0], self.w['w'][1]])
    flat[:n] -= np.float32(lr) * g / (np.sqrt(self.accum[:n]) + np.float32(1e-7))
    self.w['w'] = (flat[:3], flat[3:])


class _Infer:
  def __init__(self, cfg, precision, device, max_batch_pairs):
    self._engine = _Engine()
    self.network_output_size = cfg['model']['leg_output_width']
    _Infer.last = self


class _Flow:
  """Records what the loop hands to each step; a share's 'gradients' depend on its pairs and labels."""
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
    self.eng.last = torch.tensor([left.sum(), right.sum(), gt_orientation.sum() / 100, left.numel()],
                                 dtype=torch.float32) / 10
    return (float(left.sum()) + 0.5, float(right.sum()), float(left.numel()))

  def step(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, lr, rotate=None):
    loss = self.gradients(left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate)
    self.eng.adagrad(self.eng.last[:self.eng.gradient_size(self.whole_network)].numpy(), lr)
    return loss

  def evaluate(self, left, right):
    s = float(self.eng.w['w'][0].sum())
    return 0.3 + left.float() / 20 + s / 1000, (180 - right).to(torch.int32)


class _FrozenFlow(_Flow):
  whole_network = False


FLOWS = {'whole': _Flow, 'frozen': _FrozenFlow}
N_PAIRS = 11                 # batches of 5, 5 and 1 pairs: the last one leaves rank 1 an empty share


def _write_files(tmp):
  table = np.array([[i, (i + 1 + i // 6) % 7, 0.5, (37 * i) % 360] for i in range(N_PAIRS)], float)
  np.savez(os.path.join(tmp, 'train.npz'), overlaps=table, seq=np.array([['00', '00']] * N_PAIRS))
  np.savez(os.path.join(tmp, 'val.npz'), overlaps=table[:3], seq=np.array([['00', '00']] * 3))


def _config(tmp, name, epochs, yaw, **keys):
  return {'experiments_path': tmp, 'testname': name, 'pretrained_weightsfilename': '',
          'traindata_npzfile': os.path.join(tmp, 'train.npz'), 'validationdata_npzfile': os.path.join(tmp, 'val.npz'),
          'batch_size': 5, 'no_batches_in_epoch': 3, 'no_epochs': epochs, 'no_test_pairs': 3, 'learning_rate': 1e-3,
          'yaw_augmentation': yaw,
          'model': {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
                    'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                    'inputShape': [64, 900], 'leg_output_width': 360}, **keys}


def _run(cfg, flow, seed):
  """training.run on the fakes after np.random.seed(seed); what the run did."""
  saved = _infer.Infer
  _infer.Infer = _Infer
  try:
    np.random.seed(seed)
    hist = training.run(cfg, None, flow)
  finally:
    _infer.Infer = saved
  eng = _Infer.last._engine
  return {'hist': hist, 'calls': _Flow.instance.calls, 'state': np.random.get_state()[1].copy(),
          'weights': eng.get_weights(), 'accum': eng.accum.copy(), 'set_states': eng.set_states,
          'read_states': eng.read_states, 'loaded': eng.loaded}


def _straight_and_resumed(tmp, yaw, flow):
  straight = _run(_config(tmp, 's', 4, yaw, checkpoint=True), flow, 7)
  first = _run(_config(tmp, 'r', 2, yaw, checkpoint=True), flow, 7)
  second = _run(_config(tmp, 'r', 4, yaw, resume=True), flow, 12345)     # the saved state replaces this seed
  return straight, first, second


def _same_calls(a, b):
  assert len(a) == len(b)
  for i, (x, y) in enumerate(zip(a, b)):
    for k in range(3):
      assert np.array_equal(x[k], y[k]), (i, k)
    assert (x[3] is None) == (y[3] is None), i
    if x[3] is not None:
      for k in range(3):
        assert np.array_equal(x[3][k], y[3][k]), (i, k)


def _load(path):
  with np.load(path, allow_pickle=False) as z:
    return {k: z[k] for k in z.files}


def _history(run):
  return repr({k: v for k, v in run['hist'].items() if k != 'weights_filename'})


def _check_resumed(straight, first, second, whole, rank0=True):
  """The stopped + resumed run against the straight one, as one rank sees them."""
  # 3 steps per epoch; rank 1 of two has nothing to compute in the 1-pair step
  assert len(straight['calls']) == 2 * len(first['calls']) == (12 if rank0 else 8)
  _same_calls(straight['calls'], first['calls'] + second['calls'])     # pairs, labels, shifts and rotations
  assert _history(second) == _history(straight)
  n = 4 if whole else 2
  # the resumed run applied the accumulators the straight run had after epoch 2, after loading the weights
  assert len(second['set_states']) == 1 and second['set_states'][0].shape == (n,)
  assert len(second['loaded']) == 1
  if rank0:                                                        # rank 0 reads them for its checkpoints
    assert np.array_equal(second['set_states'][0], straight['read_states'][1])
    assert np.array_equal(second['state'], straight['state'])       # and makes every random draw
  assert np.array_equal(second['accum'], straight['accum'])
  for name, (k, b) in straight['weights'].items():
    assert np.array_equal(second['weights'][name][0], k) and np.array_equal(second['weights'][name][1], b)
  assert straight['hist']['validation'][0]['learning_rate'] != straight['hist']['validation'][1]['learning_rate']


@pytest.mark.parametrize('kind', sorted(FLOWS))
@pytest.mark.parametrize('yaw', [False, True])
def test_resumed_run_makes_the_straight_runs_steps(tmp_path, yaw, kind):
  tmp = str(tmp_path)
  _write_files(tmp)
  straight, first, second = _straight_and_resumed(tmp, yaw, FLOWS[kind])
  _check_resumed(straight, first, second, kind == 'whole')
  # the last checkpoints agree in every array, and so do the weight files
  a, b = _load(os.path.join(tmp, 's', training.CHECKPOINT)), _load(os.path.join(tmp, 'r', training.CHECKPOINT))
  assert sorted(a) == sorted(b) and int(a['epochs']) == 4
  for k in a:
    assert np.array_equal(a[k], b[k]), k
  wa = Wt.load_npz(os.path.join(tmp, 's', 'SiameseNetworkTemplate_s.weight'))
  wb = Wt.load_npz(os.path.join(tmp, 'r', 'SiameseNetworkTemplate_r.weight'))
  assert np.array_equal(wa['w'][0], wb['w'][0])
  # the log is appended to and says where the run resumed
  log = open(os.path.join(tmp, 'r', 'training.log')).read()
  assert 'iteration 2,' in log and 'iteration 3,' in log and log.index('iteration 2,') < log.index('Resuming from')
  assert 'after epoch 2 of 4' in log and 'checkpoint after epoch 4 written' in log


def test_no_keys_write_no_checkpoint_and_record_the_same_run(tmp_path):
  tmp = str(tmp_path)
  _write_files(tmp)
  plain = _run(_config(tmp, 'p', 2, True), _Flow, 7)
  ck = _run(_config(tmp, 'c', 2, True, checkpoint=True), _Flow, 7)
  assert sorted(os.listdir(os.path.join(tmp, 'p'))) == ['SiameseNetworkTemplate_p.weight', 'training.log']
  assert os.path.exists(os.path.join(tmp, 'c', training.CHECKPOINT))
  _same_calls(plain['calls'], ck['calls'])
  assert _history(plain) == _history(ck)
  assert np.array_equal(plain['state'], ck['state']) and plain['read_states'] == []
  strip = lambda path: [l.split(' ', 1)[1] for l in open(path).read().splitlines()]      # drop the time stamps
  lines_p = strip(os.path.join(tmp, 'p', 'training.log'))
  lines_c = [l for l in strip(os.path.join(tmp, 'c', 'training.log')) if 'checkpoint after epoch' not in l]
  assert lines_p == [l.replace('c/SiameseNetworkTemplate_c', 'p/SiameseNetworkTemplate_p') for l in lines_c]


# ---- refusals -----------------------------------------------------------------------------------------------
def _rewrite(path, **changes):
  arrays = _load(path)
  for k, v in changes.items():
    if v is None:
      del arrays[k]
    else:
      arrays[k] = v
  with open(path, 'wb') as f:
    np.savez(f, **arrays)


REFUSALS = {
    'missing': (lambda p: os.remove(p), {}, 'cannot read'),
    'unreadable': (lambda p: open(p, 'wb').write(b'PK\x03\x04 not a zip'), {}, 'cannot read'),
    'version': (lambda p: _rewrite(p, format_version=np.int64(2)), {}, 'format version 2'),
    'no version': (lambda p: _rewrite(p, format_version=None), {}, 'format version none'),
    'fingerprint': (None, {'learning_rate': 2e-3}, 'config key learning_rate differs'),
    'fingerprint model': (None, {'model_overlap_head': 'X'}, 'config key model.overlap_head differs'),
    'fingerprint yaw': (None, {'yaw_augmentation': True}, 'config key yaw_augmentation differs'),
    'layer': (lambda p: _rewrite(p, **{'x/kernel': np.zeros(1, np.float32), 'x/bias': np.zeros(1, np.float32)}), {},
              r"has the layers \['w', 'x'\]"),
    'shape': (lambda p: _rewrite(p, **{'w/kernel': np.zeros(4, np.float32)}), {}, 'layer w of the checkpoint'),
    'accum length': (lambda p: _rewrite(p, accum=np.zeros(3, np.float32)), {}, 'holds 3 Adagrad accumulators'),
    'accum negative': (lambda p: _rewrite(p, accum=np.array([0, -1e-9, 0, 0], np.float32)), {},
                       'negative or not finite'),
    'accum nan': (lambda p: _rewrite(p, accum=np.array([0, 0, np.nan, 0], np.float32)), {}, 'negative or not finite'),
    'accum inf': (lambda p: _rewrite(p, accum=np.array([np.inf, 0, 0, 0], np.float32)), {}, 'negative or not finite'),
    'done': (None, {'no_epochs': 2}, 'holds 2 completed epochs, no_epochs is 2'),
}


@pytest.mark.parametrize('cause', sorted(REFUSALS))
def test_resume_refuses(tmp_path, cause):
  tmp = str(tmp_path)
  _write_files(tmp)
  _run(_config(tmp, 'r', 2, False, checkpoint=True), _Flow, 7)
  damage, change, match = REFUSALS[cause]
  path = os.path.join(tmp, 'r', training.CHECKPOINT)
  if damage is not None:
    damage(path)
  cfg = _config(tmp, 'r', 4, False, resume=True)
  for k, v in change.items():
    if k.startswith('model_'):
      cfg['model'][k[len('model_'):]] = v
    else:
      cfg[k] = v
  with pytest.raises(Exception, match=match):
    _run(cfg, _Flow, 7)


def test_interrupted_write_is_not_a_checkpoint(tmp_path):
  """A temp file an interrupted write left behind is never read: alone it is no checkpoint, and next to a
  checkpoint it is ignored."""
  tmp = str(tmp_path)
  _write_files(tmp)
  _run(_config(tmp, 'r', 2, False, checkpoint=True), _Flow, 7)
  path = os.path.join(tmp, 'r', training.CHECKPOINT)
  os.replace(path, path + '.tmp')                                  # a whole file, never renamed into place
  with pytest.raises(Exception, match='cannot read'):
    _run(_config(tmp, 'r', 4, False, resume=True), _Flow, 7)
  _run(_config(tmp, 'r', 2, False, checkpoint=True), _Flow, 7)
  with open(path + '.tmp', 'wb') as f:
    f.write(b'PK\x03\x04 half a zip')
  assert len(_run(_config(tmp, 'r', 3, False, resume=True), _Flow, 7)['hist']['epoch_loss']) == 3


# ---- two gloo ranks -----------------------------------------------------------------------------------------
def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _worker(rank, world, port, tmp, yaw):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  try:
    assert data_parallel.default_group() is not None
    res = _straight_and_resumed(tmp, yaw, _Flow)
    with open(os.path.join(tmp, 'rank%d.pkl' % rank), 'wb') as f:
      pickle.dump(res, f)
  finally:
    dist.destroy_process_group()


@pytest.mark.parametrize('yaw', [False, True])
def test_two_rank_resumed_run_makes_the_straight_runs_steps(tmp_path, yaw):
  tmp = str(tmp_path)
  _write_files(tmp)
  mp.spawn(_worker, args=(2, _free_port(), tmp, yaw), nprocs=2, join=True)
  ranks = []
  for r in range(2):
    with open(os.path.join(tmp, 'rank%d.pkl' % r), 'rb') as f:
      ranks.append(pickle.load(f))
  for r, (straight, first, second) in enumerate(ranks):
    _check_resumed(straight, first, second, True, rank0=r == 0)
  # only rank 0 reads the state (for its checkpoints); every rank applies the same vector on resume
  assert ranks[1][0]['read_states'] == [] and len(ranks[0][0]['read_states']) == 4
  assert np.array_equal(ranks[0][2]['set_states'][0], ranks[1][2]['set_states'][0])
  assert sorted(os.listdir(os.path.join(tmp, 'r'))) == ['SiameseNetworkTemplate_r.weight', training.CHECKPOINT,
                                                         'training.log']
