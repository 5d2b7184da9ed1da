"""Data-parallel training on the GPU: ovn_copy_gradients / ovn_adagrad_step_sum against today's Adagrad steps and
a NumPy float32 oracle, their error paths, the weighted sum of a split batch against the whole batch, and both
training drivers on two ranks (gloo on one GPU; NCCL with two GPUs) against a one-process emulation."""
import copy
import os
import pickle
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import network as N
from overlapnet_b200 import data_parallel, synth, training, training_leg
from overlapnet_b200 import weights as Wt
from overlapnet_b200._cabi import OvnError
from overlapnet_b200.engine import HEAD_LAYERS
from test_gpu_train import _write_dataset
from test_gpu_train_leg import LEFT, MAXP, MODEL, RIGHT, _engine, _idx, _setup

pytestmark = pytest.mark.gpu

KINDS = ['frozen', 'whole']


def bits(a):
  return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _flat_layers(eng, whole):
  """(name, kernel or bias index, size) in the flat gradient order."""
  shapes = eng._layer_shapes()
  out = []
  for name in HEAD_LAYERS + (eng.leg_layers if whole else ()):
    for i in range(2):
      out.append((name, i, int(np.prod(shapes[name][i]))))
  return out


def _flatten(eng, weights, whole):
  return np.concatenate([np.asarray(weights[name][i], np.float32).ravel() for name, i, _ in _flat_layers(eng, whole)])


def _unflatten(eng, flat, whole):
  out, o = {}, 0
  for name, i, n in _flat_layers(eng, whole):
    out[(name, i)] = flat[o:o + n]
    o += n
  assert o == flat.size
  return out


def _gradients(eng, kind, x, n0, n1):
  """The gradients of pairs [n0, n1) of LEFT / RIGHT (the frozen leg's bank, or the image bank)."""
  dev = eng.device
  _, _, _, gt_ov, gt_or = _setup(True)
  li, ri = _idx(LEFT[n0:n1], dev), _idx(RIGHT[n0:n1], dev)
  if kind == 'whole':
    return eng.net_gradients(x, li, ri, gt_ov[n0:n1], gt_or[n0:n1], 0.7)
  return eng.head_gradients(eng.leg(x), li, ri, gt_ov[n0:n1], gt_or[n0:n1], 0.7)


def test_gradient_size():
  w, x, _, _, _ = _setup(True)
  eng = _engine(w)
  assert eng.gradient_size(False) == 665025 and eng.gradient_size(True) == 1769137
  assert eng.gradient_size(True) == sum(n for _, _, n in _flat_layers(eng, True))
  eng.close()


@pytest.mark.parametrize('kind', KINDS)
def test_one_part_of_weight_one_is_todays_step(kind):
  """Three steps: copy_gradients + adagrad_step_sum([g], [1]) against ovn_head_adagrad_step /
  ovn_net_adagrad_step, bit for bit after every step (each step's update divides by sqrt of the accumulator, so
  equal weights after three different gradients need equal accumulators).  The one-process step is one launch, and
  matches the NumPy float32 oracle on the gradients copy_gradients returns."""
  w, x, _, _, _ = _setup(True)
  whole = kind == 'whole'
  engs = [_engine(w), _engine(w)]
  xs = torch.from_numpy(x).to(engs[0].device)
  ref_w = _flatten(engs[0], engs[0].get_weights(), whole)
  ref_a = np.zeros(ref_w.size, np.float32)
  for step in range(3):
    lr = 1e-3 * (step + 1)
    for k, eng in enumerate(engs):
      _gradients(eng, kind, xs, step, step + 4)
      g = eng.copy_gradients(whole)
      if k == 0:
        ref_w, ref_a = adagrad_sum_oracle(ref_w, ref_a, g.cpu().numpy()[None], [1.0], lr)
        n0 = eng.launch_count()
        if whole:
          eng.net_adagrad_step(lr)
        else:
          eng.adagrad_step(lr)
        assert eng.launch_count() == n0 + 1
      else:
        eng.adagrad_step_sum(g[None], [1.0], lr, whole)
    a, b = engs[0].get_weights(), engs[1].get_weights()
    assert np.array_equal(bits(_flatten(engs[0], a, whole)), bits(ref_w)), step
    for name in a:
      for i in range(2):
        assert np.array_equal(bits(a[name][i]), bits(b[name][i])), (step, name, i)
        if not whole and name not in HEAD_LAYERS:
          assert np.array_equal(bits(a[name][i]), bits(w[name][i])), name
  for eng in engs:
    eng.check()
    eng.close()


def _fma32(a, b, c):
  """float32 fma(a, b, c), rounded once: a b is exact in float64; the sum is rounded to odd at 53 bits (exact
  error by TwoSum), which then rounds to float32 like the exact value does."""
  p = a.astype(np.float64) * b.astype(np.float64)
  c = c.astype(np.float64)
  s = p + c
  bp = s - c
  err = (c - (s - bp)) + (p - bp)
  raw = s.view(np.int64)
  fix = (err != 0) & ((raw & 1) == 0)
  raw = np.where(fix, raw + np.where((err > 0) == (s > 0), 1, -1), raw)
  return raw.view(np.float64).astype(np.float32)


def adagrad_sum_oracle(w, a, parts, weights, lr):
  """ovn_adagrad_step_sum in NumPy float32: g = sum_k weights[k] parts[k] in order (weight-0 parts skipped), then
  a = fma(g, g, a); w -= (lr g) / (sqrt(a) + 1e-7).  Returns the new (w, a)."""
  g = None
  for p, wk in zip(parts, np.asarray(weights, np.float32)):
    if wk == 0:
      continue
    v = wk * p
    g = v if g is None else g + v
  g = np.zeros_like(w) if g is None else g
  a = _fma32(g, g, a)
  return w - (np.float32(lr) * g) / (np.sqrt(a) + np.float32(1e-7)), a


@pytest.mark.parametrize('kind', KINDS)
def test_weighted_sum_of_three_parts_matches_numpy_oracle(kind):
  """On a handle that never computed a gradient (the training state is allocated by the call): two steps with three
  random parts, the middle one of weight 0, bit for bit against the oracle; the frozen leg is untouched."""
  w, _, _, _, _ = _setup(True)
  whole = kind == 'whole'
  eng = _engine(w)
  n = eng.gradient_size(whole)
  rng = np.random.default_rng(9)
  ref_w = _flatten(eng, eng.get_weights(), whole)
  ref_a = np.zeros(n, np.float32)
  for step, weights in enumerate(([0.3, 0.0, 0.7], [1 / 3.0, 0.0, 2 / 3.0])):
    parts = (rng.standard_normal((3, n)) * 10.0 ** rng.integers(-5, -1, (3, n))).astype(np.float32)
    lr = 1e-3 * (step + 1)
    eng.adagrad_step_sum(torch.from_numpy(parts).to(eng.device), weights, lr, whole)
    ref_w, ref_a = adagrad_sum_oracle(ref_w, ref_a, parts, weights, lr)
    got = eng.get_weights()
    assert np.array_equal(bits(_flatten(eng, got, whole)), bits(ref_w)), step
  if not whole:
    for name in eng.leg_layers:
      assert np.array_equal(bits(got[name][0]), bits(w[name][0])), name
  eng.check()
  eng.close()


def test_step_sum_errors():
  w, x, _, _, _ = _setup(True)
  eng = _engine(w)
  dev = eng.device
  xs = torch.from_numpy(x).to(dev)
  before = eng.get_weights()
  for whole in (False, True):                                   # no valid gradients yet
    with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
      eng.copy_gradients(whole)
  _gradients(eng, 'frozen', xs, 0, 4)
  eng.copy_gradients(False)
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG.*whole-network'):
    eng.copy_gradients(True)                                    # leg layers after a head-only call
  for whole in (False, True):
    with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG.*n_parts'):
      eng.adagrad_step_sum(torch.empty((0,), device=dev), [], 1e-3, whole)
  after = eng.get_weights()                                     # the refused calls changed nothing
  for name in before:
    for i in range(2):
      assert np.array_equal(bits(before[name][i]), bits(after[name][i])), name
  eng.check()
  eng.close()
  tc = _engine(w, precision='f16_tc')
  n = tc.gradient_size(True)
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG'):
    tc.adagrad_step_sum(torch.zeros((1, n), device=dev), [1.0], 1e-3, True)
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG'):
    tc.copy_gradients(True)
  tc.close()


@pytest.mark.parametrize('kind', KINDS)
def test_split_batch_sum_matches_the_whole_batch(kind):
  """One 8-pair batch: (4/8) g(pairs 0..3) + (4/8) g(pairs 4..7) against g(all 8) on one handle."""
  w, x, _, _, _ = _setup(True)
  whole = kind == 'whole'
  eng = _engine(w)
  xs = torch.from_numpy(x).to(eng.device)
  _gradients(eng, kind, xs, 0, MAXP)
  full = eng.copy_gradients(whole).cpu().numpy()
  bounds, weights = data_parallel.shares(MAXP, 2)
  parts = []
  for lo, hi in bounds:
    _gradients(eng, kind, xs, lo, hi)
    parts.append(eng.copy_gradients(whole).cpu().numpy())
  summed = sum(np.float64(wr) * p.astype(np.float64) for wr, p in zip(weights, parts))
  got, ref = _unflatten(eng, summed, whole), _unflatten(eng, full, whole)
  eng.close()
  for (name, i), r in ref.items():
    err = float(np.abs(got[(name, i)] - r).max()) / float(np.abs(r).max())
    tol = 1e-5 if name in HEAD_LAYERS else 1e-4
    print('%s %s[%d]: max|sum of parts - whole batch| / max|whole batch| = %.2e (bound %.0e)' % (kind, name, i, err,
                                                                                                   tol))
    assert np.abs(r).max() > 0 and err <= tol, (name, i, err)


# ---- the drivers on two ranks ---------------------------------------------------------------------------------
FLOWS = {'360OutputkLegsFixed': (training, 'FrozenLeg', training.train),
         '360OutputkLegs': (training_leg, 'WholeNetwork', training_leg.train)}


@pytest.fixture(scope='module')
def dataset(tmp_path_factory):
  """The synthetic two-sequence dataset of test_training_driver_end_to_end."""
  root = str(tmp_path_factory.mktemp('dp_data'))
  teacher = N.glorot_weights(4, MODEL, seed=0)
  eng = _engine(teacher, maxp=64)
  xs = synth.range_like_images(11, 6, 4)
  fvh = eng.leg(torch.from_numpy(xs).to(eng.device)).cpu().numpy()
  eng.close()
  _, _, _, z = N.heads_forward(fvh[:, None], np.roll(fvh, 1, 0)[:, None], teacher, MODEL, return_logit=True)
  teacher = N.spread_dense(teacher, z, target_std=1.5)
  return root, _write_dataset(root, teacher)


def _config(root, pretrained, exp, name, legs, yaw):
  return {'experiments_path': exp, 'testname': name, 'pretrained_weightsfilename': pretrained,
          'use_depth': True, 'use_normals': True, 'data_root_folder': root, 'training_seqs': '00 01',
          'batch_size': 8, 'no_batches_in_epoch': 1000, 'no_epochs': 2, 'no_test_pairs': 1000,
          'learning_rate': 1e-4, 'lr_alpha': 0.99, 'min_overlap_for_angle': 0.7, 'yaw_augmentation': yaw,
          'model': {'modelType': 'SiameseNetworkTemplate', 'legsType': legs,
                    'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                    'inputShape': [64, 900], 'leg_output_width': 360, **MODEL}}


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _dp_worker(rank, world, port, backend, cfg, out):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  device = rank if backend == 'nccl' else 0
  torch.cuda.set_device(device)
  dist.init_process_group(backend, rank=rank, world_size=world)
  try:
    module, name, train = FLOWS[cfg['model']['legsType']]
    kept = []

    class Keep(getattr(module, name)):
      def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        kept.append(self)

    setattr(module, name, Keep)
    np.random.seed(0)
    hist = train(cfg, device)
    with open(out % rank, 'wb') as f:
      pickle.dump({'hist': hist, 'weights': kept[0].eng.get_weights()}, f)
  finally:
    dist.destroy_process_group()


def _emulated(base):
  """``base`` whose step computes the two ranks' shares in turn on one handle, copies each, and applies
  adagrad_step_sum with both parts: what two ranks do, in one process."""
  class Emulated(base):
    def step(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, lr, rotate=None):
      bounds, weights = data_parallel.shares(left.numel(), 2)
      parts = torch.zeros((2, self.eng.gradient_size(self.whole_network)), dtype=torch.float32, device=self.eng.device)
      losses = []
      for r, (lo, hi) in enumerate(bounds):
        if hi == lo:
          losses.append((0.0, 0.0, 0.0))
          continue
        rot = None if rotate is None else tuple(t[lo:hi] for t in rotate)
        losses.append(self.gradients(left[lo:hi], right[lo:hi], gt_overlap[lo:hi], gt_orientation[lo:hi],
                                     min_overlap_for_angle, rot))
        self.eng.copy_gradients(self.whole_network, out=parts[r])
      self.eng.adagrad_step_sum(parts, weights, lr, self.whole_network)
      return tuple(float(sum(w * l[k] for w, l in zip(weights, losses))) for k in range(3))
  return Emulated


def _check_two_ranks(tmp_path, monkeypatch, dataset, legs, yaw, backend):
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  cfg = _config(root, pretrained, exp, 'dp', legs, yaw)
  out = str(tmp_path / 'rank%d.pkl')
  mp.spawn(_dp_worker, args=(2, _free_port(), backend, copy.deepcopy(cfg), out), nprocs=2, join=True)
  ranks = []
  for r in range(2):
    with open(out % r, 'rb') as f:
      ranks.append(pickle.load(f))
  module, name, train = FLOWS[legs]
  monkeypatch.setattr(module, name, _emulated(getattr(module, name)))
  np.random.seed(0)
  emu = train(_config(root, pretrained, exp, 'emu', legs, yaw))
  files = [Wt.load(ranks[0]['hist']['weights_filename']), Wt.load(emu['weights_filename'])]
  start = Wt.load(pretrained)
  for wname in start:
    for i in range(2):
      ref = bits(ranks[0]['weights'][wname][i])
      assert np.array_equal(bits(ranks[1]['weights'][wname][i]), ref), ('rank 1', wname, i)
      assert np.array_equal(bits(files[0][wname][i]), ref), ('weight file', wname, i)
      assert np.array_equal(bits(files[1][wname][i]), ref), ('emulation', wname, i)
    trained = not np.array_equal(files[0][wname][0], start[wname][0])
    assert trained == (legs == '360OutputkLegs' or wname in HEAD_LAYERS), wname
  for r in range(2):
    # the emulation's validation is unsharded: the same statistics on the same weights
    assert repr(ranks[r]['hist']['validation']) == repr(emu['validation'])
    assert ranks[r]['hist']['batch_losses'] == emu['batch_losses']
  print(legs, 'yaw' if yaw else '', backend, 'epoch losses', emu['epoch_loss'],
        'validation rms', [v['rms'] for v in emu['validation']])
  log = open(os.path.join(exp, 'dp', 'training.log')).read()
  assert 'data-parallel over 2 ranks' in log and 'iteration 2, batch/epoch loss' in log


@pytest.mark.parametrize('yaw', [False, True])
@pytest.mark.parametrize('legs', sorted(FLOWS))
def test_two_ranks_on_one_gpu_match_the_one_process_emulation(tmp_path, monkeypatch, dataset, legs, yaw):
  _check_two_ranks(tmp_path, monkeypatch, dataset, legs, yaw, 'gloo')


@pytest.mark.parametrize('legs', sorted(FLOWS))
def test_two_gpus_nccl_match_the_one_process_emulation(tmp_path, monkeypatch, dataset, legs):
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  _check_two_ranks(tmp_path, monkeypatch, dataset, legs, True, 'nccl')
