"""Training with the image bank in pinned host memory: both flows forced to ``image_bank='host'`` against the same
runs on the device bank, bit for bit (weight files, Engine.train_state, histories with the validation statistics,
checkpoints), a host-bank run stopped after one epoch and resumed, two gloo ranks sharing one GPU, the device
memory a host bank saves, and the automatic choice of the host bank under a small device budget."""
import copy
import gc
import os
import pickle

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from overlapnet_b200 import image_bank, training
from overlapnet_b200 import weights as Wt
from test_gpu_train_dp import FLOWS, _config, _free_port, bits, dataset  # noqa: F401

pytestmark = pytest.mark.gpu

CASES = [('360OutputkLegs', False), ('360OutputkLegs', True), ('360OutputkLegsFixed', True)]


def _train(cfg, placement, device=None):
  """One training run with the flow's image bank forced to ``placement`` (None: chosen); its history, the
  handle's weights and Adagrad state, the flow's placement and the peak of torch's device allocations during the
  run above what was allocated before it."""
  module, name, train = FLOWS[cfg['model']['legsType']]
  base = getattr(module, name)
  kept = []

  class Keep(base):
    def __init__(self, *args, **kw):
      if placement is not None:
        kw['image_bank'] = placement
      super().__init__(*args, **kw)
      kept.append(self)

  setattr(module, name, Keep)
  gc.collect()                                                   # earlier runs' flows hold device tensors
  torch.cuda.synchronize()
  start = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  try:
    hist = train(copy.deepcopy(cfg), device)
  finally:
    setattr(module, name, base)
  peak = torch.cuda.max_memory_allocated() - start
  flow = kept[0]
  eng = flow.eng
  out = {'hist': hist, 'weights': eng.get_weights(), 'state': eng.train_state(base.whole_network).cpu().numpy(),
         'placement': flow.image_bank, 'peak': peak, 'n_images': len(flow.image_rows)}
  eng.close()
  return out


def _runs(root, pretrained, exp, legs, yaw, precision, device=None, batch_size=None):
  runs = {}
  for name, placement, epochs, keys in (('device', 'device', 3, {'checkpoint': True}),
                                        ('host', 'host', 3, {'checkpoint': True}),
                                        ('split', 'host', 1, {'checkpoint': True}),
                                        ('split', 'host', 3, {'resume': True})):
    cfg = _config(root, pretrained, exp, name, legs, yaw)
    cfg.update(no_epochs=epochs, training_precision=precision, **keys)
    if batch_size is not None:
      cfg['batch_size'] = batch_size
    np.random.seed(99 if 'resume' in keys else 0)                # the resumed run restores the saved state
    runs[name if 'resume' not in keys else 'resumed'] = _train(cfg, placement, device)
  return runs


def _same(a, b, what):
  for key in ('epoch_loss', 'batch_losses', 'validation'):
    assert repr(a['hist'][key]) == repr(b['hist'][key]), (what, key)
  for name, (k, bias) in a['weights'].items():
    assert np.array_equal(bits(b['weights'][name][0]), bits(k)), (what, name)
    assert np.array_equal(bits(b['weights'][name][1]), bits(bias)), (what, name)
  assert np.array_equal(bits(b['state']), bits(a['state'])) and a['state'].any(), what


def _check(runs, exp):
  ref = runs['device']
  assert ref['placement'] == 'device' and runs['host']['placement'] == 'host' == runs['resumed']['placement']
  _same(ref, runs['host'], 'host')
  _same(ref, runs['resumed'], 'resumed')
  ref_file = Wt.load(ref['hist']['weights_filename'])
  for run in ('host', 'resumed'):
    f = Wt.load(runs[run]['hist']['weights_filename'])
    for name, (k, b) in ref_file.items():
      assert np.array_equal(bits(f[name][0]), bits(k)) and np.array_equal(bits(f[name][1]), bits(b)), (run, name)
  ck = {d: np.load(os.path.join(exp, d, training.CHECKPOINT), allow_pickle=False) for d in ('device', 'host', 'split')}
  for d in ('host', 'split'):
    assert sorted(ck[d].files) == sorted(ck['device'].files)
    for key in ck['device'].files:
      assert np.array_equal(ck[d][key], ck['device'][key]), (d, key)
  log = open(os.path.join(exp, 'host', 'training.log')).read()
  assert 'in pinned host memory' in log


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('legs,yaw', CASES)
def test_host_bank_trains_the_device_bank_bits(tmp_path, dataset, legs, yaw, precision):
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  _check(_runs(root, pretrained, exp, legs, yaw, precision), exp)


@pytest.mark.parametrize('yaw', [False, True])
def test_validation_in_several_chunks_keeps_the_device_bank_bits(tmp_path, dataset, monkeypatch, yaw):
  """batch_size 2 gives slots of 4 images, so the whole network's validation streams its 11 scans through the ring
  in chunks of 4, 4 and 3, in order of first appearance in the validation pairs.  So each leg launch groups other
  images than the whole-bank encoding, which runs in bank order, and the last chunk is partial.  The histories
  (validation included), weights, accumulators and checkpoints are still the device bank's."""
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  chunks = []
  plan = image_bank.StagingRing.plan

  def recording_plan(self, steps):
    steps = list(steps)
    if steps and all(len(lists) == 1 for lists in steps):       # the validation plans: one row list per chunk
      chunks.append(([len(lists[0]) for lists in steps], self.slot_rows,
                     np.concatenate([lists[0] for lists in steps]).tolist()))
    return plan(self, steps)

  monkeypatch.setattr(image_bank.StagingRing, 'plan', recording_plan)
  _check(_runs(root, pretrained, exp, '360OutputkLegs', yaw, 'fp32', batch_size=2), exp)
  print('validation chunks (sizes, slot rows):', chunks[0])
  assert chunks and all(c == chunks[0] for c in chunks)
  sizes, slot_rows, rows = chunks[0]
  assert slot_rows == 4 and len(sizes) >= 3 and sizes[-1] < slot_rows and sum(sizes) == 11, chunks[0]
  assert rows != sorted(rows), rows                            # not the bank order of the device encoding


def _worker(rank, world, port, root, pretrained, exp, legs, out):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(0)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  try:
    runs = {}
    for placement in ('device', 'host'):
      np.random.seed(0)
      runs[placement] = _train(_config(root, pretrained, exp, placement, legs, True), placement, 0)
    with open(out % rank, 'wb') as f:
      pickle.dump(runs, f)
  finally:
    dist.destroy_process_group()


@pytest.mark.parametrize('legs', sorted(FLOWS))
def test_two_ranks_on_one_gpu_with_host_banks(tmp_path, dataset, legs):
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  out = str(tmp_path / 'rank%d.pkl')
  mp.spawn(_worker, args=(2, _free_port(), root, pretrained, exp, legs, out), nprocs=2, join=True)
  ranks = []
  for r in range(2):
    with open(out % r, 'rb') as f:
      ranks.append(pickle.load(f))
  for r in range(2):
    assert ranks[r]['host']['placement'] == 'host'
    _same(ranks[0]['device'], ranks[r]['host'], 'rank %d' % r)
  log = open(os.path.join(exp, 'host', 'training.log')).read()
  assert 'data-parallel over 2 ranks' in log and 'over 2 ranks' in log


def test_host_bank_keeps_the_images_off_the_device(tmp_path, dataset):
  """The whole network on one sequence (5 scans) and on both (11): with the host bank, the peak of torch's device
  allocations grows by no more than the validation feature bank of the larger run; with the device bank by the
  images too."""
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  peaks, n = {}, {}
  for placement in ('device', 'host'):
    for seqs in ('01', '00 01'):
      cfg = _config(root, pretrained, exp, 'mem', '360OutputkLegs', False)
      cfg.update(no_epochs=1, training_seqs=seqs)
      np.random.seed(0)
      run = _train(cfg, placement)
      peaks[placement, seqs], n[seqs] = run['peak'], run['n_images']
  assert n['00 01'] >= 2 * n['01']
  vol, img = 360 * 128 * 4, 64 * 900 * 4 * 4                    # a feature volume, a C = 4 image
  host_growth = peaks['host', '00 01'] - peaks['host', '01']
  device_growth = peaks['device', '00 01'] - peaks['device', '01']
  print('peak device allocations (bytes):', peaks, 'scans:', n)
  assert host_growth <= n['00 01'] * vol, (host_growth, n)
  assert device_growth >= (n['00 01'] - n['01']) * img, (device_growth, n)


@pytest.mark.parametrize('legs,yaw', CASES)
def test_a_small_device_budget_chooses_the_host_bank(tmp_path, dataset, monkeypatch, legs, yaw):
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  budget = {}

  def small_free(eng):                    # a device budget below the bank's size once the working set is taken
    budget['free'] = 1 << 20
    return budget['free']

  monkeypatch.setattr(image_bank, 'free_device_bytes', small_free)
  cfg = _config(root, pretrained, exp, 'auto', legs, yaw)
  cfg.update(no_epochs=1)
  np.random.seed(0)
  run = _train(cfg, None)
  assert budget and run['placement'] == 'host' and len(run['hist']['epoch_loss']) == 1
  assert np.isfinite(run['hist']['epoch_loss'][0])
  log = open(os.path.join(exp, 'auto', 'training.log')).read()
  assert 'device budget' in log and 'on the host, pinned' in log
