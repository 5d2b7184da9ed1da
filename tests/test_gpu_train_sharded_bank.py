"""A training image bank sharded over the GPUs of a node (overlapnet_b200.image_bank.ShardedImageBank):
ovn_gather_rows against torch indexing and its refusals, two gloo processes sharing one GPU that map each other's
shards, both flows forced to ``image_bank='sharded'`` against the device bank at the same world size on 1, 2 and 3
ranks bit for bit (weight files, Engine.train_state, histories with the validation statistics, checkpoints), a
sharded two-rank run resumed on one rank, the scans each rank loads, the automatic choice of the sharded bank under
a small device budget, and NCCL on two GPUs."""
import copy
import ctypes as C
import os
import pickle

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from overlapnet_b200 import _cabi, image_bank, training
from overlapnet_b200 import weights as Wt
from overlapnet_b200._cabi import OvnError
from overlapnet_b200.engine import Engine
from overlapnet_b200.infer import Infer
from test_gpu_train_dp import FLOWS, _config, _free_port, bits, dataset  # noqa: F401

pytestmark = pytest.mark.gpu

CASES = [('360OutputkLegs', False), ('360OutputkLegs', True), ('360OutputkLegsFixed', True)]
MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
USE = {4: {}, 25: {'use_class_probabilities': True, 'use_intensity': True}}


# ---- ovn_gather_rows in one process ------------------------------------------------------------------------
def _engine(C_, precision='fp32'):
  eng = Engine(use=USE[C_], model=MODEL, precision=precision, max_batch_scans=4, max_batch_pairs=8)
  assert eng.C == C_
  return eng


def _shards(eng, sizes, seed):
  """Own shards of ``sizes`` images filled with random values: (views, device addresses, first rows)."""
  g = torch.Generator(device=eng.device).manual_seed(seed)
  views, ptrs = [], []
  for k in sizes:
    v, p, ipc = eng.shard_create(k)
    assert len(ipc) == 64 and (k == 0 or v.data_ptr() == p) and tuple(v.shape) == (k, eng.H, eng.W, eng.C)
    v.copy_(torch.rand(v.shape, generator=g, device=eng.device))
    views.append(v)
    ptrs.append(p)
  return views, ptrs, [0] + list(np.cumsum(sizes))


@pytest.mark.parametrize('C_,precision', [(4, 'f16_tc'), (25, 'fp32')])
def test_gather_rows_matches_torch_indexing(C_, precision):
  """1-3 shards of uneven sizes, rows repeated and out of order, n = 1, 7, 64 and (C = 4) past the 1024 rows of one
  launch: the slot equals torch indexing of the whole bank bit for bit, in ceil(n / 1024) launches."""
  eng = _engine(C_, precision)
  rng = np.random.default_rng(C_)
  eng.profile_enable(True)
  for sizes in ([5], [3, 1], [2, 4, 3]):
    views, ptrs, first = _shards(eng, sizes, sum(sizes))
    bank = torch.cat(views)
    for n in (1, 7, 64) + ((1100,) if C_ == 4 and len(sizes) == 2 else ()):
      rows = rng.integers(0, bank.shape[0], n)
      if n > 1:
        rows[-1] = rows[0]                                       # a repeated row
      out = torch.full((n,) + tuple(bank.shape[1:]), float('nan'), device=eng.device)
      eng.profile_read('gather_rows')
      n0 = eng.launch_count()
      eng.gather_rows(ptrs, first, rows, out)
      assert eng.launch_count() == n0 + -(-n // 1024)
      torch.cuda.synchronize()
      ms, launches = eng.profile_read('gather_rows')
      assert launches == -(-n // 1024) and ms > 0
      ref = bank[torch.from_numpy(rows).to(eng.device)]
      assert torch.equal(out.view(torch.int32), ref.view(torch.int32)), (sizes, n)
      del out, ref
    del views, bank
    for p in ptrs:
      eng.shard_close(p)
  eng.check()
  eng.close()


def _raw_gather(eng, shards, first, row_bytes, rows, n, out):
  s = (C.c_void_p * len(shards))(*shards)
  f = np.ascontiguousarray(first, np.int64)
  r = np.ascontiguousarray(rows, np.int64)
  return _cabi.lib().ovn_gather_rows(eng._h, s, f.ctypes.data_as(C.c_void_p), len(shards), int(row_bytes),
                                     r.ctypes.data_as(C.c_void_p), int(n), C.c_void_p(out.data_ptr()), eng._stream())


def test_gather_rows_refuses_bad_arguments():
  """Each refused call is OVN_ERR_INVALID_ARG with a message, copies nothing into a sentinel-filled slot and leaves
  the handle working; a shard that is no shard of the handle is refused by ovn_shard_close."""
  eng = _engine(4)
  views, ptrs, first = _shards(eng, [2, 3], 1)
  rb = views[0][0].numel() * 4
  out = torch.full((4,) + tuple(views[0].shape[1:]), -7.0, device=eng.device)
  bad = [('row -1', ptrs, first, rb, [0, -1], 2), ('row past the bank', ptrs, first, rb, [5], 1),
         ('row_bytes % 16', ptrs, first, rb - 4, [0], 1), ('row_bytes 0', ptrs, first, 0, [0], 1),
         ('misaligned shard', [ptrs[0], ptrs[1] + 4], first, rb, [0], 1),
         ('NULL shard', [ptrs[0], 0], first, rb, [0], 1), ('n < 0', ptrs, first, rb, [0], -1),
         ('decreasing first', ptrs, [0, 4, 3], rb, [0], 1), ('first[0] != 0', ptrs, [1, 2, 5], rb, [1], 1)]
  L = _cabi.lib()
  for what, shards, f, row_bytes, rows, n in bad:
    st = _raw_gather(eng, shards, f, row_bytes, rows, n, out)
    assert L.ovn_status_string(st) == b'OVN_ERR_INVALID_ARG', what
    assert L.ovn_last_error(eng._h), what
    torch.cuda.synchronize()
    assert bool((out == -7.0).all()), what
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.shard_close(out.data_ptr())
  eng.gather_rows(ptrs, first, [4, 0, 2, 4], out)              # the handle still works
  assert torch.equal(out, torch.cat(views)[[4, 0, 2, 4]])
  eng.check()
  eng.close()


# ---- two processes sharing one GPU -------------------------------------------------------------------------
class _PatternInfer:
  """What ShardedImageBank reads of an Infer: the handle and a cue loader whose image of scan s is a fixed
  function of s alone, so every rank knows every row; it records the scans it loads."""

  def __init__(self, eng):
    self._engine, self.seq, self.loaded = eng, None, []

  @staticmethod
  def image(eng, seq, name):
    i = int(seq) * 1000 + int(name)
    return (np.arange(eng.H * eng.W * eng.C, dtype=np.float32).reshape(eng.H, eng.W, eng.C) * 1e-3 + i)

  def _prepare_inputs(self, names):
    self.loaded.extend((self.seq, n) for n in names)
    return np.stack([self.image(self._engine, self.seq, n) for n in names])


def _gather_worker(rank, world, port, out):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(0)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  res = {}
  try:
    from overlapnet_b200 import data_parallel
    from overlapnet_b200.image_bank import bank_rows
    eng = _engine(4)
    infer = _PatternInfer(eng)
    keys = {('00', '%06d' % i) for i in range(3)} | {('01', '%06d' % i) for i in range(2)}
    rows = bank_rows(keys)
    bank = image_bank.ShardedImageBank(infer, rows, data_parallel.default_group())
    res['first'], res['rank_rows'], res['loaded'] = bank.first, bank.rank_rows, sorted(infer.loaded)
    res['mine'] = sorted(k for k, r in rows.items() if bank.first[rank] <= r < bank.first[rank + 1])
    res['open'] = eng.open_shard_count()
    order = [4, 0, 3, 3, 1, 2, 0] if rank == 0 else [2, 2, 4, 1, 0]   # both ranks' rows, repeated, out of order
    slot = torch.empty((len(order), eng.H, eng.W, eng.C), device=eng.device)
    bank.stage(order, slot)
    by_row = {r: k for k, r in rows.items()}
    ref = np.stack([_PatternInfer.image(eng, *by_row[r]) for r in order])
    res['exact'] = bool(np.array_equal(slot.cpu().numpy().view(np.uint32), ref.view(np.uint32)))
    try:                                                           # a zeroed IPC handle
      eng.shard_open(bytes(64))
      res['zeroed'] = None
    except OvnError as e:
      res['zeroed'] = str(e)
    slot.zero_()
    bank.stage(order, slot)                                        # the handle still works
    res['after_zeroed'] = bool(np.array_equal(slot.cpu().numpy().view(np.uint32), ref.view(np.uint32)))
    bank.close()
    res['open_after_close'] = eng.open_shard_count()
    eng.check()
    eng.close()
  finally:
    with open(out % rank, 'wb') as f:
      pickle.dump(res, f)
    dist.destroy_process_group()


def test_two_processes_gather_each_others_rows(tmp_path):
  out = str(tmp_path / 'rank%d.pkl')
  mp.spawn(_gather_worker, args=(2, _free_port(), out), nprocs=2, join=True)
  for r in range(2):
    with open(out % r, 'rb') as f:
      res = pickle.load(f)
    assert res['first'] == [0, 3, 5] and res['rank_rows'] == (3, 2)[r]
    assert res['loaded'] == res['mine'], r                        # each rank loaded exactly its own scans
    assert res['open'] == 1 and res['exact'] and res['after_zeroed'], r
    assert res['zeroed'] is not None and 'OVN_ERR_CUDA' in res['zeroed'] and 'cudaIpcOpenMemHandle' in res['zeroed']
    assert res['open_after_close'] == 0


# ---- training ----------------------------------------------------------------------------------------------
def _train(cfg, placement, device=None):
  """One training run with the flow's image bank forced to ``placement`` (None: chosen): its history, the
  handle's weights and Adagrad state, the placement, and for a sharded bank the shard's shape, the scans this
  process loaded through the cue loader and the mappings left open after the run."""
  module, name, train = FLOWS[cfg['model']['legsType']]
  base = getattr(module, name)
  kept, loaded = [], []
  prepare = Infer._prepare_inputs

  class Keep(base):
    def __init__(self, *args, **kw):
      if placement is not None:
        kw['image_bank'] = placement
      super().__init__(*args, **kw)
      kept.append(self)
      if self.image_bank == 'sharded':
        self.shard = (tuple(self.images.images.shape), self.images.first, self.images.own == self.images.images.data_ptr())

  def counting(self, names):
    loaded.extend((self.seq, n) for n in names)
    return prepare(self, names)

  setattr(module, name, Keep)
  Infer._prepare_inputs = counting
  try:
    hist = train(copy.deepcopy(cfg), device)
  finally:
    setattr(module, name, base)
    Infer._prepare_inputs = prepare
  flow = kept[0]
  eng = flow.eng
  out = {'hist': hist, 'weights': eng.get_weights(), 'state': eng.train_state(base.whole_network).cpu().numpy(),
         'placement': flow.image_bank, 'rows': flow.image_rows, 'loaded': loaded}
  if flow.image_bank == 'sharded':
    out.update(shard=flow.shard, closed=flow.images.closed, open_after=eng.open_shard_count())
  eng.close()
  return out


def _same(a, b, what):
  for key in ('epoch_loss', 'batch_losses', 'validation'):
    assert repr(a['hist'][key]) == repr(b['hist'][key]), (what, key)
  for name, (k, bias) in a['weights'].items():
    assert np.array_equal(bits(b['weights'][name][0]), bits(k)), (what, name)
    assert np.array_equal(bits(b['weights'][name][1]), bits(bias)), (what, name)
  assert np.array_equal(bits(b['state']), bits(a['state'])) and a['state'].any(), what


def _same_files(exp, a, b):
  """The weight files and checkpoints of the runs in directories a and b agree bit for bit."""
  fa = Wt.load(os.path.join(exp, a, _weight_name(exp, a)))
  fb = Wt.load(os.path.join(exp, b, _weight_name(exp, b)))
  for name, (k, bias) in fa.items():
    assert np.array_equal(bits(fb[name][0]), bits(k)) and np.array_equal(bits(fb[name][1]), bits(bias)), (b, name)
  ca = np.load(os.path.join(exp, a, training.CHECKPOINT), allow_pickle=False)
  cb = np.load(os.path.join(exp, b, training.CHECKPOINT), allow_pickle=False)
  assert sorted(ca.files) == sorted(cb.files)
  for key in ca.files:
    assert np.array_equal(ca[key], cb[key]), (b, key)


def _weight_name(exp, d):
  names = [f for f in os.listdir(os.path.join(exp, d)) if f.endswith('.weight')]
  assert len(names) == 1, names
  return names[0]


def _sharded_ok(run, world, rank):
  """The sharded run held ceil or floor(n / world) images on this rank, in its own shard, and closed every mapping."""
  shape, first, own = run['shard']
  n = len(run['rows'])
  assert shape[0] == first[rank + 1] - first[rank] in (n // world, -(-n // world)) and own
  assert run['closed'] and run['open_after'] == 0


def _cfg(root, pretrained, exp, name, legs, yaw, precision='fp32', **kw):
  cfg = _config(root, pretrained, exp, name, legs, yaw)
  cfg.update(training_precision=precision, checkpoint=True, **kw)
  return cfg


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('legs,yaw', CASES)
def test_one_rank_sharded_bank_trains_the_device_bank_bits(tmp_path, dataset, legs, yaw, precision):
  """One process: the bank is one own shard, gathered into the ring's slots."""
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  runs = {}
  for placement in ('device', 'sharded'):
    np.random.seed(0)
    runs[placement] = _train(_cfg(root, pretrained, exp, placement, legs, yaw, precision), placement)
  assert runs['device']['placement'] == 'device' and runs['sharded']['placement'] == 'sharded'
  _same(runs['device'], runs['sharded'], 'sharded')
  _sharded_ok(runs['sharded'], 1, 0)
  _same_files(exp, 'device', 'sharded')
  log = open(os.path.join(exp, 'sharded', 'training.log')).read()
  assert 'sharded over the GPUs of 1 ranks' in log


def test_validation_in_several_chunks_keeps_the_device_bank_bits(tmp_path, dataset):
  """batch_size 2 gives slots of 4 images: the whole network's validation gathers its 11 scans from the shard in
  several chunks, and the bits are still the device bank's."""
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  runs = {}
  for placement in ('device', 'sharded'):
    np.random.seed(0)
    runs[placement] = _train(_cfg(root, pretrained, exp, placement, '360OutputkLegs', False, batch_size=2), placement)
  _same(runs['device'], runs['sharded'], 'sharded')
  _same_files(exp, 'device', 'sharded')


def _rank_worker(rank, world, port, backend, jobs, out):
  """Runs ``jobs`` = [(key, cfg, placement, patch)] in order on this rank; patch 'budget:<bytes>' makes the device
  budget of every rank that many bytes (free memory = budget, working set = 0)."""
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  device = rank if backend == 'nccl' else 0
  torch.cuda.set_device(device)
  dist.init_process_group(backend, rank=rank, world_size=world)
  try:
    runs = {}
    for key, cfg, placement, patch in jobs:
      saved = image_bank.free_device_bytes, image_bank.working_set_bytes
      if patch:
        budget = int(patch.split(':')[1])
        image_bank.free_device_bytes = lambda eng: budget
        image_bank.working_set_bytes = lambda *a, **kw: 0
      try:
        np.random.seed(0)
        runs[key] = _train(cfg, placement, device)
      finally:
        image_bank.free_device_bytes, image_bank.working_set_bytes = saved
    with open(out % rank, 'wb') as f:
      pickle.dump(runs, f)
  finally:
    dist.destroy_process_group()


def _spawn(tmp_path, world, jobs, backend='gloo'):
  out = str(tmp_path / 'rank%d.pkl')
  mp.spawn(_rank_worker, args=(world, _free_port(), backend, jobs, out), nprocs=world, join=True)
  ranks = []
  for r in range(world):
    with open(out % r, 'rb') as f:
      ranks.append(pickle.load(f))
  return ranks


def _check_ranks(ranks, exp, world, keys):
  """Every rank's sharded run against rank 0's device run, its shard and its loads."""
  for key in keys:
    ref = ranks[0][key + '/device']
    assert ref['placement'] == 'device'
    for r in range(world):
      run = ranks[r][key + '/sharded']
      assert run['placement'] == 'sharded'
      _same(ref, run, (key, r))
      _sharded_ok(run, world, r)
      if key.startswith('360OutputkLegs-False'):               # only the image bank loads scans in this flow
        shape, first, _ = run['shard']
        mine = sorted(k for k, row in run['rows'].items() if first[r] <= row < first[r + 1])
        assert sorted(run['loaded']) == mine, (key, r)
    _same_files(exp, key + '-device', key + '-sharded')


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('world', [2, 3])
def test_ranks_sharded_bank_trains_the_device_bank_bits(tmp_path, dataset, world, precision):
  """Two and three gloo ranks sharing one GPU (11 scans: shards of 6 and 5, or 4, 4 and 3), each flow: the sharded
  bank against the device bank at the same world size, every rank; each rank loads only its own scans."""
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  jobs, keys = [], []
  for legs, yaw in CASES:
    key = '%s-%s' % (legs, yaw)
    keys.append(key)
    for placement in ('device', 'sharded'):
      jobs.append((key + '/' + placement, _cfg(root, pretrained, exp, key + '-' + placement, legs, yaw, precision),
                   placement, None))
  ranks = _spawn(tmp_path, world, jobs)
  _check_ranks(ranks, exp, world, keys)
  log = open(os.path.join(exp, keys[0] + '-sharded', 'training.log')).read()
  assert 'sharded over the GPUs of %d ranks' % world in log and 'data-parallel over %d ranks' % world in log


@pytest.mark.parametrize('legs,yaw', [('360OutputkLegs', True), ('360OutputkLegsFixed', True)])
def test_three_ranks_with_gradient_chunks_give_the_one_rank_bits(tmp_path, dataset, legs, yaw):
  """gradient_chunks 4: the sharded bank on three ranks trains the bits of the device bank on one."""
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  cfg = _cfg(root, pretrained, exp, 'sharded3', legs, yaw, gradient_chunks=4)
  ranks = _spawn(tmp_path, 3, [('sharded', cfg, 'sharded', None)])
  np.random.seed(0)
  one = _train(_cfg(root, pretrained, exp, 'device1', legs, yaw, gradient_chunks=4), 'device')
  for r in range(3):
    _same(one, ranks[r]['sharded'], ('rank', r))
    _sharded_ok(ranks[r]['sharded'], 3, r)
  _same_files(exp, 'device1', 'sharded3')


def test_two_rank_sharded_run_resumed_on_one_rank(tmp_path, dataset):
  """gradient_chunks 4: a two-rank sharded run stopped after epoch 1, resumed on one rank with the device bank,
  gives the uninterrupted one-rank run's bits."""
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  legs, yaw = '360OutputkLegs', True
  split = _cfg(root, pretrained, exp, 'split', legs, yaw, gradient_chunks=4, no_epochs=1)
  ranks = _spawn(tmp_path, 2, [('split', split, 'sharded', None)])
  assert ranks[0]['split']['placement'] == 'sharded' and len(ranks[0]['split']['hist']['epoch_loss']) == 1
  np.random.seed(99)                                             # the resumed run restores the saved state
  resumed = _train(_cfg(root, pretrained, exp, 'split', legs, yaw, gradient_chunks=4, resume=True), 'device')
  np.random.seed(0)
  straight = _train(_cfg(root, pretrained, exp, 'straight', legs, yaw, gradient_chunks=4), 'device')
  _same(straight, resumed, 'resumed')
  _same_files(exp, 'straight', 'split')


def test_a_small_device_budget_chooses_the_sharded_bank(tmp_path, dataset):
  """Two ranks whose budget holds one shard (6 images) but not the bank (11) choose the sharded bank and train; a
  budget below one shard chooses the host bank."""
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  img = 64 * 900 * 4 * 4
  jobs = [('sharded', _cfg(root, pretrained, exp, 'auto-sharded', '360OutputkLegs', True, no_epochs=1), None,
           'budget:%d' % (8 * img)),
          ('host', _cfg(root, pretrained, exp, 'auto-host', '360OutputkLegs', True, no_epochs=1), None,
           'budget:%d' % (5 * img))]
  ranks = _spawn(tmp_path, 2, jobs)
  for r in range(2):
    assert ranks[r]['sharded']['placement'] == 'sharded' and ranks[r]['host']['placement'] == 'host'
    for key in ('sharded', 'host'):
      assert np.isfinite(ranks[r][key]['hist']['epoch_loss'][0])
    _sharded_ok(ranks[r]['sharded'], 2, r)
  _same(ranks[0]['sharded'], ranks[0]['host'], 'sharded against host')
  log = open(os.path.join(exp, 'auto-sharded', 'training.log')).read()
  assert "sharded over the ranks' GPUs" in log and 'smallest over the ranks' in log
  log = open(os.path.join(exp, 'auto-host', 'training.log')).read()
  assert 'on the host, pinned' in log and 'in pinned host memory' in log


def test_two_gpus_nccl_sharded_bank(tmp_path, dataset):
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  root, pretrained = dataset
  exp = str(tmp_path / 'exp')
  key = '360OutputkLegs-True'
  jobs = [(key + '/' + p, _cfg(root, pretrained, exp, key + '-' + p, '360OutputkLegs', True), p, None)
          for p in ('device', 'sharded')]
  _check_ranks(_spawn(tmp_path, 2, jobs, 'nccl'), exp, 2, [key])
