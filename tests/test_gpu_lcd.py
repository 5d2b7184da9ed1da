"""The online loop-closure flow on the GPU (SURVEY 8f-1; demo/demo3_lcd.py:85-123 on top of
Infer.infer_multiple, infer.py:162-203): 230 frames through ``LoopClosureDetector`` + the real
``Infer`` with its incrementally prepared GPU-resident bank, checked against ``InferRef`` (the oracle's
restatement of the reference's call semantics) on gated candidates; and the same flow with the bank
sharded over two GPUs (``ShardedInfer``, NCCL) against the single-GPU run."""
import copy
import os
import socket

import numpy as np
import pytest
import torch

from oracle import network as N
from oracle.infer_ref import InferRef
from overlapnet_b200 import lcd, synth, weights as W

pytestmark = pytest.mark.gpu

MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
         'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
         'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
         'additional_unsymmetric_layer3a': True}
N_FRAMES, LAP = 230, 200


def trajectory(n=N_FRAMES):
  t = np.arange(n) * 0.6
  side = 30.0
  s = t % (4 * side)
  x = np.where(s < side, s, np.where(s < 2 * side, side, np.where(s < 3 * side, 3 * side - s, 0.0)))
  y = np.where(s < side, 0.0, np.where(s < 2 * side, s - side, np.where(s < 3 * side, side, 4 * side - s)))
  return np.stack([x, y], 1)


def frame_cloud(i):
  """Frame i >= LAP revisits the place of frame i - LAP, seen under another heading."""
  base = synth.kitti_like_cloud(3000 + (i % LAP), n_points=20000)
  if i < LAP:
    return base
  ang = np.deg2rad(10.0 + (i % 7) * 20.0)
  c, s = np.cos(ang), np.sin(ang)
  pts = base.copy()
  pts[:, 0], pts[:, 1] = c * base[:, 0] - s * base[:, 1], s * base[:, 0] + c * base[:, 1]
  return pts


def make_dataset(root):
  """Preprocessed cue files laid out like the reference's (depth/ normal/ %06d.npy), written by the
  product's own projection kernels (bit-exact against the reference, tests/test_gpu_projection.py)."""
  from overlapnet_b200.engine import Engine
  seq = os.path.join(root, '07')
  os.makedirs(os.path.join(seq, 'depth'), exist_ok=True)
  os.makedirs(os.path.join(seq, 'normal'), exist_ok=True)
  eng = Engine(model=MODEL, precision='fp32', max_batch_scans=16, max_batch_pairs=1)
  for s0 in range(0, N_FRAMES, 16):
    ids = list(range(s0, min(N_FRAMES, s0 + 16)))
    x = eng.preprocess(eng.upload_clouds([frame_cloud(i) for i in ids])).cpu().numpy()
    for k, i in enumerate(ids):
      np.save(os.path.join(seq, 'depth', '%06d.npy' % i), x[k, :, :, 0])
      np.save(os.path.join(seq, 'normal', '%06d.npy' % i), x[k, :, :, 1:4])
  eng.close()
  w = N.glorot_weights(4, MODEL, seed=5)
  # spread the overlaps over (0,1) (tests/test_gpu_network.py): Dense rescaled on a few (reference, current) pairs
  ids = [LAP + 3, 3, 4, 50, 120, LAP + 10, 10]
  imgs = np.stack([np.concatenate([np.load(os.path.join(seq, 'depth', '%06d.npy' % i))[..., None],
                                   np.load(os.path.join(seq, 'normal', '%06d.npy' % i))], -1) for i in ids])
  fv = N.leg_forward(imgs.astype(np.float32), w, MODEL)
  li, ri = np.array([1, 2, 3, 4, 6, 1]), np.array([0, 0, 0, 0, 5, 5])
  _, _, _, z0 = N.heads_forward(fv[li], fv[ri], w, MODEL, return_logit=True)
  w = N.spread_dense(w, z0, target_std=1.5)
  wpath = os.path.join(root, 'weights.npz')
  W.save_npz(wpath, w)
  cfg = {'pretrained_weightsfilename': wpath, 'use_depth': True, 'use_normals': True,
         'use_class_probabilities': False, 'use_class_probabilities_pca': False, 'use_intensity': False,
         'data_root_folder': root, 'infer_seqs': '07', 'batch_size': 16, 'model': copy.deepcopy(MODEL)}
  return cfg, w


class Recorder:
  """Passes infer_multiple through and keeps what was asked and answered."""

  def __init__(self, infer):
    self.infer, self.log = infer, {}

  def infer_multiple(self, idx, refs):
    res = self.infer.infer_multiple(idx, refs)
    if res is not None:
      self.log[int(idx)] = (np.asarray(refs).copy(), np.atleast_1d(res[0]).copy(), res[1].copy())
    return res


def run_lcd(infer):
  rec = Recorder(infer)
  det = lcd.LoopClosureDetector(rec)
  traj = trajectory()
  cov = np.zeros((6, 6))
  cov[:2, :2] = np.diag([4.0, 4.0])
  found = {}
  for i in range(N_FRAMES):
    r = det.step(i, traj[i], cov)
    if r is not None:
      found[i] = r
  return rec.log, found


@pytest.fixture(scope='module')
def dataset(tmp_path_factory):
  return make_dataset(str(tmp_path_factory.mktemp('lcd')))


def test_lcd_on_growing_gpu_bank_matches_reference_semantics(dataset):
  from overlapnet_b200.infer import Infer
  cfg, w = dataset
  inf = Infer(copy.deepcopy(cfg), precision='f16_tc')
  log, found = run_lcd(inf)
  assert len(inf.feature_volumes) == N_FRAMES                   # one appended volume per frame, in order
  scored = sorted(log)
  assert scored and min(scored) >= 150 and len(scored) >= 20    # candidates only exist once the loop closes (100 frames + 50 m)
  # oracle: InferRef fed with exactly the frames involved in a few scored queries
  ref = InferRef(copy.deepcopy(cfg), w)
  n_checked = 0
  for idx in (scored[0], scored[len(scored) // 2], scored[-1]):
    refs, ov, yaw = log[idx]
    pick = np.unique(np.linspace(0, len(refs) - 1, 3).astype(int))
    fv = ref.create_feature_volumes(['%06d' % idx] + ['%06d' % int(refs[k]) for k in pick])
    ov_r, yaw_r, corr_r = N.heads_forward(fv[1:], np.repeat(fv[:1], len(pick), 0), w, MODEL)   # LEFT = refs, RIGHT = current
    assert np.abs(ov[pick] - ov_r).max() <= 1e-3, (idx, ov[pick], ov_r)
    for k, p in enumerate(pick):
      if int(yaw[p]) != int(yaw_r[k]):
        kg, kr = 180 - int(yaw[p]), 180 - int(yaw_r[k])
        assert corr_r[k, kr] - corr_r[k, kg] <= 2e-4 * np.abs(corr_r[k]).max()
    n_checked += len(pick)
  assert n_checked >= 6
  # the driver's decision rule on the recorded answers (demo3_lcd.py:118-120)
  for idx, (refs, ov, _) in log.items():
    if ov.max() > 0.3:
      assert found[idx] == int(refs[np.argmax(ov)])
    else:
      assert idx not in found
  # same frames through infer_multiple_vs_multiple give the same numbers as the growing bank
  idx = scored[-1]
  refs, ov, yaw = log[idx]
  names = ['%06d' % idx] + ['%06d' % int(r) for r in refs[:3]]
  ov2, yaw2 = inf.infer_multiple_vs_multiple(names, [0, 0, 0][:len(names) - 1], [1, 2, 3][:len(names) - 1])
  assert np.abs(np.atleast_1d(ov2) - ov[:len(names) - 1]).max() <= 1e-3      # another feature centre, same gate
  assert np.array_equal(yaw2, yaw[:len(names) - 1])


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _sharded_worker(rank, world, port, cfg, out_path):
  import torch.distributed as dist
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(rank)
  dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
  from overlapnet_b200.sharded_infer import ShardedInfer
  inf = ShardedInfer(copy.deepcopy(cfg), precision='f16_tc', device=rank)
  log, found = run_lcd(inf)
  assert inf.local_frames == list(range(rank, N_FRAMES, world))
  if rank == 0:
    keys = sorted(log)
    np.savez(out_path, keys=np.array(keys), found_k=np.array(sorted(found)), found_v=np.array([found[k] for k in sorted(found)]),
             **{'ov_%d' % k: log[k][1] for k in keys}, **{'yaw_%d' % k: log[k][2] for k in keys})
  else:
    assert not log
  dist.barrier()
  dist.destroy_process_group()


def test_lcd_on_bank_sharded_over_two_gpus(dataset, tmp_path):
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  import torch.multiprocessing as mp
  from overlapnet_b200.infer import Infer
  cfg, _ = dataset
  out = str(tmp_path / 'sharded.npz')
  mp.spawn(_sharded_worker, args=(2, _free_port(), cfg, out), nprocs=2, join=True)
  got = np.load(out)
  log, found = run_lcd(Infer(copy.deepcopy(cfg), precision='f16_tc'))
  assert sorted(log) == got['keys'].tolist()
  for k in log:
    assert np.array_equal(got['ov_%d' % k], log[k][1])             # every rank calibrates on frame 0: bit-identical
    assert np.array_equal(got['yaw_%d' % k], log[k][2])
  assert sorted(found) == got['found_k'].tolist()


def _search_worker(rank, world, port, out_path):
  import torch.distributed as dist
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(rank)
  dev = torch.device('cuda', rank)
  dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
  from overlapnet_b200.engine import Engine
  from overlapnet_b200.search import ShardedSearch, engine_heads_fn, engine_rows_fn, shard_range
  n_total = 13                                             # odd: shards of 7 and 6
  bank_np = synth.feature_volumes(4, n_total)[:, 0]
  w = N.glorot_weights(4, MODEL, seed=8)
  eng = Engine(model=MODEL, precision='f16_tc', device=rank, max_batch_scans=1, max_batch_pairs=8)
  eng.load_weights(w)
  eng.calibrate(torch.from_numpy(bank_np[0]))              # the same numeric centres on every rank
  lo, hi = shard_range(n_total, rank, world)
  shard = torch.from_numpy(bank_np[lo:hi].copy()).to(dev)
  res = {}
  for transport in ('symm', 'collective'):
    ss = ShardedSearch(engine_heads_fn(eng), shard, n_total, transport=transport)
    assert ss.transport == transport
    q = torch.from_numpy(bank_np[5].copy()).to(dev) if rank == 0 else torch.zeros((360, 128), device=dev)
    for rep in range(3):                                   # repeated queries reuse the buffers / flags
      r = ss.query(q)
    if rank == 0:
      res[transport] = (r[0].cpu().numpy(), r[1].cpu().numpy())
    else:
      assert r is None
  ap = ss.all_pairs(rows_fn=engine_rows_fn(eng))
  eng.check()
  if rank == 0:
    np.savez(out_path, symm_ov=res['symm'][0], symm_yaw=res['symm'][1], coll_ov=res['collective'][0],
             coll_yaw=res['collective'][1], ap_ov=ap[0].cpu().numpy(), ap_yaw=ap[1].cpu().numpy())
  dist.barrier()
  dist.destroy_process_group()


def test_sharded_search_and_all_pairs_on_two_gpus(tmp_path):
  """ShardedSearch on NCCL / CUDA: the peer-memory transport ('symm': kernels read the query from and
  write their results into rank 0's memory, own signal kernels) and the collective fallback give exactly
  what one GPU computes; so do the all-pairs rows scored with ovn_heads_rows_vs_bank."""
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  import torch.multiprocessing as mp
  from overlapnet_b200.engine import Engine
  out = str(tmp_path / 'search.npz')
  mp.spawn(_search_worker, args=(2, _free_port(), out), nprocs=2, join=True)
  got = np.load(out)
  n_total = 13
  bank_np = synth.feature_volumes(4, n_total)[:, 0]
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=8)
  eng.load_weights(N.glorot_weights(4, MODEL, seed=8))
  eng.calibrate(torch.from_numpy(bank_np[0]))
  bank = torch.from_numpy(bank_np).to(eng.device)
  ov, yaw, _ = eng.heads_1vsN(bank, bank[5], n_cand=n_total)
  for tag in ('symm', 'coll'):
    assert np.array_equal(got[tag + '_ov'], ov.cpu().numpy()) and np.array_equal(got[tag + '_yaw'], yaw.cpu().numpy())
  assert int(yaw[5]) == 0
  ap_ov, ap_yaw = eng.heads_rows_vs_bank(bank, 0, n_total)
  eng.check()
  assert np.array_equal(got['ap_ov'], ap_ov.cpu().numpy()) and np.array_equal(got['ap_yaw'], ap_yaw.cpu().numpy())
  # row i = query i against every candidate j (LEFT = bank[j], RIGHT = bank[i]); the head is not symmetric
  o2, y2, _ = eng.heads(bank, torch.tensor([3, 7], dtype=torch.int32), torch.tensor([7, 3], dtype=torch.int32))
  assert np.array_equal(ap_ov.cpu().numpy()[[7, 3], [3, 7]], o2.cpu().numpy())
  assert np.array_equal(np.diag(ap_yaw.cpu().numpy()), np.zeros(n_total, np.int32))
  eng.close()
