"""Loop-closure evaluation on the GPU: k_rows_topk against a NumPy lexsort on crafted rows, ovn_heads_prefix_topk
against ovn_heads_1vsN plus a NumPy top-k, bit for bit, the refusals, evaluate_clouds against a host composition
on a synthetic two-lap sequence, and two ranks against one."""
import copy
import os
import socket

import numpy as np
import pytest
import torch

from oracle import network as N
from overlapnet_b200 import lcd_eval, synth, weights as W
from overlapnet_b200._cabi import OvnError, lib
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
         'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
         'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
         'additional_unsymmetric_layer3a': True}


def numpy_topk(ov, yaw, n, k):
  """The records' definition: overlap descending (NaN first, -0 == +0), then index ascending."""
  rows = ov.shape[0]
  t_ov = np.full((rows, k), -1.0, np.float32)
  t_idx = np.full((rows, k), -1, np.int32)
  t_yaw = np.zeros((rows, k), np.int32)
  for r in range(rows):
    v = ov[r, :n[r]]
    nan = np.isnan(v)
    key = np.where(nan, 0.0, v.astype(np.float64)) + 0.0
    order = np.lexsort((np.arange(n[r]), -key, ~nan))[:k]
    m = order.size
    t_ov[r, :m], t_idx[r, :m], t_yaw[r, :m] = v[order], order, yaw[r, :n[r]][order]
  return t_ov, t_idx, t_yaw


def same(a, b):
  return all(np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32)) for x, y in zip(a, b))


def _engine(precision='f16_tc', seed=3, max_batch_pairs=1101):
  eng = Engine(model=MODEL, precision=precision, max_batch_scans=1, max_batch_pairs=max_batch_pairs)
  eng.load_weights(N.glorot_weights(4, MODEL, seed=seed))
  return eng


@pytest.mark.parametrize('k', [1, 5, 32])
def test_rows_topk_equals_numpy_lexsort(k):
  rng = np.random.default_rng(k)
  lengths = [0, 1, max(k - 1, 0), k, 4541, 100000, 37]
  stride = max(lengths)
  ov = np.round(rng.random((len(lengths), stride)) * 8).astype(np.float32) / 8      # many ties
  ov[6, :37] = rng.choice(np.array([0.0, -0.0, 0.5, np.nan, -np.nan, np.inf, -np.inf, -1.0], np.float32), 37)
  ov[4, [17, 3000, 4000]] = np.nan                                                 # NaN ranks first
  ov[5, 99999] = np.inf
  yaw = rng.integers(-180, 180, ov.shape).astype(np.int32)
  eng = _engine()
  d_ov, d_yaw = torch.from_numpy(ov).cuda(), torch.from_numpy(yaw).cuda()
  eng.profile_enable(True)
  got = [t.cpu().numpy() for t in eng.rows_topk(d_ov, d_yaw, lengths, k)]
  ms, launches = eng.profile_read('rows_topk')
  eng.check()
  assert launches == 1
  want = numpy_topk(ov, yaw, lengths, k)
  assert same(got, want), (got, want)
  eng.close()


def bank_with_duplicates(n=1101):
  fv = synth.feature_volumes(11, 32)[:, 0]
  src = np.arange(n) % 32
  roll = (np.arange(n) // 32) * 7
  bank = np.stack([np.roll(fv[s], r, axis=0) for s, r in zip(src, roll)])
  bank[600:640] = bank[0:40]                                   # duplicated volumes: tied overlaps in a row
  return bank


@pytest.mark.parametrize('precision,prepared', [('f16_tc', True), ('f16_tc', False), ('fp32', False)])
def test_heads_prefix_topk_equals_1vsN_and_numpy(precision, prepared):
  bank_np = bank_with_duplicates()
  n = bank_np.shape[0]
  eng = _engine(precision, max_batch_pairs=1101 if precision == 'f16_tc' else 64)   # fp32's GEMM grid limit
  bank = torch.from_numpy(bank_np).cuda()
  eng.calibrate(bank[0])
  if prepared:
    eng.bank_prepare(bank)
  rng = np.random.default_rng(7)
  lo, hi = (640, 672) if precision == 'f16_tc' else (650, 658)
  c = rng.integers(0, n + 1, hi - lo)
  c[0], c[1], c[2], c[3] = 0, n, 1, 700                        # empty prefix, the whole bank, one, past the duplicates
  ov = np.zeros((hi - lo, n), np.float32)
  yaw = np.zeros((hi - lo, n), np.int32)
  for r in range(hi - lo):
    if c[r]:
      o, y, _ = eng.heads_1vsN(bank, bank[lo + r], n_cand=int(c[r]))
      ov[r, :c[r]], yaw[r, :c[r]] = o.cpu().numpy(), y.cpu().numpy()
  eng.check()
  assert np.array_equal(ov[3, :40], ov[3, 600:640])             # the duplicated candidates tie
  for k in (1, 5, 32):
    got = [t.cpu().numpy() for t in eng.heads_prefix_topk(bank, lo, hi, c, k)]
    eng.check()
    assert same(got, numpy_topk(ov, yaw, c, k)), (precision, prepared, k)
    assert np.all(got[1][0] == -1) and np.all(got[1][2, 1:] == -1) and got[1][2, 0] == 0
  eng.close()


def test_heads_prefix_topk_over_two_scratch_fills():
  fv = synth.feature_volumes(13, 32)[:, 0]
  n = 2202
  bank_np = np.stack([np.roll(fv[i % 32], (i // 32) * 5, axis=0) for i in range(n)])
  eng = _engine()
  bank = torch.from_numpy(bank_np).cuda()
  eng.calibrate(bank[0])
  eng.bank_prepare(bank)
  rows, k = 2200, 5
  c = np.full(rows, 1101)                                      # 2 422 200 pairs > 2^21: two fills
  eng.profile_enable(True)
  got = [t.cpu().numpy() for t in eng.heads_prefix_topk(bank, 0, rows, c, k)]
  _, launches = eng.profile_read('rows_topk')
  assert launches == 2
  ov = torch.empty((rows, 1101), dtype=torch.float32, device=eng.device)
  yaw = torch.empty((rows, 1101), dtype=torch.int32, device=eng.device)
  for r in range(rows):
    eng.heads_1vsN(bank, bank[r], n_cand=1101, out=(ov[r], yaw[r]))
  eng.check()
  want = numpy_topk(ov.cpu().numpy(), yaw.cpu().numpy(), c, k)
  assert same(got, want)
  # the public reduction on the same scores agrees
  assert same([t.cpu().numpy() for t in eng.rows_topk(ov, yaw, c, k)], want)
  eng.close()


def test_refusals_launch_nothing():
  eng = _engine()
  bank = torch.from_numpy(synth.feature_volumes(5, 8)[:, 0]).cuda()
  before = eng.launch_count()
  bad = [dict(k=0), dict(k=33), dict(c=[-1, 2]), dict(c=[9, 2]), dict(lo=1, hi=0, c=[]), dict(lo=7, hi=9, c=[1, 1])]
  for b in bad:
    with pytest.raises(OvnError, match='INVALID_ARG'):
      eng.heads_prefix_topk(bank, b.get('lo', 0), b.get('hi', 2), b.get('c', [1, 2]), b.get('k', 5))
  ov = torch.zeros((2, 4), device=eng.device)
  yaw = torch.zeros((2, 4), dtype=torch.int32, device=eng.device)
  for n, k in (([5, 1], 1), ([-1, 1], 1), ([1, 1], 0), ([1, 1], 33)):
    with pytest.raises(OvnError, match='INVALID_ARG'):
      eng.rows_topk(ov, yaw, n, k)
  out = eng._topk_out(2, 5)
  nn = np.array([1, 2], np.int32)
  import ctypes as C
  st = lib().ovn_heads_prefix_topk(eng._h, None, 8, 0, 2, nn.ctypes.data_as(C.c_void_p), 5,
                                   *[C.c_void_p(t.data_ptr()) for t in out], None)
  assert st != 0
  st = lib().ovn_rows_topk(eng._h, C.c_void_p(ov.data_ptr()), C.c_void_p(yaw.data_ptr()), 2, 4, None, 5,
                           *[C.c_void_p(t.data_ptr()) for t in out], None)
  assert st != 0
  assert eng.launch_count() == before
  eng.heads_prefix_topk(bank, 0, 2, [1, 2], 5)                 # the handle still works
  eng.check()
  eng.close()


# ---- evaluate_clouds on a two-lap sequence ------------------------------------------------------------------
LAP, STEP = 60, 1.0


def two_lap_sequence():
  """120 scans on a circle of 60 m: the second lap is the first lap's clouds at its poses, 1 cm to the side."""
  r = LAP * STEP / (2 * np.pi)
  poses = []
  for i in range(2 * LAP):
    a = 2 * np.pi * (i % LAP) / LAP
    T = np.eye(4)
    T[:2, :2] = [[np.cos(a + np.pi / 2), -np.sin(a + np.pi / 2)], [np.sin(a + np.pi / 2), np.cos(a + np.pi / 2)]]
    T[0, 3], T[1, 3] = r * np.cos(a), r * np.sin(a)
    if i >= LAP:
      T[0, 3] += 0.01
    poses.append(T)
  clouds = [synth.kitti_like_cloud(500 + (i % LAP), n_points=6000) for i in range(2 * LAP)]
  return clouds, np.array(poses)


@pytest.fixture(scope='module')
def sequence(tmp_path_factory):
  root = str(tmp_path_factory.mktemp('lcd_eval'))
  clouds, poses = two_lap_sequence()
  w = N.glorot_weights(4, MODEL, seed=5)
  imgs = []
  eng = Engine(model=MODEL, precision='fp32', max_batch_scans=4, max_batch_pairs=1)
  x = eng.preprocess(eng.upload_clouds([clouds[i] for i in (3, 10, 40, LAP + 3)])).cpu().numpy()
  eng.close()
  fv = N.leg_forward(x, w, MODEL)
  _, _, _, z0 = N.heads_forward(fv[[0, 1, 2]], fv[[3, 3, 3]], w, MODEL, return_logit=True)
  w = N.spread_dense(w, z0, target_std=1.5)
  wpath = os.path.join(root, 'weights.npz')
  W.save_npz(wpath, w)
  seq = os.path.join(root, '07')
  for sub in ('depth', 'normal'):
    os.makedirs(os.path.join(seq, sub), exist_ok=True)
  eng = Engine(model=MODEL, precision='fp32', max_batch_scans=16, max_batch_pairs=1)
  for s0 in range(0, len(clouds), 16):                        # cue files for the host composition's Infer
    ids = list(range(s0, min(len(clouds), s0 + 16)))
    x = eng.preprocess(eng.upload_clouds([clouds[i] for i in ids])).cpu().numpy()
    for j, i in enumerate(ids):
      np.save(os.path.join(seq, 'depth', '%06d.npy' % i), x[j, :, :, 0])
      np.save(os.path.join(seq, 'normal', '%06d.npy' % i), x[j, :, :, 1:4])
  eng.close()
  cfg = {'pretrained_weightsfilename': wpath, 'use_depth': True, 'use_normals': True,
         'use_class_probabilities': False, 'use_class_probabilities_pca': False, 'use_intensity': False,
         'data_root_folder': root, 'infer_seqs': '07', 'batch_size': 1, 'model': copy.deepcopy(MODEL)}
  return clouds, poses, cfg, root


EVAL = dict(top_k=5, exclude_frames=20, exclude_distance=10.0)


def test_evaluate_clouds_equals_a_host_composition(sequence, tmp_path):
  from overlapnet_b200 import gt
  from overlapnet_b200.infer import Infer
  from overlapnet_b200.sharded_infer import ShardedInfer
  clouds, poses, cfg, _ = sequence
  summary, res = lcd_eval.evaluate_clouds(Infer(copy.deepcopy(cfg)), clouds, poses, out_dir=str(tmp_path), **EVAL)
  assert os.path.exists(tmp_path / 'lcd_results.npz') and os.path.exists(tmp_path / 'lcd_summary.json')
  c = lcd_eval.past_prefix(poses[:, :2, 3], EVAL['exclude_frames'], EVAL['exclude_distance'])
  assert np.array_equal(res['c'], c) and c.max() > 0
  # host composition: demo 3's per-frame calls (calibrated on frame 0 like the evaluation), a NumPy top-k, the
  # per-frame ground truth and the NumPy metrics
  inf = ShardedInfer(copy.deepcopy(cfg))
  n, k = len(clouds), EVAL['top_k']
  ov = np.zeros((n, n), np.float32)
  yaw = np.zeros((n, n), np.int32)
  for i in range(n):
    r = inf.infer_multiple(i, list(range(c[i])))
    if r is not None:
      ov[i, :c[i]], yaw[i, :c[i]] = np.atleast_1d(r[0]), r[1]
  t_ov, t_idx, t_yaw = numpy_topk(ov, yaw, c, k)
  assert same((res['top_overlap'], res['top_index'], res['top_yaw']), (t_ov, t_idx, t_yaw))
  gt_best = np.full(n, -1.0)
  gt_top = np.full((n, k), -1.0)
  for i in np.flatnonzero(c > 0):
    g = gt.overlap_yaw_from_clouds(clouds, poses, int(i))[:, 2]
    gt_best[i] = g[:c[i]].max()
    ok = t_idx[i] >= 0
    gt_top[i, ok] = g[t_idx[i, ok]]
  assert np.array_equal(res['gt_best'], gt_best) and np.array_equal(res['gt_top_overlap'], gt_top)
  assert res['positive'].sum() > 0                              # the second lap revisits the first
  want, curve = lcd_eval.metrics(t_ov, t_idx, gt_top, gt_best)
  for key, v in want.items():
    assert summary[key] == v or (np.isnan(v) and np.isnan(summary[key])), key
  assert np.array_equal(res['curve_precision'], curve['precision'])
  assert res['yaw_error'].size == summary['true_positives_at_f1_max']
  assert np.all((res['yaw_error'] >= 0) & (res['yaw_error'] <= 180))


def _free_port():
  s = socket.socket()
  s.bind(('127.0.0.1', 0))
  p = s.getsockname()[1]
  s.close()
  return p


def _rank_worker(rank, world, port, cfg, out_dir):
  import torch.distributed as dist
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(0)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  try:
    from overlapnet_b200.infer import Infer
    clouds, poses = two_lap_sequence()
    lcd_eval.evaluate_clouds(Infer(copy.deepcopy(cfg)), clouds, poses, out_dir=out_dir, **EVAL)
  except Exception:
    import traceback
    with open(os.path.join(os.path.dirname(out_dir), 'rank%d.err' % rank), 'w') as f:
      f.write(traceback.format_exc())
    raise
  finally:
    dist.destroy_process_group()


def test_two_ranks_write_the_one_rank_results(sequence, tmp_path):
  import torch.multiprocessing as mp
  from overlapnet_b200.infer import Infer
  clouds, poses, cfg, _ = sequence
  cfg = dict(copy.deepcopy(cfg), batch_size=16)                 # encode batches cut across the ranks' shares
  one, two = str(tmp_path / 'one'), str(tmp_path / 'two')
  lcd_eval.evaluate_clouds(Infer(copy.deepcopy(cfg)), clouds, poses, out_dir=one, **EVAL)
  try:
    mp.spawn(_rank_worker, args=(2, _free_port(), cfg, two), nprocs=2, join=True)
  finally:
    for r in range(2):                                          # every rank's own error, not only the first seen
      err = tmp_path / ('rank%d.err' % r)
      if err.exists():
        print(err.read_text())
  with open(os.path.join(one, 'lcd_results.npz'), 'rb') as f1, open(os.path.join(two, 'lcd_results.npz'), 'rb') as f2:
    assert f1.read() == f2.read()
