"""Point-to-plane ICP on the GPU (ovn_icp_pairs): recovery of known transforms, bit-identical pairs in any batch and
handle, the refusals and the device error, and loop-closure evaluation with registration.  Every iteration's stages
are checked against the float64 stage model in tests/test_gpu_icp_stages.py."""
import copy
import ctypes as C
import math
import os
import socket

import numpy as np
import pytest
import torch

from icp_cases import (GATE_ROTATION_DEG, GATE_TRANSLATION, KITTI_TRANSFORMS, STREET_RIGHT, kitti_pair, rz,
                       street_pair)
from oracle import icp
from oracle import network as N
from overlapnet_b200 import gt, lcd_eval, registration, synth, weights as W
from overlapnet_b200._cabi import ICP_STATUS, IcpParams, OvnError, lib
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

GEOMETRIES = {'64x900': dict(proj_H=64, proj_W=900), '32x2048': dict(proj_H=32, proj_W=2048, fov_up=15.0, fov_down=-15.0),
              '128x1024': dict(proj_H=128, proj_W=1024, fov_up=2.0, fov_down=-24.9)}


def _engine(geometry='64x900'):
  return Engine(precision='fp32', max_batch_scans=16, max_batch_pairs=1, **GEOMETRIES[geometry])


def _geometry(eng):
  c = eng.cfg
  return icp.geometry(c.proj_H, c.proj_W, c.fov_up_deg, c.fov_down_deg, c.max_range)


def yaw_seed_of(T, Wf=360):
  return registration.seed_pose(gt.yaw_bin(np.eye(4), T, Wf), Wf)


def cases(geometry):
  """[(LEFT, RIGHT, T*)] of a geometry: every known transform and street pair at 64x900, two street pairs elsewhere."""
  if geometry == '64x900':
    return [kitti_pair(y, t) for y, t in KITTI_TRANSFORMS] + [street_pair(k) for k in range(len(STREET_RIGHT))]
  return [street_pair(0), street_pair(3)]


def stack_images(eng, clouds):
  return registration.images(eng, clouds, list(range(len(clouds))))


def run(eng, vertex, normal, src, dst, init, want_stage=False, **params):
  out = eng.icp(vertex, normal, src, dst, init, params, want_stage)
  eng.check()
  return {k: v.cpu().numpy() for k, v in out.items()}


# ---- recovery -----------------------------------------------------------------------------------------------------
def test_recovers_the_known_transforms():
  eng = _engine()
  cs = cases('64x900')
  vertex, normal = stack_images(eng, [c for L, R, _ in cs for c in (L, R)])
  n = len(cs)
  src, dst = np.arange(n) * 2 + 1, np.arange(n) * 2
  truth = np.stack([T for _, _, T in cs])
  res = run(eng, vertex, normal, np.r_[src, src], np.r_[dst, dst],
            np.concatenate([np.stack([yaw_seed_of(T) for T in truth]), np.broadcast_to(np.eye(4), (n, 4, 4))]))
  te, re = registration.pose_error(res['pose'], np.concatenate([truth, truth]))
  re = np.degrees(re)
  print('yaw seed: <= %.4f m, <= %.4f deg; identity: %s deg' % (te[:n].max(), re[:n].max(), np.round(re[n:], 3)))
  assert np.all(te[:n] < GATE_TRANSLATION) and np.all(re[:n] < GATE_ROTATION_DEG)
  half_turn = [i for i, (y, _) in enumerate(KITTI_TRANSFORMS) if abs(y) > 170][0]
  assert re[n + half_turn] > 10.0                          # from the identity the half turn is not found
  assert np.all(res['valid'] > 0) and np.all(res['inliers'] <= res['valid'])
  eng.close()


# ---- determinism ----------------------------------------------------------------------------------------------------
def bits(x):
  return np.ascontiguousarray(x).view(np.uint8)


def _same(a, b):
  return all(np.array_equal(bits(a[k]), bits(b[k])) for k in a)


def test_a_pair_has_the_same_bits_in_any_batch_and_handle():
  cs = [street_pair(k) for k in range(len(STREET_RIGHT))]
  clouds = [c for L, R, _ in cs for c in (L, R)]
  init = np.stack([yaw_seed_of(T) for _, _, T in cs])
  eng = _engine()
  vertex, normal = stack_images(eng, clouds)
  pick = lambda r, i: {k: v[i:i + 1] for k, v in r.items()}
  alone = run(eng, vertex, normal, [1], [0], init[:1], want_stage=True)
  rng = np.random.default_rng(0)
  other = rng.integers(0, len(cs), 298)
  idx = np.r_[0, other, 0]
  batch = run(eng, vertex, normal, idx * 2 + 1, idx * 2, init[idx], want_stage=True)
  assert _same(alone, pick(batch, 0)) and _same(alone, pick(batch, 299))
  for j in range(1, 299):                                   # every repeat of every pair agrees with its first
    first = int(np.flatnonzero(idx == idx[j])[0])
    assert _same(pick(batch, first), pick(batch, j))
  assert _same(alone, run(eng, vertex, normal, [1], [0], init[:1], want_stage=True))
  eng2 = _engine()
  v2, n2 = stack_images(eng2, clouds[:2])
  assert _same(alone, run(eng2, v2, n2, [1], [0], init[:1], want_stage=True))
  eng.close()
  eng2.close()


# ---- refusals and the device error ------------------------------------------------------------------------------------
def test_refusals_launch_nothing_and_a_bad_index_poisons_only_its_pair():
  eng = _engine()
  L, R, T = street_pair(0)
  vertex, normal = stack_images(eng, [L, R])
  init = yaw_seed_of(T)[None]
  before = eng.launch_count()
  bad = [dict(iterations=0), dict(iterations=201), dict(d_start=0.2, d_end=0.3), dict(d_end=0.0),
         dict(cos_normal=1.5), dict(cos_normal=-0.1), dict(gamma=0.0), dict(gamma=1.5), dict(d_start=float('nan')),
         dict(eps_rot=float('inf')), dict(min_inliers=-1), dict(eps_trans=-1.0)]
  for b in bad:
    with pytest.raises(OvnError, match='INVALID_ARG'):
      eng.icp(vertex, normal, [1], [0], init, b)
  for value in (float('nan'), float('inf')):
    x = init.copy()
    x[0, 1, 3] = value
    with pytest.raises(OvnError, match='INVALID_ARG'):
      eng.icp(vertex, normal, [1], [0], x)
  prm = IcpParams()
  lib().ovn_icp_default_params(C.byref(prm))
  p = lambda t: C.c_void_p(t.data_ptr())
  src = torch.ones(1, dtype=torch.int32, device=eng.device)
  dst = torch.zeros(1, dtype=torch.int32, device=eng.device)
  dinit = torch.as_tensor(init, device=eng.device).contiguous()
  out = torch.empty(19, dtype=torch.float64, device=eng.device)
  args = [p(vertex), p(normal), 2, p(src), p(dst), p(dinit), 1, C.byref(prm), p(out), None, None, None]
  for i in (0, 1, 3, 4, 5, 8):                              # each required pointer NULL in turn
    a = list(args)
    a[i] = None
    assert lib().ovn_icp_pairs(eng._h, *a) != 0
  for i, v in ((2, 0), (6, -1)):                            # n_scans < 1, np < 0
    a = list(args)
    a[i] = v
    assert lib().ovn_icp_pairs(eng._h, *a) != 0
  a = list(args)
  a[7] = None
  assert lib().ovn_icp_pairs(eng._h, *a) != 0
  a = list(args)
  a[6] = 0
  assert lib().ovn_icp_pairs(eng._h, *a) == 0                # np = 0: a no-op
  assert eng.launch_count() == before
  # an index outside [0, n_scans): the flag, a poisoned pair, the others untouched, the handle usable
  good = run(eng, vertex, normal, [1], [0], init, want_stage=True)
  res = eng.icp(vertex, normal, [1, 2, 1, -1], [0, 0, 0, 0], np.repeat(init, 4, 0), want_stage=True)
  with pytest.raises(OvnError, match='outside'):
    eng.check()
  res = {k: v.cpu().numpy() for k, v in res.items()}
  for i in (1, 3):
    assert res['status'][i] == ICP_STATUS['bad_index'] and np.all(np.isnan(res['pose'][i]))
    assert np.all(res['assoc'][i] == -1) and np.all(np.isnan(res['system'][i]))
  for i in (0, 2):
    assert _same(good, {k: v[i:i + 1] for k, v in res.items()})
  assert _same(good, run(eng, vertex, normal, [1], [0], init, want_stage=True))
  eng.close()


# ---- loop-closure evaluation with registration ----------------------------------------------------------------------
MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
         'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
         'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
         'additional_unsymmetric_layer3a': True}
LAP_STEP = 5.0              # metres between scans around the 40 m block
EVAL = dict(top_k=3, exclude_frames=10, exclude_distance=20.0)


def street_loop_poses():
  """Two laps around the city block [0, 40]^2 of the street scene along its roads, 5 m per scan; the second lap runs
  1.5 m to the side."""
  poses = []
  for lap, off in ((0, 0.0), (1, 1.5)):
    for k in range(int(160 / LAP_STEP)):
      s = k * LAP_STEP
      side, u = int(s // 40), s % 40
      x, y, yaw = [(u, off, 0.0), (40 - off, u, 90.0), (40 - u, 40 - off, 180.0), (off, 40 - u, 270.0)][side]
      poses.append(rz(math.radians(yaw), (x, y, 1.73)))
  return np.array(poses)


def street_loop_clouds(poses):
  return [synth.street_scene_cloud(T, seed=11) for T in poses]


@pytest.fixture(scope='module')
def loop(tmp_path_factory):
  root = str(tmp_path_factory.mktemp('lcd_register'))
  poses = street_loop_poses()
  clouds = street_loop_clouds(poses)
  w = N.glorot_weights(4, MODEL, seed=5)
  wpath = os.path.join(root, 'weights.npz')
  W.save_npz(wpath, w)
  cfg = {'pretrained_weightsfilename': wpath, 'use_depth': True, 'use_normals': True,
         'use_class_probabilities': False, 'use_class_probabilities_pca': False, 'use_intensity': False,
         'data_root_folder': root, 'infer_seqs': '07', 'batch_size': 4, 'model': copy.deepcopy(MODEL)}
  return clouds, poses, cfg


def test_evaluate_clouds_registers_the_top_records(loop, tmp_path):
  from overlapnet_b200.infer import Infer
  from overlapnet_b200.evaluate import yaw_to_argmax
  clouds, poses, cfg = loop
  s0, plain = lcd_eval.evaluate_clouds(Infer(copy.deepcopy(cfg)), clouds, poses, out_dir=str(tmp_path / 'plain'),
                                       **EVAL)
  infer = Infer(copy.deepcopy(cfg))
  s1, res = lcd_eval.evaluate_clouds(infer, clouds, poses, out_dir=str(tmp_path / 'reg'), register=True, **EVAL)
  assert not any(k.startswith('registration') for k in plain) and 'registration' not in s0
  for key, v in plain.items():
    assert np.array_equal(bits(v), bits(res[key])), key
  assert set(s1) == set(s0) | {'registration'}
  for k in s0:
    assert s0[k] == s1[k] or (isinstance(s0[k], float) and math.isnan(s0[k]) and math.isnan(s1[k])), k
  # the host composition: registration.register on the same records, in pairs of another chunking
  rows = np.flatnonzero(res['top_index'][:, 0] >= 0)
  assert rows.size > 0
  left = res['top_index'][rows, 0]
  eng = infer._engine
  seeds = registration.seed_pose(yaw_to_argmax(res['top_yaw'][rows, 0]), eng.Wf)
  want = registration.register(eng, clouds, np.r_[left, left], np.r_[rows, rows],
                               np.concatenate([seeds, np.broadcast_to(np.eye(4), seeds.shape)]), pairs_per_call=7)
  m = rows.size
  got = res['registration_pose'][rows]
  assert np.array_equal(bits(got[:, 0]), bits(want['pose'][:m]))
  assert np.array_equal(bits(got[:, 1]), bits(want['pose'][m:]))
  assert np.array_equal(res['registration_status'][rows], np.stack([want['status'][:m], want['status'][m:]], 1))
  gt_pose = np.linalg.solve(poses[left], poses[rows])
  assert np.array_equal(res['registration_gt_pose'][rows], gt_pose)
  te, re = registration.pose_error(want['pose'][:m], gt_pose)
  np.testing.assert_array_equal(res['registration_error'][rows, 0], np.stack([te, np.degrees(re)], -1))
  r = s1['registration']
  assert r['true_positives'] == s1['true_positives_at_f1_max']
  print('registration summary:', r)


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
    poses = street_loop_poses()
    lcd_eval.evaluate_clouds(Infer(copy.deepcopy(cfg)), street_loop_clouds(poses), poses, out_dir=out_dir,
                             register=True, **EVAL)
  except Exception:
    import traceback
    with open(os.path.join(os.path.dirname(out_dir), 'rank%d.err' % rank), 'w') as f:
      f.write(traceback.format_exc())
    raise
  finally:
    dist.destroy_process_group()


def test_two_ranks_write_the_one_rank_results(loop, tmp_path):
  import torch.multiprocessing as mp
  from overlapnet_b200.infer import Infer
  clouds, poses, cfg = loop
  one, two = str(tmp_path / 'one'), str(tmp_path / 'two')
  lcd_eval.evaluate_clouds(Infer(copy.deepcopy(cfg)), clouds, poses, out_dir=one, register=True, **EVAL)
  try:
    mp.spawn(_rank_worker, args=(2, _free_port(), cfg, two), nprocs=2, join=True)
  finally:
    for r in range(2):
      err = tmp_path / ('rank%d.err' % r)
      if err.exists():
        print(err.read_text())
  with open(os.path.join(one, 'lcd_results.npz'), 'rb') as f1, open(os.path.join(two, 'lcd_results.npz'), 'rb') as f2:
    assert f1.read() == f2.read()
