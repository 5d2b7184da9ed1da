"""All-pairs ground truth (``gt.overlap_yaw_all_pairs`` / ``ovn_gt_pairs_count``) against the per-frame
path ``overlap_yaw_from_clouds``, which it must reproduce bit for bit: the golden fixture, a synthetic
looping sequence with pruned pairs, the pruning bound's edge, tilings and device budgets, error paths,
the demo4 CLI end to end into one training epoch, and two GPUs."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from make_golden_gt import gt_test_clouds, se3  # noqa: E402
from oracle import gt as G  # noqa: E402
from overlapnet_b200 import evaluate, gt, gt_files, synth, training  # noqa: E402
from overlapnet_b200._cabi import OvnError  # noqa: E402
from test_gpu_gt import overlap_tolerance  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def per_frame(clouds, poses, frames):
  return np.concatenate([gt.overlap_yaw_from_clouds(clouds, poses, int(f)) for f in frames])


def loop_sequence(n=40, n_points=4000, radius=90.0, seed=3):
  """Scans on a circle of ``radius`` metres: pairs more than ~130 m apart are pruned (cloud radius 80 m).
  Rotations carry a 1e-6 perturbation, as SLAM poses are not exactly orthonormal."""
  rng = np.random.default_rng(seed)
  clouds = [synth.kitti_like_cloud(seed * 1000 + i, n_points=n_points) for i in range(n)]
  poses = []
  for i in range(n):
    th = 2 * np.pi * i / n
    T = se3(np.rad2deg(th) + 90.0, rng.normal(0, 1), rng.normal(0, 1),
            [radius * np.cos(th), radius * np.sin(th), rng.normal(0, 0.5)])
    T[:3, :3] += rng.normal(0, 1e-6, (3, 3))
    poses.append(T)
  return clouds, np.stack(poses)


@pytest.fixture(scope='module')
def golden():
  clouds, poses = gt_test_clouds(GOLDEN)
  return clouds, poses, np.load(os.path.join(GOLDEN, 'gt_overlap_yaw.npz'))


@pytest.fixture(scope='module')
def loop():
  clouds, poses = loop_sequence()
  return clouds, poses, per_frame(clouds, poses, range(len(clouds)))


def test_golden_every_frame_equals_per_frame_path(golden):
  clouds, poses, gold = golden
  res = gt.overlap_yaw_all_pairs(clouds, poses)
  n = len(clouds)
  assert res.counts.dtype == np.int32 and res.counts.shape == (n, n) and res.yaw_bin.shape == (n, n)
  rows = gt.all_pairs_rows(res)
  assert rows.dtype == np.float64 and np.array_equal(rows, per_frame(clouds, poses, range(n)))
  for f in range(n):
    pts = G.homogeneous_points(clouds[f])
    own = G.range_image_f64(pts)
    uncertain = G.explain_range_image(pts, own, G.geometry(f32=False))[2]
    assert abs(int(res.valid_num[f]) - np.count_nonzero(own > 0)) <= np.count_nonzero(uncertain)
  for frame in (0, 3):
    want = gold['mapping_frame%d' % frame]
    got = rows[frame * n:(frame + 1) * n]
    assert np.array_equal(got[:, [0, 1, 3]], want[:, [0, 1, 3]])
    assert np.all(np.abs(got[:, 2] - want[:, 2]) <= overlap_tolerance(clouds, poses, frame))


def test_loop_sequence_bit_identical_and_pruned(loop):
  clouds, poses, want = loop
  res = gt.overlap_yaw_all_pairs(clouds, poses)
  n = len(clouds)
  print('loop sequence: %d of %d pairs pruned, %d with count > 0' % (res.n_pruned, n * n,
                                                                    np.count_nonzero(res.counts)))
  assert np.array_equal(gt.all_pairs_rows(res), want)
  assert 0 < res.n_pruned < n * n
  assert np.count_nonzero(res.counts) > n                     # not only the self pairs overlap


@pytest.mark.parametrize('budget,tiles', [(4000 * 16 * 7 + 5, (0, 0)), (None, (1, 1)), (None, (3, 5)),
                                          (None, (32, 64)), (4000 * 16 * 13, (7, 2))])
def test_result_independent_of_blocks_and_tiles(loop, budget, tiles):
  clouds, poses, want = loop
  frames = [0, 1, 2, 17, 30, 39]
  res = gt.overlap_yaw_all_pairs(clouds, poses, frames=frames, device_budget_bytes=budget,
                                 tile_cur=tiles[0], tile_ref=tiles[1])
  rows = gt.all_pairs_rows(res)
  n = len(clouds)
  assert np.array_equal(rows, np.concatenate([want[f * n:(f + 1) * n] for f in frames]))
  full = gt.overlap_yaw_all_pairs(clouds, poses, frames=frames)
  assert res.n_pruned == full.n_pruned and np.array_equal(res.counts, full.counts)


def test_lazy_clouds_and_unsorted_frames(loop):
  clouds, poses, want = loop
  lazy = [(lambda c=c: c) for c in clouds]
  n = len(clouds)
  frames = [5, 4, 20, 21, 3]
  res = gt.overlap_yaw_all_pairs(lazy, poses, frames=frames, device_budget_bytes=4000 * 16 * 9)
  assert np.array_equal(gt.all_pairs_rows(res), np.concatenate([want[f * n:(f + 1) * n] for f in frames]))


def test_pair_just_inside_the_bound_is_counted():
  # scan 1 (radius 1 m) sits 50.99 m away: bound 50.99 - 1 - 1e-3 < 50, its point lands at 49.99 m in the
  # same pixel as frame 0's point at 49.7 m; scan 2 sits 51.01 m away: bound >= 50, pruned, count 0
  cur = np.array([[49.7, 0, 0, 0.5]], np.float32)
  ref = np.array([[-1.0, 0, 0, 0.5]], np.float32)
  poses = np.stack([np.eye(4), np.eye(4), np.eye(4)])
  poses[1, 0, 3], poses[2, 0, 3] = 50.99, 51.01
  clouds = [cur, ref, ref]
  res = gt.overlap_yaw_all_pairs(clouds, poses, frames=[0])
  assert res.counts.tolist() == [[1, 1, 0]] and res.valid_num.tolist() == [1] and res.n_pruned == 1
  assert np.array_equal(gt.all_pairs_rows(res), gt.overlap_yaw_from_clouds(clouds, poses, 0))
  assert gt.depth_lower_bound(np.linalg.inv(poses[0]).dot(poses[1]), 1.0) < 50.0
  assert gt.depth_lower_bound(np.linalg.inv(poses[0]).dot(poses[2]), 1.0) >= 50.0


def test_error_paths_leave_the_handle_usable(golden):
  clouds, poses, _ = golden
  with pytest.raises(IndexError):
    gt.overlap_yaw_all_pairs(clouds, poses, frames=[0, 5])
  with pytest.raises(IndexError):
    gt.overlap_yaw_all_pairs(clouds, poses, frames=[-1])
  with pytest.raises(ValueError):
    gt.overlap_yaw_all_pairs(clouds, poses[:4])
  with pytest.raises(ValueError):
    gt.overlap_yaw_all_pairs(clouds[:2] + [np.zeros((0, 4), np.float32)], poses[:3])
  with pytest.raises(ValueError):
    gt.overlap_yaw_all_pairs(clouds, poses, device_budget_bytes=1000)          # no cloud fits
  eng = gt._engine(3.0, -25.0, 64, 900, 50)
  batch = eng.upload_clouds(clouds[:2])
  d_pose = torch.from_numpy(poses[:2].reshape(2, 16).copy()).to(eng.device)
  cur = eng.gt_range(batch)
  with pytest.raises(OvnError, match='OVN_ERR_CAPACITY'):
    eng.gt_pairs_count(batch, d_pose, eng.gt_scan_radius(batch), cur, d_pose, tile_cur=33)
  res = gt.overlap_yaw_all_pairs(clouds, poses, frames=[3])
  assert np.array_equal(gt.all_pairs_rows(res), gt.overlap_yaw_from_clouds(clouds, poses, 3))


def _kitti_folder(root, seq, n=10, n_points=20000):
  """A KITTI-layout sequence: velodyne/*.bin, camera poses.txt (3 m steps along the camera's z) and calib.txt."""
  d = os.path.join(root, seq)
  os.makedirs(os.path.join(d, 'velodyne'))
  for i in range(n):
    synth.kitti_like_cloud(500 + i, n_points=n_points).tofile(os.path.join(d, 'velodyne', '%06d.bin' % i))
  Tr = np.array([[0, -1, 0, 0], [0, 0, -1, -0.08], [1, 0, 0, -0.27]], np.float64)
  with open(os.path.join(d, 'calib.txt'), 'w') as f:
    f.write('P0: ' + ' '.join(['0'] * 12) + '\nTr: ' + ' '.join('%.6e' % v for v in Tr.ravel()) + '\n')
  with open(os.path.join(d, 'poses.txt'), 'w') as f:
    for i in range(n):
      T = se3(0.0, 2.0 * i, 0.0, [0.1 * i, 0.0, 3.0 * i])[:3]
      f.write(' '.join('%.9e' % v for v in T.ravel()) + '\n')
  return d


@pytest.mark.parametrize('mode', [['--all-frames'], ['--frames', '0:10']])
def test_cli_end_to_end_into_training(tmp_path, capsys, mode):
  from oracle import network as N
  from overlapnet_b200 import gen_depth_data, gen_normal_data
  root, seq = str(tmp_path / 'data'), 'seqA'
  d = _kitti_folder(root, seq)
  cfg = tmp_path / 'demo.yml'
  cfg.write_text('Demo4:\n  poses_file: "%s"\n  calib_file: "%s"\n  scan_folder: "%s"\n  dst_folder: "%s"\n'
                 % (os.path.join(d, 'poses.txt'), os.path.join(d, 'calib.txt'), os.path.join(d, 'velodyne'), d))
  np.random.seed(0)
  dst = gt_files.main([str(cfg), '--seq', seq] + mode)
  out = capsys.readouterr().out
  assert 'finished generating training data and validation data' in out and 'size of normalized data' in out
  assert sorted(os.listdir(dst)) == ['ground_truth_overlap_yaw.npz', 'train_set.npz', 'validation_set.npz']
  full = np.load(os.path.join(dst, 'ground_truth_overlap_yaw.npz'), allow_pickle=True)
  rows = full['overlaps']
  assert rows.shape == (100, 4) and np.array_equal(rows[:, 0], np.repeat(np.arange(10.0), 10))
  assert np.array_equal(rows[:, 1], np.tile(np.arange(10.0), 10))
  poses = gt_files.kitti_poses_in_lidar(gt.load_poses(os.path.join(d, 'poses.txt')),
                                        gt.load_calib(os.path.join(d, 'calib.txt')))
  clouds = [gt._read_scan(os.path.join(d, 'velodyne', '%06d.bin' % i)) for i in range(10)]
  assert np.array_equal(rows[20:30], gt.overlap_yaw_from_clouds(clouds, poses, 2))
  for name in ('train_set', 'validation_set', 'ground_truth_overlap_yaw'):
    f1, f2, d1, d2, ov, orient = evaluate.load_overlap_npz([os.path.join(dst, name + '.npz')])
    assert len(f1) > 0 and set(d1) == {seq} and np.all((ov >= 0) & (ov <= 1))
  gen_depth_data(os.path.join(d, 'velodyne'), d)
  gen_normal_data(os.path.join(d, 'velodyne'), d)
  model = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
  pretrained = str(tmp_path / 'pretrained.weight')
  training.save_weights(pretrained, N.glorot_weights(4, model, seed=0))
  tcfg = {'experiments_path': str(tmp_path / 'exp'), 'testname': 'gt', 'pretrained_weightsfilename': pretrained,
          'use_depth': True, 'use_normals': True, 'data_root_folder': root, 'training_seqs': seq,
          'batch_size': 4, 'no_batches_in_epoch': 100, 'no_epochs': 1, 'no_test_pairs': 100,
          'learning_rate': 1e-4, 'lr_alpha': 0.99, 'min_overlap_for_angle': 0.7,
          'model': {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegsFixed',
                    'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                    'inputShape': [64, 900], 'leg_output_width': 360, **model}}
  hist = training.train(tcfg)
  assert len(hist['epoch_loss']) == 1 and np.isfinite(hist['epoch_loss'][0])
  assert os.path.isfile(hist['weights_filename'])


def _two_gpu_worker(rank, port, clouds, poses, out_path):
  import torch.distributed as dist
  torch.cuda.set_device(rank)
  dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=2)
  try:
    res = gt.overlap_yaw_all_pairs(clouds, poses)
    if rank == 0:
      np.savez(out_path, frames=res.frames, counts=res.counts, valid_num=res.valid_num, yaw_bin=res.yaw_bin,
               n_pruned=res.n_pruned)
    else:
      assert res is None
  finally:
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_gpus_bit_identical_to_one(loop, tmp_path):
  import socket
  import torch.multiprocessing as mp
  clouds, poses, _ = loop
  one = gt.overlap_yaw_all_pairs(clouds, poses)
  with socket.socket() as s:
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
  out = str(tmp_path / 'two.npz')
  mp.spawn(_two_gpu_worker, args=(port, clouds, poses, out), nprocs=2, join=True)
  two = np.load(out)
  for k in ('frames', 'counts', 'valid_num', 'yaw_bin'):
    assert np.array_equal(two[k], getattr(one, k)), k
  assert int(two['n_pruned']) == one.n_pruned
