"""demo4's ground-truth post-processing without a GPU: normalize_data / split_train_val against the
reference's functions (live, when the reference is mounted) and against known answers, the pruning
bound of the all-pairs kernel, and the CLI's arguments, pose conversion and file layout."""
import importlib
import os
import sys

import numpy as np
import pytest

from overlapnet_b200 import evaluate, gt_files
from overlapnet_b200.gt import depth_lower_bound

REF_UTILS = '/root/reference/src/utils'


def mapping(seed, n=600):
  """Rows [frame, ref, overlap, yaw] with overlaps over every bin, including exact edges and 1.0."""
  rng = np.random.default_rng(seed)
  m = np.zeros((n, 4))
  m[:, 0] = 3
  m[:, 1] = np.arange(n)
  m[:, 2] = rng.uniform(0, 1, n)
  m[:8, 2] = [0.0, 0.1, 0.2, 0.3, 0.4, 0.5, 0.9, 1.0]
  m[:, 3] = rng.integers(0, 361, n)
  return m


def ref_module(name):
  if REF_UTILS not in sys.path:
    sys.path.insert(0, REF_UTILS)
  return importlib.import_module(name)


@pytest.mark.skipif(not os.path.isdir(REF_UTILS), reason='reference not mounted')
@pytest.mark.parametrize('seed', [0, 1, 2])
def test_normalize_data_equals_reference(seed, capsys):
  ref = ref_module('normalize_data').normalize_data
  m = mapping(seed)
  np.random.seed(seed)
  want = ref(m)
  want_next = np.random.random()
  want_out = capsys.readouterr().out
  np.random.seed(seed)
  got = gt_files.normalize_data(m)
  assert capsys.readouterr().out == want_out
  assert got.dtype == want.dtype and np.array_equal(got, want)
  assert np.random.random() == want_next            # the same draws were consumed


@pytest.mark.skipif(not os.path.isdir(REF_UTILS), reason='reference not mounted')
@pytest.mark.parametrize('n', [10, 57, 600])
def test_split_train_val_equals_reference(n, capsys):
  pytest.importorskip('sklearn')
  ref = ref_module('split_train_val').split_train_val
  m = mapping(n, n)
  np.random.seed(n)
  want = ref(m)
  want_out = capsys.readouterr().out
  np.random.seed(n)
  got = gt_files.split_train_val(m)
  assert capsys.readouterr().out == want_out
  for g, w in zip(got, want):
    assert np.array_equal(g, w)


def test_normalize_data_known_answer(capsys):
  m = mapping(5)
  ov = m[:, 2]
  edges = [0.0, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9]
  bins = [m[(ov < hi) & (ov >= lo)] for lo, hi in zip(edges[:-1], edges[1:])] + [m[(ov >= 0.9) & (ov <= 1)]]
  low = bins[:5]
  np.random.seed(7)
  picks = [np.random.choice(len(b), len(low[4])) for b in low]
  want = np.concatenate([b[p] for b, p in zip(low, picks)] + bins[5:])
  np.random.seed(7)
  got = gt_files.normalize_data(m)
  assert np.array_equal(got, want)
  assert capsys.readouterr().out == 'size of normalized data:  %d\n' % len(want)
  # sampling with replacement: the four lower bins have exactly the size of [0.4, 0.5)
  assert np.count_nonzero(got[:, 2] < 0.5) == 5 * len(low[4])


def test_normalize_data_keeps_reference_quirks():
  m = np.array([[0, 0, 0.45, 0], [0, 1, 0.95, 0], [0, 2, 1.5, 0]])
  with pytest.raises(ValueError):                   # bins below 0.4 are empty, [0.4, 0.5) is not
    gt_files.normalize_data(m)
  m = np.array([[0, 0, 0.05, 0], [0, 1, 0.95, 0], [0, 2, 1.0, 0], [0, 3, 1.5, 0]])
  got = gt_files.normalize_data(m)                  # [0.4, 0.5) empty: every lower bin sampled to 0 rows
  assert got[:, 1].tolist() == [1, 2]               # overlap > 1 dropped


def test_split_train_val_known_answer():
  m = mapping(3, 95)
  np.random.seed(11)
  perm = np.random.permutation(95)
  np.random.seed(11)
  train, test = gt_files.split_train_val(m)
  assert np.array_equal(test, m[perm[:9]]) and np.array_equal(train, m[perm[9:]])
  with pytest.raises(ValueError):
    gt_files.split_train_val(m[:9])                 # a tenth of 9 rows is 0


def test_pruning_bound_never_exceeds_true_depth():
  rng = np.random.default_rng(0)
  from oracle.gt import homogeneous_points
  for trial in range(300):
    q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    if trial % 2:
      q = q + rng.normal(0, 1e-3, (3, 3))           # SLAM poses are not exactly orthonormal
    A = np.eye(4)
    A[:3, :3] = q
    A[:3, 3] = rng.normal(0, 80, 3)
    B = np.eye(4)
    B[:3, :3] = np.linalg.qr(rng.standard_normal((3, 3)))[0]
    B[:3, 3] = rng.normal(0, 80, 3)
    B[3, :3] = rng.normal(0, 1e-12, 3)              # an inverted pose's last row is not exactly [0 0 0 1]
    cloud = (rng.standard_normal((500, 4)) * rng.uniform(1, 60)).astype(np.float32)
    p = homogeneous_points(cloud)
    radius = float(np.sqrt(np.max(np.sum(p[:, :3] ** 2, axis=1))))
    depth = np.linalg.norm(A.dot(B.dot(p.T)).T[:, :3], axis=1)
    assert depth_lower_bound(A.dot(B), radius) <= depth.min()


def test_pruning_bound_is_tight_for_rigid_poses():
  T = np.eye(4)
  T[:3, 3] = [51.0, 0, 0]
  assert abs(depth_lower_bound(T, 1.0) - 49.999) < 1e-9


def test_cli_arguments():
  a = gt_files.parse_args([])
  assert (a.config, a.seq, a.all_frames, a.frames) == ('config/demo.yml', '07', False, None)
  a = gt_files.parse_args(['my.yml', '--seq', '00', '--all-frames'])
  assert (a.config, a.seq, a.all_frames) == ('my.yml', '00', True)
  with pytest.raises(SystemExit):
    gt_files.parse_args(['--all-frames', '--frames', '1'])
  assert gt_files.parse_frames('3,1,1, 5', 10) == [1, 3, 5]
  assert gt_files.parse_frames('2:5,8:', 10) == [2, 3, 4, 8, 9]
  with pytest.raises(ValueError):
    gt_files.parse_frames('10', 10)


def test_kitti_pose_conversion():
  rng = np.random.default_rng(2)
  poses = np.tile(np.eye(4), (3, 1, 1))
  poses[:, :3, :] = rng.normal(size=(3, 3, 4))
  Tr = np.eye(4)
  Tr[:3, :] = rng.normal(size=(3, 4))
  got = gt_files.kitti_poses_in_lidar(poses, Tr)
  for i in range(3):
    want = np.linalg.inv(Tr).dot(np.linalg.inv(poses[0])).dot(poses[i]).dot(Tr)
    assert np.array_equal(got[i], want)


def test_saved_files_load_like_the_reference_format(tmp_path, capsys):
  m = mapping(4, 50)
  dst = gt_files.save_ground_truth(str(tmp_path), '05', m, m[:40], m[40:])
  assert 'creating new depth folder' in capsys.readouterr().out
  assert sorted(os.listdir(dst)) == ['ground_truth_overlap_yaw.npz', 'train_set.npz', 'validation_set.npz']
  z = np.load(os.path.join(dst, 'train_set.npz'), allow_pickle=True)
  assert sorted(z.files) == ['overlaps', 'seq'] and z['seq'].dtype == object and z['seq'].shape == (40, 2)
  f1, f2, d1, d2, ov, orient = evaluate.load_overlap_npz([os.path.join(dst, 'validation_set.npz')], shuffle=False)
  assert f1 == ['000003'] * 10 and f2[0] == '%06d' % 40 and set(d1) == set(d2) == {'05'}
  assert np.array_equal(ov, m[40:, 2]) and np.array_equal(orient, m[40:, 3])
  gt_files.save_ground_truth(str(tmp_path), '05', m, m[:40], m[40:])      # an existing folder is reused
  assert 'generating depth data in' in capsys.readouterr().out
