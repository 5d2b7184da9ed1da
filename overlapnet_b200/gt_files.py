"""The ground-truth files of the reference's ``demo/demo4_gen_gt_files.py`` (:79-109), which
``training.py`` reads: ``<dst>/ground_truth/{train_set,validation_set,ground_truth_overlap_yaw}.npz``.

  python -m overlapnet_b200.gt_files [config/demo.yml] [--seq 07] [--all-frames | --frames 0,10,20]

The configuration is demo.yml's ``Demo4`` section (poses_file, calib_file, scan_folder, dst_folder).
By default the ground truth is that of frame 0 against every scan, as in the demo; ``--all-frames`` or
``--frames`` use every pair of those frames (``gt.overlap_yaw_all_pairs``), rows concatenated
frame-major.  ``normalize_data`` and ``split_train_val`` make the same global ``np.random`` calls as the
reference's (src/utils/normalize_data.py, src/utils/split_train_val.py), so the same ``np.random.seed``
gives the same files.  No plot is drawn."""
import argparse
import os
import sys

import numpy as np

# lower edges of the ten overlap bins of normalize_data: [0, 0.1), [0.1, 0.2), ..., [0.9, 1]
_BIN_EDGES = (0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9)


def normalize_data(ground_truth_mapping):
  """Balance the overlap distribution: the five bins below 0.5 are each resampled, with replacement,
  to the size of the [0.4, 0.5) bin; the bins from 0.5 to 1 are kept whole.  Rows with an overlap
  above 1 are dropped.  Like the reference, ``np.random.choice`` raises ValueError when a bin below 0.4
  is empty while [0.4, 0.5) is not."""
  gt_map = ground_truth_mapping
  ov = gt_map[:, 2]
  bins = [gt_map[ov < _BIN_EDGES[0]]]
  for lo, hi in zip(_BIN_EDGES[:-1], _BIN_EDGES[1:]):
    bins.append(gt_map[(ov < hi) & (ov >= lo)])
  bins.append(gt_map[(ov <= 1) & (ov >= _BIN_EDGES[-1])])
  n_target = len(bins[4])
  for k in range(5):                                  # bins 0-9 ... 40-49, in this order
    bins[k] = bins[k][np.random.choice(len(bins[k]), n_target)]
  dist_norm_data = np.concatenate(bins)
  print("size of normalized data: ", len(dist_norm_data))
  return dist_norm_data


def split_train_val(ground_truth_mapping):
  """Split off a tenth (rounded down) of the rows for validation, as sklearn's
  ``train_test_split(x, test_size=int(len(x) / 10))`` does with the global NumPy generator: one
  ``np.random.permutation``, test = its first rows, train = the rest.  Returns (train_set, test_set)."""
  n = len(ground_truth_mapping)
  test_size = int(n / 10)
  if test_size <= 0 or test_size >= n:
    raise ValueError('test_size=%d should be either positive and smaller than the number of samples %d'
                     % (test_size, n))
  perm = np.random.permutation(n)
  train_set, test_set = ground_truth_mapping[perm[test_size:]], ground_truth_mapping[perm[:test_size]]
  print('finished generating training data and validation data')
  return train_set, test_set


def kitti_poses_in_lidar(poses, T_cam_velo):
  """demo4_gen_gt_files.py:67-76: camera poses -> LiDAR poses relative to the first scan,
  T_velo_cam . pose0^-1 . pose . T_cam_velo."""
  T_cam_velo = np.asarray(T_cam_velo).reshape((4, 4))
  T_velo_cam = np.linalg.inv(T_cam_velo)
  pose0_inv = np.linalg.inv(poses[0])
  return np.array([T_velo_cam.dot(pose0_inv).dot(pose).dot(T_cam_velo) for pose in poses])


def parse_frames(text, n):
  """'0,5,7' or '10:20' (a half-open range) -> sorted unique frame indices in [0, n)."""
  frames = set()
  for part in text.split(','):
    part = part.strip()
    if not part:
      continue
    if ':' in part:
      a, b = part.split(':')
      frames.update(range(int(a) if a else 0, int(b) if b else n))
    else:
      frames.add(int(part))
  frames = sorted(frames)
  if not frames or frames[0] < 0 or frames[-1] >= n:
    raise ValueError('--frames must name frames in [0, %d), got %r' % (n, text))
  return frames


def save_ground_truth(dst_folder, seq_idx, ground_truth_mapping, train_data, validation_data):
  """demo4_gen_gt_files.py:85-107: the three npz files, each with ``overlaps`` and an object array
  ``seq`` of the sequence label, in ``<dst_folder>/ground_truth``.  Returns that folder."""
  dst = os.path.join(dst_folder, 'ground_truth')
  try:
    os.stat(dst)
    print('generating depth data in: ', dst)
  except OSError:
    print('creating new depth folder: ', dst)
    os.mkdir(dst)
  for name, data in (('train_set', train_data), ('validation_set', validation_data),
                     ('ground_truth_overlap_yaw', ground_truth_mapping)):
    seq = np.empty((data.shape[0], 2), dtype=object)
    seq[:] = seq_idx
    np.savez_compressed(os.path.join(dst, name), overlaps=data, seq=seq)
  print('Finish saving the ground truth data for training and testing at: ', dst)
  return dst


def parse_args(argv):
  p = argparse.ArgumentParser(prog='python -m overlapnet_b200.gt_files',
                              description='Generate the overlap / yaw ground-truth files of a KITTI-layout sequence.')
  p.add_argument('config', nargs='?', default='config/demo.yml', help='YAML file with a Demo4 section')
  p.add_argument('--seq', default='07', help='sequence label stored with every row (default: 07)')
  g = p.add_mutually_exclusive_group()
  g.add_argument('--all-frames', action='store_true', help='every frame against every scan')
  g.add_argument('--frames', help="these frames against every scan: '0,5,9' or 'a:b'")
  return p.parse_args(argv)


def generate(config, seq_idx='07', frames=None):
  """Run demo4 for the loaded YAML dict.  ``frames``: None = frame 0 through ``com_overlap_yaw``
  (exactly the demo), 'all' or a list = every pair of those frames.  Returns the ground_truth folder."""
  from . import gt
  from .preprocess import _read_scan, load_files
  c = config['Demo4']
  scan_paths = load_files(c['scan_folder'])
  T_cam_velo = gt.load_calib(c['calib_file'])
  poses = kitti_poses_in_lidar(gt.load_poses(c['poses_file']), T_cam_velo)
  if frames is None:
    ground_truth_mapping = gt.com_overlap_yaw(scan_paths, poses, frame_idx=0)
  else:
    print('Start to compute ground truth overlap and yaw for every pair ...')
    clouds = [(lambda p=p: _read_scan(p)) for p in scan_paths]
    res = gt.overlap_yaw_all_pairs(clouds, poses, None if frames == 'all' else frames)
    ground_truth_mapping = gt.all_pairs_rows(res)
    print('Finish generating ground_truth_mapping! (%d pairs, %d skipped as out of range)'
          % (ground_truth_mapping.shape[0], res.n_pruned))
  dist_norm_data = normalize_data(ground_truth_mapping)
  train_data, validation_data = split_train_val(dist_norm_data)
  return save_ground_truth(c['dst_folder'], seq_idx, ground_truth_mapping, train_data, validation_data)


def main(argv=None):
  from .config import load_config
  args = parse_args(sys.argv[1:] if argv is None else argv)
  config = load_config(args.config)
  frames = None
  if args.all_frames:
    frames = 'all'
  elif args.frames:
    from .preprocess import load_files
    frames = parse_frames(args.frames, len(load_files(config['Demo4']['scan_folder'])))
  return generate(config, args.seq, frames)


if __name__ == '__main__':
  main()
