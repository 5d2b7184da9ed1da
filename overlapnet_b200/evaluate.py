"""The evaluation flow of the reference's ``src/two_heads/testing.py`` (:207-352) on the GPU path:
load the ground-truth pair lists, encode every distinct scan once, run both heads on all pairs,
compute the overlap / yaw error statistics and write ``validation_results.npz``.

testing.py is a script; here the same steps are functions so that they can be tested:
``load_overlap_npz``   overlap_orientation_npz_file2string_string_nparray.py:8-87 (both npz formats)
``testdata_files``     the three test-set selection rules of testing.py:67-92
``evaluate_pairs``     testing.py:233-271 (dedup + leg + heads), :274-323 (statistics), :339-352 (npz)
``run_testing``        the script body driven by the same YAML dict
Plots (matplotlib) are not produced.  All network arithmetic goes through ``Infer`` -> C ABI."""
import logging
import os

import numpy as np

logger = logging.getLogger('overlapnet_b200.evaluate')


def load_overlap_npz(npzfilenames, shuffle=True):
  """(imgf1, imgf2, dir1, dir2, overlap, orientation) from ground-truth npz files: scan ids as
  '%06d' strings, sequence names ('' for the single-array format), overlap and yaw-bin arrays."""
  imgf1_all, imgf2_all, dir1_all, dir2_all, overlap_all, orientation_all = [], [], [], [], [], []
  for name in npzfilenames:
    h = np.load(name, allow_pickle=True)
    table = h[h.files[0]] if len(h.files) == 1 else h['overlaps']
    n = table.shape[0]
    imgf1 = np.char.mod('%06d', table[:, 0])
    imgf2 = np.char.mod('%06d', table[:, 1])
    overlap, orientation = table[:, 2], table[:, 3]
    if len(h.files) == 1:                       # old format: no sequence column
      dir1 = dir2 = np.array([''] * n)
    else:
      dir1, dir2 = np.asarray(h['seq'][:, 0]), np.asarray(h['seq'][:, 1])
    if shuffle:
      perm = np.random.permutation(n)
      imgf1, imgf2, dir1, dir2 = imgf1[perm], imgf2[perm], dir1[perm], dir2[perm]
      overlap, orientation = overlap[perm], orientation[perm]
    imgf1_all.extend(imgf1.tolist()); imgf2_all.extend(imgf2.tolist())
    dir1_all.extend(dir1.tolist()); dir2_all.extend(dir2.tolist())
    overlap_all.append(np.asarray(overlap, dtype=float))
    orientation_all.append(np.asarray(orientation, dtype=float))
  cat = lambda parts: np.concatenate(parts) if parts else np.zeros(0)
  return imgf1_all, imgf2_all, dir1_all, dir2_all, cat(overlap_all), cat(orientation_all)


def testdata_files(config):
  """testing.py:67-92: 'testing_seqs' -> the sequence's complete ground truth; else 'training_seqs'
  -> their validation sets; else the single file 'testdata_npzfile'."""
  root = config.get('data_root_folder', '')
  if 'testing_seqs' in config:
    return [os.path.join(root, seq, 'ground_truth/ground_truth_overlap_yaw.npz') for seq in [config['testing_seqs']]]
  if 'training_seqs' in config:
    return [os.path.join(root, seq, 'ground_truth/validation_set.npz') for seq in config['training_seqs'].split()]
  return [config['testdata_npzfile']]


def pair_indices(imgf1, imgf2):
  """testing.py:244-254: the distinct scans (here in sorted order; the reference uses set order)
  and, per pair, their positions (n, 2)."""
  allimgs = np.array(sorted(set(imgf1) | set(imgf2)))
  idx = np.zeros((len(imgf1), 2), dtype=np.int64)
  idx[:, 0] = np.searchsorted(allimgs, imgf1)
  idx[:, 1] = np.searchsorted(allimgs, imgf2)
  return allimgs.tolist(), idx


def error_statistics(model_overlap, model_argmax, gt_overlap, gt_orientation, network_output_size=360):
  """testing.py:274-323: mean / max / RMS of |overlap error| and of the circular yaw-bin error over
  the pairs with ground-truth overlap > 0.7."""
  d_ov = np.abs(np.asarray(model_overlap, dtype=float) - gt_overlap)
  stats = {'overlap_mean': float(np.mean(d_ov)), 'overlap_max': float(np.max(d_ov)),
           'overlap_rms': float(np.sqrt(np.mean(d_ov * d_ov)))}
  a = np.abs(np.asarray(model_argmax, dtype=float) - gt_orientation)
  d_yaw = np.minimum(a, network_output_size - a)[gt_overlap > 0.7]
  if d_yaw.size:
    stats.update(yaw_mean=float(np.mean(d_yaw)), yaw_max=float(np.max(d_yaw)),
                 yaw_rms=float(np.sqrt(np.mean(d_yaw * d_yaw))), yaw_pairs=int(d_yaw.size))
  else:
    stats.update(yaw_mean=float('nan'), yaw_max=float('nan'), yaw_rms=float('nan'), yaw_pairs=0)
  return stats


def yaw_to_argmax(yaw):
  """The correlation head's argmax from the yaw ``Infer`` returns: yaw = 180 - argmax at every
  leg_output_width (infer.py:158, :198, :233), so argmax = 180 - yaw, in [0, leg_output_width)."""
  return 180 - np.asarray(yaw, dtype=np.int64)


def evaluate_pairs(infer, imgf1, imgf2, gt_overlap, gt_orientation, out_dir=None):
  """Encode each distinct scan once, run the heads on every pair with LEFT = imgf1, RIGHT = imgf2
  (ImagePairOverlapSequenceFeatureVolume.py:44-45), and evaluate.  Returns (overlapmatrix (n,4)
  [imgf1, imgf2, overlap, argmax], stats); writes ``validation_results.npz`` when out_dir is given."""
  allimgs, idx = pair_indices(imgf1, imgf2)
  logger.info('  Number of feature volumes: %d', len(allimgs))
  infer._set_bank(infer._create_feature_volumes_device(allimgs))
  infer._fv_as_array = True
  logger.info('Compute head for all %d test pairs ...', idx.shape[0])
  overlap, yaw = infer._run_heads(idx)
  overlap = np.squeeze(overlap, axis=1)
  argmax = yaw_to_argmax(yaw)
  stats = error_statistics(overlap, argmax, gt_overlap, gt_orientation, infer.network_output_size)
  m = np.zeros((len(imgf1), 4))
  m[:, 0] = np.array(imgf1).astype(float)
  m[:, 1] = np.array(imgf2).astype(float)
  m[:, 2] = overlap
  m[:, 3] = argmax
  if out_dir is not None:
    os.makedirs(out_dir, exist_ok=True)
    np.savez(os.path.join(out_dir, 'validation_results.npz'), m)           # testing.py:352 (key arr_0)
  return m, stats


def run_testing(config, precision='f16_tc'):
  """The body of testing.py for a loaded YAML dict.  Returns (overlapmatrix, stats)."""
  from .infer import Infer
  files = testdata_files(config)
  logger.info('load test data from %s ...', files)
  imgf1, imgf2, dir1, _, gt_overlap, gt_orientation = load_overlap_npz(files, shuffle=False)
  n = min(int(config.get('no_test_pairs', len(imgf1))), len(imgf1))        # testing.py:219-226
  imgf1, imgf2, gt_overlap, gt_orientation = imgf1[:n], imgf2[:n], gt_overlap[:n], gt_orientation[:n]
  cfg = dict(config)
  for key, default in (('use_depth', True), ('use_normals', True), ('use_class_probabilities', False),
                       ('use_class_probabilities_pca', False), ('use_intensity', False)):
    cfg.setdefault(key, default)                                           # testing.py:97-120 defaults
  # testing.py:216 loads the images from the sequence stored in the ground-truth npz (test_dir1[0]) and
  # ignores config['infer_seqs']; the config value is only a fallback for the old npz format (dir1 == '')
  if len(dir1) and str(dir1[0]) != '':
    cfg['infer_seqs'] = str(dir1[0])
  else:
    cfg.setdefault('infer_seqs', '')
  if 'imgpath' in cfg:
    cfg['data_root_folder'] = cfg['imgpath']
  infer = Infer(cfg, precision=precision)
  out_dir = os.path.join(config.get('experiments_path', '/tmp'), config.get('testname', 'experiment_test'))
  m, stats = evaluate_pairs(infer, imgf1, imgf2, gt_overlap, gt_orientation, out_dir)
  logger.info('Evaluation overlap on test data:')
  logger.info('  Evaluation: mean difference:   %f', stats['overlap_mean'])
  logger.info('  Evaluation: max  difference:   %f', stats['overlap_max'])
  logger.info('  Evaluation: RMS error        : %f', stats['overlap_rms'])
  logger.info('Evaluation yaw orientation (overlap>0.7) on test data:')
  logger.info('  Evaluation: mean difference:   %f', stats['yaw_mean'])
  logger.info('  Evaluation: max  difference:   %f', stats['yaw_max'])
  logger.info('  Evaluation: RMS error        : %f', stats['yaw_rms'])
  return m, stats
