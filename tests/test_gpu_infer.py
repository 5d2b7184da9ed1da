"""The drop-in ``Infer`` class against the oracle's restatement of the reference's call semantics
(infer.py:124-265): same .npy inputs, same LEFT/RIGHT convention, same return shapes and dtypes,
same error behaviour."""
import copy
import os

import numpy as np
import pytest

from oracle import network as N
from oracle import projection as P
from oracle.infer_ref import InferRef
from overlapnet_b200 import synth, weights as W

pytestmark = pytest.mark.gpu

MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
         'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
         'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
         'additional_unsymmetric_layer3a': True}


def check_yaw(yaw_gpu, yaw_ref, corr_ref, rel=2e-4):
  for p in range(len(yaw_ref)):
    if int(yaw_gpu[p]) != int(yaw_ref[p]):
      kg, kr = 180 - int(yaw_gpu[p]), 180 - int(yaw_ref[p])
      assert corr_ref[p, kr] - corr_ref[p, kg] <= rel * np.abs(corr_ref[p]).max(), (p, yaw_gpu[p], yaw_ref[p])


@pytest.fixture(scope='module')
def dataset(tmp_path_factory):
  """A preprocessed data folder laid out like the reference's (depth/ normal/ *.npy), generated
  with the oracle from seeded synthetic clouds, plus seeded weights in the .npz container."""
  root = tmp_path_factory.mktemp('data')
  seq = root / '07'
  (seq / 'depth').mkdir(parents=True)
  (seq / 'normal').mkdir()
  base = synth.kitti_like_cloud(900, n_points=60000)
  for i in range(4):
    if i < 3:
      ang = np.deg2rad(25.0 * i)                       # same scene rotated about z: a known yaw
      c, s = np.cos(ang), np.sin(ang)
      pts = base.copy()
      pts[:, 0], pts[:, 1] = c * base[:, 0] - s * base[:, 1], s * base[:, 0] + c * base[:, 1]
    else:
      pts = synth.kitti_like_cloud(901, n_points=60000)
    rng, vert, _, _ = P.range_projection(pts)
    np.save(str(seq / 'depth' / ('%06d.npy' % i)), rng)
    np.save(str(seq / 'normal' / ('%06d.npy' % i)), P.gen_normal_map(rng, vert))
  w = N.glorot_weights(4, MODEL, seed=3)
  # spread the overlaps of the four scans' pairs over (0,1) (tests/test_gpu_network.py explains why)
  imgs = np.stack([np.concatenate([np.load(str(seq / 'depth' / ('%06d.npy' % i)))[..., None],
                                   np.load(str(seq / 'normal' / ('%06d.npy' % i)))], -1) for i in range(4)])
  fvs = N.leg_forward(imgs.astype(np.float32), w, MODEL)
  li, ri = np.array([1, 0, 0, 1, 3, 1, 2]), np.array([0, 1, 2, 2, 0, 3, 0])   # no self pair: its logit is an outlier
  _, _, _, z0 = N.heads_forward(fvs[li], fvs[ri], w, MODEL, return_logit=True)
  w = N.spread_dense(w, z0, target_std=1.5)
  wpath = str(root / 'weights.npz')
  W.save_npz(wpath, w)
  cfg = {'pretrained_weightsfilename': wpath, 'use_depth': True, 'use_normals': True,
         'use_class_probabilities': False, 'use_class_probabilities_pca': False, 'use_intensity': False,
         'data_root_folder': str(root), 'infer_seqs': '07', 'batch_size': 16, 'model': copy.deepcopy(MODEL)}
  return cfg, w


@pytest.mark.parametrize('prec', ['fp32', 'f16_tc'])
def test_infer_api_matches_reference_semantics(dataset, prec):
  from overlapnet_b200.infer import Infer
  cfg, w = dataset
  cfg = copy.deepcopy(cfg)
  inf = Infer(cfg, precision=prec)
  ref = InferRef(copy.deepcopy(cfg), w)
  assert cfg['model']['inputShape'] == [64, 900, 4]            # mutated in place like infer.py:76-82
  assert inf.no_input_channels == 4 and inf.batch_size == 16 and inf.seq == '07'

  # ---- infer_one: LEFT = file2, RIGHT = file1; overlap (1,) f32, yaw (1,) int
  ov, yaw = inf.infer_one('/any/where/000000.bin', '000001.bin')
  ov_r, yaw_r, corr_r = ref.infer_one('000000.bin', '000001.bin')
  assert ov.shape == (1,) and ov.dtype == np.float32 and yaw.shape == (1,) and yaw.dtype.kind == 'i'
  assert list(inf.filenames) == ['000001', '000000']
  assert abs(float(ov[0]) - float(ov_r[0])) <= 1e-3
  check_yaw(yaw, yaw_r, corr_r)

  # ---- create_feature_volumes: (n,1,360,128) float32
  fv = inf.create_feature_volumes(['000000', '000003'])
  fv_r = ref.create_feature_volumes(['000000', '000003'])
  assert fv.shape == (2, 1, 360, 128) and fv.dtype == np.float32
  assert np.abs(fv - fv_r).max() / np.abs(fv_r).max() <= (2e-5 if prec == 'fp32' else 1e-4)

  # ---- infer_multiple: stateful bank, ids must come 0,1,2,...
  assert inf.infer_multiple(0, []) is None and ref.infer_multiple(0, []) is None
  r1 = inf.infer_multiple(1, [0])
  r1_ref = ref.infer_multiple(1, [0])
  assert r1[0].shape == () and r1[1].shape == (1,)              # squeeze() of one pair is 0-d (infer.py:197)
  assert abs(float(r1[0]) - float(r1_ref[0])) <= 1e-3
  r2 = inf.infer_multiple(2, [0, 1])
  r2_ref = ref.infer_multiple(2, [0, 1])
  assert r2[0].shape == (2,) and r2[1].shape == (2,)
  assert np.abs(r2[0] - r2_ref[0]).max() <= 1e-3
  check_yaw(r2[1], r2_ref[1], r2_ref[2])
  assert len(inf.feature_volumes) == 3 and inf.feature_volumes[0].shape == (1, 360, 128)

  # ---- infer_multiple_vs_multiple: LEFT = second_idxs, RIGHT = first_idxs
  names = ['000000', '000001.bin', '/x/000003.bin']
  r3 = inf.infer_multiple_vs_multiple(names, [0, 1, 2], [2, 1, 1])
  r3_ref = ref.infer_multiple_vs_multiple(names, [0, 1, 2], [2, 1, 1])
  assert np.abs(r3[0] - r3_ref[0]).max() <= 1e-3
  check_yaw(r3[1], r3_ref[1], r3_ref[2])
  assert r3[1][1] == 0                                           # a scan against itself
  assert inf.feature_volumes.shape == (3, 1, 360, 128)
  assert inf.infer_multiple_vs_multiple(names, [], []) is None


def test_infer_error_behaviour(dataset):
  from overlapnet_b200.infer import Infer
  cfg, _ = dataset
  inf = Infer(copy.deepcopy(cfg), precision='fp32')
  with pytest.raises(Exception, match='only works with .bin files'):
    inf.infer_one('a.pcd', 'b.bin')
  with pytest.raises(Exception, match='same size'):
    inf.infer_multiple_vs_multiple(['000000'], [0, 0], [0])
  with pytest.raises(Exception, match='Could not read depth image'):
    inf.create_feature_volumes(['999999'])
  bad = copy.deepcopy(cfg)
  bad['infer_seqs'] = 'nope'
  inf2 = Infer(bad, precision='fp32')
  with pytest.raises(Exception, match='first generate preprocessed input data'):
    inf2.infer_one('000000.bin', '000001.bin')
  worse = copy.deepcopy(cfg)
  worse['model']['legsType'] = 'NoSuchLegs'
  with pytest.raises(AttributeError):
    Infer(worse)
  missing = copy.deepcopy(cfg)
  del missing['use_depth']
  with pytest.raises(KeyError):                                  # infer.py:63 reads it unguarded
    Infer(missing)


def test_infer_raw_cloud_extension(dataset, tmp_path):
  """Extension: raw .bin scans through the fused projection kernels give the same answer as the
  .npy round trip of the reference flow."""
  from overlapnet_b200.infer import Infer
  cfg, _ = dataset
  inf = Infer(copy.deepcopy(cfg), precision='fp32')
  base = synth.kitti_like_cloud(900, n_points=60000)
  ang = np.deg2rad(25.0)
  rot = base.copy()
  rot[:, 0] = np.cos(ang) * base[:, 0] - np.sin(ang) * base[:, 1]
  rot[:, 1] = np.sin(ang) * base[:, 0] + np.cos(ang) * base[:, 1]
  base.tofile(str(tmp_path / '000000.bin'))
  rot.tofile(str(tmp_path / '000001.bin'))
  ov_raw, yaw_raw = inf.infer_one_raw(str(tmp_path / '000000.bin'), str(tmp_path / '000001.bin'))
  ov_npy, yaw_npy = inf.infer_one('000000.bin', '000001.bin')
  assert np.array_equal(ov_raw, ov_npy) and np.array_equal(yaw_raw, yaw_npy)


def test_evaluation_flow_matches_reference_semantics(dataset, tmp_path):
  """testing.py:207-352 on the GPU path: every distinct scan encoded once, LEFT = imgf1, RIGHT =
  imgf2, statistics and validation_results.npz -- against the oracle run pair by pair."""
  from overlapnet_b200 import evaluate as E
  cfg, w = dataset
  cfg = copy.deepcopy(cfg)
  gt = np.array([[0, 1, 0.93, 155.0], [1, 0, 0.93, 205.0], [2, 0, 0.80, 230.0], [3, 1, 0.05, 17.0], [0, 0, 1.0, 180.0]])
  (tmp_path / '07' / 'ground_truth').mkdir(parents=True)
  seq = np.empty((len(gt), 2), dtype=object); seq[:] = '07'
  np.savez_compressed(str(tmp_path / '07' / 'ground_truth' / 'ground_truth_overlap_yaw.npz'), overlaps=gt, seq=seq)
  run_cfg = dict(cfg, testing_seqs='07', imgpath=cfg['data_root_folder'], data_root_folder=str(tmp_path),
                 experiments_path=str(tmp_path), testname='exp', no_test_pairs=10 ** 9)
  del run_cfg['infer_seqs']
  m, stats = E.run_testing(run_cfg, precision='fp32')
  saved = np.load(str(tmp_path / 'exp' / 'validation_results.npz'))['arr_0']
  assert np.array_equal(saved, m) and m.shape == (5, 4)
  assert np.array_equal(m[:, :2], gt[:, :2])
  ref = InferRef(copy.deepcopy(cfg), w)
  for row in m:
    a, b = '%06d.bin' % int(row[0]), '%06d.bin' % int(row[1])
    ov_r, yaw_r, corr_r = ref.infer_one(b, a)               # infer_one: LEFT = file2, RIGHT = file1
    assert abs(row[2] - float(ov_r[0])) <= 1e-3
    check_yaw(np.array([180 - int(row[3])]), yaw_r, corr_r)
  want = E.error_statistics(m[:, 2], m[:, 3], gt[:, 2], gt[:, 3])
  assert stats == want and stats['yaw_pairs'] == 4


def test_infer_four_cue_input_matches_reference_semantics(tmp_path):
  """BASELINE config 3's input: depth + normal + 20 class probabilities + intensity = 25 channels in the
  reference's channel order (ImagePairOverlapOrientationSequence.py:143-207), read from the folders the
  reference's feeder reads (depth/ normal/ probability/ intensity/), through the drop-in Infer."""
  from overlapnet_b200.infer import Infer
  root = tmp_path
  seq = root / '07'
  for sub in ('depth', 'normal', 'probability', 'intensity'):
    (seq / sub).mkdir(parents=True)
  x = synth.range_like_images(17, 3, 25)                          # depth, normal x3, prob x20, intensity
  # three scans of DIFFERENT statistics (nearer / farther scene, other class mix, darker returns): three iid-noise
  # images give near-identical volumes, a logit std of 0.0018 and an 850x amplification at spread 1.5 -- a
  # numerical-analysis stress case (tools/precision_study.py), not a scan pair
  x[1, ..., 0] *= 0.4
  x[2, ..., 0] *= 1.8
  x[1, ..., 4:24] = np.roll(x[1, ..., 4:24], 5, axis=-1) * 0.5
  x[2, ..., 24] *= 0.2
  for i in range(3):
    np.save(str(seq / 'depth' / ('%06d.npy' % i)), x[i, :, :, 0])
    np.save(str(seq / 'normal' / ('%06d.npy' % i)), x[i, :, :, 1:4])
    np.save(str(seq / 'probability' / ('%06d.npy' % i)), x[i, :, :, 4:24])
    np.save(str(seq / 'intensity' / ('%06d.npy' % i)), x[i, :, :, 24])
  w = N.glorot_weights(25, MODEL, seed=4)
  fvs = N.leg_forward(x, w, MODEL)
  li, ri = np.array([1, 0, 2, 1]), np.array([0, 2, 1, 2])
  _, _, _, z0 = N.heads_forward(fvs[li], fvs[ri], w, MODEL, return_logit=True)
  w = N.spread_dense(w, z0, target_std=1.5)
  wpath = str(root / 'w.npz')
  W.save_npz(wpath, w)
  cfg = {'pretrained_weightsfilename': wpath, 'use_depth': True, 'use_normals': True, 'use_class_probabilities': True,
         'use_class_probabilities_pca': False, 'use_intensity': True, 'data_root_folder': str(root),
         'infer_seqs': '07', 'batch_size': 16, 'model': copy.deepcopy(MODEL)}
  inf = Infer(copy.deepcopy(cfg), precision='f16_tc')
  ref = InferRef(copy.deepcopy(cfg), w)
  assert inf.no_input_channels == 25 and inf.inputShape == [64, 900, 25]
  names = ['000000', '000001', '000002']
  fv = inf.create_feature_volumes(names)
  fv_r = ref.create_feature_volumes(names)
  assert np.abs(fv - fv_r).max() / np.abs(fv_r).max() <= 1e-4
  got = inf.infer_multiple_vs_multiple(names, [0, 2, 1, 2], [1, 0, 2, 1])     # LEFT = second_idxs, RIGHT = first_idxs
  want = ref.infer_multiple_vs_multiple(names, [0, 2, 1, 2], [1, 0, 2, 1])
  assert np.abs(got[0] - want[0]).max() <= 1e-3
  check_yaw(got[1], want[1], want[2])
