"""Monte Carlo localization on the GPU: the Philox words, determinism across handles, the network path against its host
composition, convergence with a sensor that knows the true pose, and the refusals.  Every stage against its float64
model is tests/test_gpu_mcl_stages.py."""
import copy
import math

import numpy as np
import pytest
import torch

from oracle import mcl as om
from overlapnet_b200 import mcl, synth
from overlapnet_b200._cabi import OvnError
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
         'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
         'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
         'additional_unsymmetric_layer3a': True}
SIGMA = (0.3, 0.2, math.radians(3.0))
WIDTH = 360


def _engine():
  return Engine(model=MODEL, precision='fp32', max_batch_scans=1, max_batch_pairs=16)


def holey_map(seed, K=40):
  """K keyframes scattered over 60 m x 40 m, rasterised within 4 m, with a block of cells cut out."""
  rng = np.random.default_rng(seed)
  kf = np.stack([rng.uniform(0, 60, K), rng.uniform(0, 40, K), rng.uniform(-np.pi, np.pi, K)], 1)
  idx = mcl.MapIndex(kf[:, :2], 0.5, 4.0)
  raster = idx.raster.copy()
  raster[10:30, 20:60] = -1                                    # a hole inside the map
  assert (raster >= 0).any() and (raster < 0).any()
  return kf, raster, idx


def _np(t):
  return t.cpu().numpy()


@pytest.mark.parametrize('seed', [0, 1, 0xDEADBEEF, 2 ** 64 - 1])
def test_philox_words_are_bit_exact(seed):
  eng = _engine()
  rng = np.random.default_rng(7)
  ctr = rng.integers(0, 2 ** 32, (5000, 4), dtype=np.uint64).astype(np.uint32)
  ctr[:3] = [[0, 0, 0, 0], [2 ** 32 - 1] * 4, [1, 2, 3, 4]]
  got = _np(eng.mcl_philox(seed, ctr)).view(np.uint32)
  assert np.array_equal(got, om.philox(seed, ctr))
  eng.close()


def _run(eng, kf, raster, idx, n, seed, steps):
  eng.mcl_set_map(kf, raster, idx.x0, idx.y0, idx.cell)
  eng.mcl_init('global', n, seed, init_radius=3.0)
  out = []
  for t in range(steps):
    odom = (1.0 + 0.1 * math.sin(t), 0.2 * math.cos(t), 0.05 * math.sin(0.3 * t))
    touched, nt = eng.mcl_predict(odom, SIGMA)
    ids = touched[:nt].cpu().numpy().astype(np.int64)
    ov = torch.as_tensor((np.sin(ids * 0.7 + t) * 0.5 + 0.5).astype(np.float32)).cuda()
    yaw = torch.as_tensor((ids * 37 + t) % 360 - 180).to(torch.int32).cuda()
    est = eng.mcl_update(ov, yaw, nt, 0.15, math.radians(20), 0.5)
    out.append((_np(eng.mcl_particles()), est))
  return out


def test_twenty_steps_are_bit_identical_across_handles():
  kf, raster, idx = holey_map(11)
  a = _run(_engine(), kf, raster, idx, 100003, 42, 20)
  b = _run(_engine(), kf, raster, idx, 100003, 42, 20)
  assert any(e['resampled'] for _, e in a)
  for (pa, ea), (pb, eb) in zip(a, b):
    assert np.array_equal(pa.view(np.uint64), pb.view(np.uint64))
    assert ea == eb


def test_step_equals_encode_heads_and_step_observed():
  """The network path is plumbing: step(cloud) = encode + heads_1vsN(touched) + step_observed, bit for bit."""
  from overlapnet_b200.infer import Infer
  cfg = {'pretrained_weightsfilename': '', 'use_depth': True, 'use_normals': True, 'use_class_probabilities': False,
         'use_class_probabilities_pca': False, 'use_intensity': False, 'data_root_folder': '', 'infer_seqs': '',
         'batch_size': 4, 'model': copy.deepcopy(MODEL)}
  infer = Infer(cfg)
  K = 6
  poses = np.tile(np.eye(4), (K, 1, 1))
  for k in range(K):
    a = 0.3 * k
    poses[k, :2, :2] = [[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]]
    poses[k, 0, 3] = 2.0 * k
  clouds = [synth.kitti_like_cloud(900 + k, n_points=8000) for k in range(K)]
  m = mcl.OverlapMCL(infer, clouds, poses, max_distance=3.0)
  query = synth.kitti_like_cloud(77, n_points=8000)
  odoms = [(0.0, 0.0, 0.0), (1.0, 0.1, 0.05), (1.5, -0.2, 0.1)]
  m.init_global(5000, 3, init_radius=2.0)
  direct = [m.step(query, o) for o in odoms]
  p_direct = m.particles()
  eng = infer._engine
  m.init_global(5000, 3, init_radius=2.0)
  composed = []
  for o in odoms:
    q = infer.encode_clouds([query])[0]
    composed.append(m.step_observed(o, lambda ids: eng.heads_1vsN(m.bank, q, cand_idx=ids)[:2]))
  assert direct == composed and any(e['n_touched'] > 0 for e in direct)
  assert np.array_equal(p_direct.view(np.uint64), m.particles().view(np.uint64))


# ---- convergence with a sensor that knows the true pose ---------------------------------------------------------
# Thresholds checked first with oracle/mcl.py's filter on the CPU at 10^4 particles, seeds 0..4, 300 steps of this
# scenario: every seed within 2 m from step 30 on; after step 50 the largest position error was 1.57 m and the
# largest yaw error 0.78 degrees (0.78 bins).
CONV = dict(cell=0.5, max_distance=3.0, sigma_overlap=0.05, sigma_yaw=math.radians(10.0),
            motion_sigma=(0.1, 0.1, math.radians(1.0)))


@pytest.mark.parametrize('seed', range(5))
def test_global_localization_converges_with_a_true_sensor(seed):
  poses = om.scenario()
  kfi, qi = mcl.split_sequence(len(poses), 2)                 # keyframes every 2 m, queries between them
  kf, truth = poses[kfi], poses[qi]
  odom = mcl.odometry(truth)
  idx = mcl.MapIndex(kf[:, :2], CONV['cell'], CONV['max_distance'])
  eng = _engine()
  eng.mcl_set_map(kf, idx.raster, idx.x0, idx.y0, idx.cell)
  eng.mcl_init('global', 10 ** 5, seed, init_radius=1.0)
  T = 200
  pos, yaw = np.zeros(T), np.zeros(T)
  for t in range(T):
    touched, nt = eng.mcl_predict(odom[t], CONV['motion_sigma'])
    ov, yw = om.fake_sensor(truth[t], kf)(touched[:nt].cpu().numpy())
    e = eng.mcl_update(torch.as_tensor(ov).cuda(), torch.as_tensor(yw).cuda(), nt, CONV['sigma_overlap'],
                       CONV['sigma_yaw'], 0.5)
    pos[t] = math.hypot(e['x'] - truth[t, 0], e['y'] - truth[t, 1])
    yaw[t] = abs(mcl.wrap_pi(e['theta'] - truth[t, 2])) / (2 * math.pi / WIDTH)
  c = mcl.convergence_step(pos, 2.0)
  print('seed %d: converged at step %d, largest errors after step 50: %.2f m, %.2f bins'
        % (seed, c, pos[50:].max(), yaw[50:].max()))
  assert 0 <= c <= 50 and pos[50:].max() < 2.0 and yaw[50:].max() <= 2.0
  eng.close()


# ---- refusals ---------------------------------------------------------------------------------------------------
def _refused(fn):
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    fn()


def test_invalid_arguments_are_refused_and_the_handle_stays_usable():
  eng = _engine()
  kf, raster, idx = holey_map(3)
  _refused(lambda: eng.mcl_init('global', 10, 1, init_radius=1.0))                      # no map yet
  _refused(lambda: eng.mcl_set_map(kf, raster, idx.x0, idx.y0, 0.0))                    # cell
  _refused(lambda: eng.mcl_set_map(kf, raster, idx.x0, idx.y0, float('nan')))
  bad = raster.copy()
  bad[0, 0] = kf.shape[0]
  _refused(lambda: eng.mcl_set_map(kf, bad, idx.x0, idx.y0, idx.cell))                   # raster entry
  bad[0, 0] = -2
  _refused(lambda: eng.mcl_set_map(kf, bad, idx.x0, idx.y0, idx.cell))
  _refused(lambda: eng.mcl_set_map(kf[:0], raster, idx.x0, idx.y0, idx.cell))            # no keyframe
  _refused(lambda: eng.mcl_set_map(kf, raster[:0], idx.x0, idx.y0, idx.cell))            # empty raster
  eng.mcl_set_map(kf, raster, idx.x0, idx.y0, idx.cell)
  _refused(lambda: eng.mcl_predict((1, 0, 0), SIGMA))                                    # no particles yet
  for n in (0, -1, (1 << 24) + 1):
    _refused(lambda: eng.mcl_init('global', n, 1, init_radius=1.0))
  _refused(lambda: eng.mcl_init('global', 10, 1, init_radius=-1.0))
  _refused(lambda: eng.mcl_init('pose', 10, 1, pose=(0, 0, 0), sigma=(1, -1, 1)))
  eng.mcl_init('global', 1000, 1, init_radius=5.0)
  for stage in ('motion', 'lookup', 'loglik', 'weights', 'prefix', 'ancestors', 'scalars'):
    _refused(lambda: eng.mcl_stage(stage))                                             # nothing held yet
  _refused(lambda: eng.mcl_update(None, None, 0, 0.1, 0.1, 0.5))                         # update before predict
  _refused(lambda: eng.mcl_predict((1, 0, 0), (0.1, -0.1, 0.1)))                         # sigma < 0
  _refused(lambda: eng.mcl_predict((float('inf'), 0, 0), SIGMA))
  touched, nt = eng.mcl_predict((1, 0, 0), SIGMA)
  assert nt > 0
  ov = torch.full((nt + 1,), 0.5, device='cuda')
  yaw = torch.zeros((nt + 1,), dtype=torch.int32, device='cuda')
  _refused(lambda: eng.mcl_update(ov, yaw, nt + 1, 0.1, 0.1, 0.5))                       # count differs
  _refused(lambda: eng.mcl_update(ov, yaw, nt, 0.0, 0.1, 0.5))                           # sigma <= 0
  _refused(lambda: eng.mcl_update(ov, yaw, nt, 0.1, -1.0, 0.5))
  _refused(lambda: eng.mcl_update(ov, yaw, nt, 0.1, 0.1, 1.5))                           # rho
  _refused(lambda: eng.mcl_update(None, None, nt, 0.1, 0.1, 0.5))                        # NULL with n > 0
  est = eng.mcl_update(ov, yaw, nt, 0.1, 0.1, 0.5)                                       # the next valid call
  assert est['n_touched'] == nt and np.isfinite(est['x'])
  _refused(lambda: eng.mcl_update(ov, yaw, nt, 0.1, 0.1, 0.5))                           # no second update
  if not est['resampled']:
    _refused(lambda: eng.mcl_stage('ancestors'))                                        # no resampling held
  touched, nt = eng.mcl_predict((1, 0, 0), SIGMA)
  eng.mcl_update(ov, yaw, nt, 0.1, 0.1, 0.5)
  eng.close()


def test_no_touched_keyframe_skips_the_heads():
  """Every particle outside the raster: no keyframe is touched, the update takes no heads output, and the
  weights stay uniform."""
  eng = _engine()
  kf, raster, idx = holey_map(4)
  eng.mcl_set_map(kf, raster, idx.x0, idx.y0, idx.cell)
  eng.mcl_init('pose', 2000, 5, pose=(-1e4, -1e4, 0.0), sigma=(1.0, 1.0, 0.1))
  touched, nt = eng.mcl_predict((1.0, 0.0, 0.0), SIGMA)
  assert nt == 0
  est = eng.mcl_update(None, None, 0, 0.1, 0.1, 0.5)
  assert est['n_touched'] == 0 and not est['resampled']
  np.testing.assert_allclose(_np(eng.mcl_stage('weights')), 1.0 / 2000, rtol=1e-12)
  eng.close()


def test_cli_runs_end_to_end_on_a_synthetic_sequence(tmp_path):
  import json
  import yaml
  n = 12
  scans = tmp_path / 'velodyne'
  scans.mkdir()
  lines = []
  for i in range(n):
    synth.kitti_like_cloud(300 + i, n_points=6000).tofile(str(scans / ('%06d.bin' % i)))
    T = np.eye(4)[:3]
    T[0, 3] = 1.0 * i
    lines.append(' '.join('%.9f' % v for v in T.reshape(-1)))
  (tmp_path / 'poses.txt').write_text('\n'.join(lines) + '\n')
  (tmp_path / 'calib.txt').write_text('Tr: 1 0 0 0 0 1 0 0 0 0 1 0\n')
  net = {'pretrained_weightsfilename': '', 'use_depth': True, 'use_normals': True, 'use_class_probabilities': False,
         'use_intensity': False, 'batch_size': 4, 'model': copy.deepcopy(MODEL),
         'experiments_path': str(tmp_path / 'exp'), 'testname': 'mcl_cli'}
  (tmp_path / 'net.yml').write_text(yaml.safe_dump(net))
  demo = {'Demo3': {'network_config': str(tmp_path / 'net.yml'), 'scan_folder': str(scans),
                    'poses_file': str(tmp_path / 'poses.txt'), 'calib_file': str(tmp_path / 'calib.txt')}}
  (tmp_path / 'demo.yml').write_text(yaml.safe_dump(demo))
  s = mcl.main([str(tmp_path / 'demo.yml'), '--keyframe-stride', '2', '--particles', '2000', '--runs', '2',
                '--max-distance', '3'])
  out = tmp_path / 'exp' / 'mcl_cli'
  assert json.loads((out / 'mcl_summary.json').read_text()) == json.loads(json.dumps(s))
  r = np.load(str(out / 'mcl_results.npz'))
  assert s['keyframes'] == 6 and s['queries'] == 6 and s['runs'] == 2
  assert r['estimate'].shape == (2, 6, 3) and r['convergence_step'].shape == (2,)
  assert list(r['queries']) == [1, 3, 5, 7, 9, 11] and np.allclose(r['odometry'][1:], [2.0, 0.0, 0.0])
