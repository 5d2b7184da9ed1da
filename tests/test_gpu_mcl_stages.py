"""Every stage of Monte Carlo localization on the GPU against the float64 stage model oracle/mcl_stages.py, each from
the GPU's own input to it: initialisation, motion, lookup, touched list, log-likelihood, max, S, weights and
log-weights, the six sums through the ESS and the estimate, the resampling decision, the prefix sum, u0, the
ancestors and the gather.  Cases: the launch-geometry edges of N, maps of 1 to 5 000 keyframes, widths 360, 225 and
405, positions on raster-cell edges and far outside the raster, headings at +-pi and relative yaws on bin edges,
uniform, single-particle and subnormal weights, rho 0 and 1, a drive 1 km from the origin.  Then the refusals of
an update whose observations are not finite or leave no finite log-weight.  Prints the largest error / bound of
each stage and the decisions that fell in a tie band."""
import math

import numpy as np
import pytest
import torch

from oracle import mcl as om
from oracle import mcl_stages as M
from overlapnet_b200 import mcl
from overlapnet_b200._cabi import OvnError
from overlapnet_b200.engine import Engine
from test_geometry import head_model, image_size

pytestmark = pytest.mark.gpu

MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
         'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
         'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
         'additional_unsymmetric_layer3a': True}
SIGMA = (0.3, 0.2, math.radians(3.0))
WORST = {}
COUNTS = {'ties': 0, 'resampled': 0, 'steps': 0}


@pytest.fixture(scope='module', autouse=True)
def report():
  yield
  print('\nlargest error / bound per stage: ' + ', '.join('%s %.3g' % kv for kv in sorted(WORST.items())))
  print('%(steps)d updates checked, %(resampled)d resampled, %(ties)d decisions in a tie band' % COUNTS)


def _engine(width=360):
  if width == 360:
    return Engine(model=MODEL, precision='fp32', max_batch_scans=1, max_batch_pairs=16)
  s = {225: 15, 405: 27}[width]
  model = head_model(width, s)
  H, W = image_size(model, width)
  return Engine(model=model, precision='fp32', max_batch_scans=1, max_batch_pairs=16, proj_H=H, proj_W=W)


def _np(t):
  return t.cpu().numpy()


def gate(stage, ratio):
  r = np.asarray(ratio, np.float64)
  worst = float(r.max()) if r.size else 0.0
  WORST[stage] = max(WORST.get(stage, 0.0), worst)
  assert worst <= 1.0, (stage, worst, int(np.count_nonzero(r > 1)), r.size)


def exact(stage, bad):
  WORST[stage + ' (mismatches)'] = WORST.get(stage + ' (mismatches)', 0) + int(bad)
  assert bad == 0, (stage, bad)


def holey_map(seed, K=40, origin=(0.0, 0.0)):
  """K keyframes scattered over 60 m x 40 m, rasterised within 4 m, with a block of cells cut out."""
  rng = np.random.default_rng(seed)
  kf = np.stack([origin[0] + rng.uniform(0, 60, K), origin[1] + rng.uniform(0, 40, K), rng.uniform(-np.pi, np.pi, K)],
                1)
  idx = mcl.MapIndex(kf[:, :2], 0.5, 4.0)
  raster = idx.raster.copy()
  raster[10:30, 20:60] = -1
  return kf, raster, (idx.x0, idx.y0, idx.cell)


def line_map(K, spacing=0.5):
  """K keyframes every ``spacing`` m along x, one raster cell each (cell k holds keyframe k), 2 rows."""
  kf = np.stack([spacing * (np.arange(K) + 0.5), np.ones(K) * 0.5 * spacing, np.linspace(-3.0, 3.0, K)], 1)
  raster = np.tile(np.arange(K, dtype=np.int32), (2, 1))
  return kf, raster, (0.0, 0.0, spacing)


class Filter:
  """One handle's filter, every stage checked against the model as it runs."""

  def __init__(self, eng, kf, raster, geo, width=360):
    self.eng, self.kf, self.raster, self.geo, self.width = eng, np.asarray(kf, np.float64), raster, geo, width
    eng.mcl_set_map(self.kf, raster, *geo)

  def init_global(self, n, seed, radius):
    self.eng.mcl_init('global', n, seed, init_radius=radius)
    self.p, self.n, self.seed, self.step_no = _np(self.eng.mcl_particles()), n, seed, 0
    gate('init global', M.check_init_global(n, seed, self.kf, radius, self.p))
    self.lw0 = self.p[3, 0]

  def init_pose(self, n, seed, pose, sigma):
    self.eng.mcl_init('pose', n, seed, pose=pose, sigma=sigma)
    self.p, self.n, self.seed, self.step_no = _np(self.eng.mcl_particles()), n, seed, 0
    gate('init pose', M.check_init_pose(n, seed, pose, sigma, self.p))
    self.lw0 = self.p[3, 0]

  def predict(self, odom, sigma):
    touched, nt = self.eng.mcl_predict(odom, sigma)
    self.step_no += 1
    mo = _np(self.eng.mcl_stage('motion'))
    gate('motion', M.check_motion(self.p[0], self.p[1], self.p[2], self.seed, self.step_no, odom, sigma, mo))
    k = _np(self.eng.mcl_stage('lookup'))
    exact('lookup', np.count_nonzero(k != om.lookup(mo[0], mo[1], self.raster, *self.geo)))
    exact('touched', M.check_touched(k, self.kf.shape[0], _np(touched), nt))
    self.mo, self.k, self.ids = mo, k, _np(touched[:nt]).astype(np.int64)
    return self.ids

  def update(self, ov, yaw, s_o, s_psi, rho):
    nt = self.ids.size
    est = self.eng.mcl_update(torch.as_tensor(ov).cuda() if nt else None, torch.as_tensor(yaw).cuda() if nt else None,
                              nt, s_o, s_psi, rho)
    mo, n = self.mo, self.n
    ll = _np(self.eng.mcl_stage('loglik'))
    gate('loglik', M.check_loglik(self.k, mo[2], self.kf[:, 2], self.ids, ov, yaw, self.width, s_o, s_psi, ll))
    scal = _np(self.eng.mcl_stage('scalars'))
    w = _np(self.eng.mcl_stage('weights'))
    p = _np(self.eng.mcl_particles())
    rep = M.check_update(self.p[3], ll, mo[0], mo[1], mo[2], rho * float(n), scal, w,
                         None if est['resampled'] else p[3], self.seed, self.step_no)
    for key in ('S', 'weights', 'ess', 'x', 'y', 'theta') + (() if est['resampled'] else ('lw',)):
      gate(key, rep[key])
    exact('max, decision, u0', rep['exact'])
    COUNTS['ties'] += rep['tie']
    COUNTS['steps'] += 1
    exact('estimate readback', int(est['x'] != scal[3] or est['y'] != scal[4] or est['theta'] != scal[5]
                                   or est['ess'] != scal[2] or est['resampled'] != bool(scal[6])))
    if est['resampled']:
      COUNTS['resampled'] += 1
      cdf = _np(self.eng.mcl_stage('prefix'))
      exact('prefix', M.check_prefix(w, cdf))
      anc = _np(self.eng.mcl_stage('ancestors'))
      exact('ancestors', M.check_ancestors(cdf, scal[7], anc))
      exact('gather', np.count_nonzero(p[:3].view(np.uint64) != mo[:, anc].view(np.uint64))
            + np.count_nonzero(p[3].view(np.uint64) != np.float64(self.lw0).view(np.uint64)))
    else:
      exact('gather', np.count_nonzero(p[:3].view(np.uint64) != mo.view(np.uint64)))
    self.p = p
    return est, ll, w


def observe(rng, ids, mo=None, k=None, kf=None, width=360):
  """Random overlaps and yaws, with one overlap of 1 and one yaw on the expected bin."""
  nt = ids.size
  ov = rng.random(nt).astype(np.float32)
  yaw = rng.integers(-180, 540, nt).astype(np.int32)
  if nt:
    ov[0] = 1.0
    if mo is not None:
      i = np.flatnonzero(k == ids[-1])[0]
      yaw[-1] = 180 - M.expected_bin(om.wrap_pi(mo[2][i] - kf[ids[-1], 2]), width) % width
  return ov, yaw


# ---- the launch-geometry edges of N ------------------------------------------------------------------------------
NS = [1, 2, 255, 256, 257, 2047, 2048, 2049, 65537, 262143, 262144, 262145, 10 ** 6]


@pytest.mark.parametrize('n', NS)
def test_every_stage_at_the_launch_edges(n):
  eng = _engine()
  f = Filter(eng, *holey_map(n))
  f.init_global(n, 1234 + n, 6.0)
  rng = np.random.default_rng(n)
  for step, rho in enumerate((1.0, 0.0) if n >= 262143 else (1.0, 0.0, 1.0)):
    odom = (rng.uniform(-2, 2), rng.uniform(-1, 1), rng.uniform(-0.3, 0.3))
    ids = f.predict(odom, SIGMA)
    if n >= 2047:
      assert (f.k < 0).any() and (f.k >= 0).any()            # particles outside the raster and in its hole
    ov, yaw = observe(rng, ids, f.mo, f.k, f.kf)
    f.update(ov, yaw, 0.2, math.radians(15), rho)
  eng.close()


def test_pose_init_and_one_step_at_2_24():
  n = 1 << 24
  eng = _engine()
  f = Filter(eng, *holey_map(24))
  f.init_pose(n, 99, (20.0, 10.0, 3.1), (8.0, 6.0, 0.5))
  rng = np.random.default_rng(24)
  ids = f.predict((1.0, 0.5, 0.1), SIGMA)
  f.update(*observe(rng, ids, f.mo, f.k, f.kf), 0.2, math.radians(15), 1.0)
  eng.close()


# ---- maps: tiles of the compact, widths ---------------------------------------------------------------------------
@pytest.mark.parametrize('K', [1, 1023, 1024, 1025, 5000])
def test_every_stage_over_compact_tiles(K):
  """A line of K keyframes, one cell each; the particles sit on every keyframe, so the touched lists hold the first
  and last keyframe of each 1024-keyframe tile."""
  eng = _engine()
  kf, raster, geo = line_map(K)
  f = Filter(eng, kf, raster, geo)
  n = 8 * K + 3
  f.init_global(n, 7 + K, 0.0)                               # radius 0: each particle on its keyframe
  rng = np.random.default_rng(K)
  for rho in (1.0, 0.0):
    ids = f.predict((0.0, 0.0, 0.0), (0.02, 0.0, 0.01))
    tiles = set(range(0, K, 1024)) | set(range(1023, K, 1024)) | {K - 1}
    assert tiles <= set(ids.tolist()) or rho == 0.0
    f.update(*observe(rng, ids, f.mo, f.k, f.kf), 0.3, math.radians(10), rho)
  eng.close()


@pytest.mark.parametrize('width', [360, 225, 405])
def test_every_stage_at_each_width_with_edges(width):
  """Keyframes on raster-cell edges and one ulp to either side, and 1e3 to 1e15 m outside the raster; the
  keyframes' headings are set from the particles' own exact headings (no theta noise) so that the relative yaw lies
  on a bin edge or one ulp beside it, and headings of exactly +-pi."""
  eng = _engine(width)
  cell, x0, y0 = 0.5, 0.3, -0.7
  rows, cols = 8, 64
  base_x = x0 + cell * np.arange(1, 21)
  xs = np.concatenate([base_x, np.nextafter(base_x, -np.inf), np.nextafter(base_x, np.inf)])
  ys = np.full(xs.size, y0 + 3 * cell)
  ys[::7] = np.nextafter(ys[::7], -np.inf)
  far = np.array([1e3, -1e3, 1e9, -1e9, 1e15, -1e15])
  xs = np.concatenate([xs, far, np.full(6, 2.0)])
  ys = np.concatenate([ys, np.full(6, 1.0), far])
  K = xs.size
  raster = (np.arange(rows * cols, dtype=np.int32) % K).reshape(rows, cols)
  kf = np.stack([xs, ys, np.zeros(K)], 1)
  n, seed = 4 * K + 1, 31 + width
  # first run: the headings the particles hold after a predict without theta noise
  f = Filter(eng, kf, raster, (x0, y0, cell), width)
  f.init_global(n, seed, 0.0)
  f.predict((0.0, 0.0, 0.0), (0.0, 0.0, 0.0))
  th1 = f.mo[2]
  k0 = f.k.copy()
  first = {int(k): int(np.flatnonzero(k0 == k)[0]) for k in np.unique(k0[k0 >= 0])}
  # second run: the map's keyframe headings put those particles' relative yaw on a bin edge or one ulp beside it
  targets = [0.0, -math.pi / 2, math.pi / 2, math.pi, -math.pi]
  kth = np.zeros(K)
  for j, (kk, i) in enumerate(sorted(first.items())):
    t = th1[i] - targets[j % len(targets)]
    kth[kk] = [t, np.nextafter(t, -np.inf), np.nextafter(t, np.inf)][(j // len(targets)) % 3]
  kf[:, 2] = kth
  f = Filter(eng, kf, raster, (x0, y0, cell), width)
  f.init_global(n, seed, 0.0)
  rng = np.random.default_rng(width)
  for rho in (0.0, 1.0):
    ids = f.predict((0.0, 0.0, 0.0), (0.0, 0.0, 0.0))
    f.update(*observe(rng, ids, f.mo, f.k, f.kf, width), 0.25, math.radians(20), rho)
  # headings of exactly +-pi: a pose init without theta noise
  for pt in (math.pi, -math.pi):
    f.init_pose(2049, seed, (xs[0], ys[0], pt), (0.0, 0.0, 0.0))
    assert np.all(f.p[2] == om.PI)
    ids = f.predict((0.0, 0.0, 0.0), (0.0, 0.0, 0.0))
    assert np.all(f.mo[2] == om.PI)
    f.update(*observe(rng, ids, f.mo, f.k, f.kf, width), 0.25, math.radians(20), 1.0)
  eng.close()


# ---- weights ------------------------------------------------------------------------------------------------------
def test_uniform_weights_without_a_particle_on_the_map():
  eng = _engine()
  f = Filter(eng, *holey_map(4))
  f.init_pose(2049, 5, (-1e4, -1e4, 0.0), (1.0, 1.0, 0.1))
  for rho in (1.0, 0.0):
    ids = f.predict((1.0, 0.0, 0.0), SIGMA)
    assert ids.size == 0
    _, _, w = f.update(np.zeros(0, np.float32), np.zeros(0, np.int32), 0.1, 0.1, rho)
    assert np.all(w == w[0])
  eng.close()


def test_one_particle_holds_the_weight_and_the_rest_go_subnormal():
  """K = 5000 keyframes for 2049 particles: most keyframes hold at most one.  One touched keyframe observes 1,
  the rest observe spread overlaps with sigma_overlap 0.02, so log-likelihoods spread past 745 and weights go
  subnormal and to 0; then one particle holds nearly all the weight (ESS about 1)."""
  eng = _engine()
  kf, raster, geo = line_map(5000)
  f = Filter(eng, kf, raster, geo)
  f.init_global(2049, 3, 0.0)
  rng = np.random.default_rng(3)
  ids = f.predict((0.0, 0.0, 0.0), (0.0, 0.0, 0.0))
  ov = rng.random(ids.size).astype(np.float32)
  ov[np.bincount(f.k[f.k >= 0], minlength=5000)[ids] == 1] *= 0.5
  est, ll, w = f.update(ov, np.full(ids.size, 180, np.int32), 0.02, 10.0, 0.0)
  assert (w == 0).any() and ((w > 0) & (w < np.finfo(np.float64).tiny)).any()
  ids = f.predict((0.0, 0.0, 0.0), (0.0, 0.0, 0.0))
  single = int(np.flatnonzero(np.bincount(f.k[f.k >= 0], minlength=5000)[ids] == 1)[0])
  ov = np.zeros(ids.size, np.float32)
  ov[single] = 1.0
  est, _, w = f.update(ov, np.full(ids.size, 180, np.int32), 0.01, 10.0, 1.0)
  assert est['ess'] < 1.001 and est['resampled']
  eng.close()


def test_a_drive_one_kilometre_from_the_origin():
  eng = _engine()
  f = Filter(eng, *holey_map(8, origin=(1000.0, -700.0)))
  f.init_global(65537, 8, 4.0)
  rng = np.random.default_rng(8)
  for t in range(6):
    ids = f.predict((1.5, 0.1 * math.sin(t), 0.05), SIGMA)
    f.update(*observe(rng, ids, f.mo, f.k, f.kf), 0.15, math.radians(10), 0.5)
  eng.close()


# ---- handles reused at other sizes ---------------------------------------------------------------------------------
def _steps(eng, n, seed, steps=3):
  kf, raster, geo = holey_map(11)
  eng.mcl_set_map(kf, raster, *geo)
  eng.mcl_init('global', n, seed, init_radius=3.0)
  out = []
  for t in range(steps):
    touched, nt = eng.mcl_predict((1.0, 0.2, 0.05 * t), SIGMA)
    ids = _np(touched[:nt]).astype(np.int64)
    ov = torch.as_tensor((np.sin(ids * 0.7 + t) * 0.5 + 0.5).astype(np.float32)).cuda()
    yaw = torch.as_tensor((ids * 37 + t) % 360 - 180).to(torch.int32).cuda()
    est = eng.mcl_update(ov, yaw, nt, 0.15, math.radians(20), 1.0 if t % 2 else 0.0)
    out.append((_np(eng.mcl_particles()).view(np.uint64), est))
  return out


def _same(a, b):
  for (pa, ea), (pb, eb) in zip(a, b):
    assert np.array_equal(pa, pb) and ea == eb


def test_a_reused_handle_gives_the_bits_of_a_fresh_one():
  eng = _engine()
  _steps(eng, 1 << 24, 1, steps=1)
  after_big = _steps(eng, 31, 5)
  kf, raster, geo = line_map(5000)                           # a larger map in between
  eng.mcl_set_map(kf, raster, *geo)
  eng.mcl_init('global', 1000, 2, init_radius=0.0)
  eng.mcl_predict((0.0, 0.0, 0.0), SIGMA)
  after_map = _steps(eng, 31, 5)
  eng.close()
  fresh = _engine()
  want = _steps(fresh, 31, 5)
  fresh.close()
  _same(after_big, want)
  _same(after_map, want)


# ---- refusals: observations that are not finite --------------------------------------------------------------------
def _predicted(n=4099, seed=17):
  eng = _engine()
  kf, raster, geo = holey_map(17)
  eng.mcl_set_map(kf, raster, *geo)
  eng.mcl_init('global', n, seed, init_radius=5.0)
  touched, nt = eng.mcl_predict((1.0, 0.0, 0.1), SIGMA)
  assert nt > 2
  return eng, nt


def _obs(nt):
  rng = np.random.default_rng(nt)
  return rng.random(nt).astype(np.float32) * 0.9, rng.integers(-180, 180, nt).astype(np.int32)


def _held_as_after_predict(eng, before, mo):
  assert np.array_equal(_np(eng.mcl_particles()).view(np.uint64), before.view(np.uint64))
  assert np.array_equal(_np(eng.mcl_stage('motion')).view(np.uint64), mo.view(np.uint64))
  for stage in ('loglik', 'weights', 'scalars'):
    with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
      eng.mcl_stage(stage)


@pytest.mark.parametrize('bad', [float('nan'), float('inf'), float('-inf')])
def test_an_overlap_that_is_not_finite_is_refused(bad):
  eng, nt = _predicted()
  before, mo = _np(eng.mcl_particles()), _np(eng.mcl_stage('motion'))
  ov, yaw = _obs(nt)
  ov[nt // 2] = bad
  with pytest.raises(OvnError, match='overlap is not finite'):
    eng.mcl_update(torch.as_tensor(ov).cuda(), torch.as_tensor(yaw).cuda(), nt, 0.2, 0.3, 1.0)
  _held_as_after_predict(eng, before, mo)
  eng.close()


def test_no_finite_log_weight_is_refused():
  """sigma_overlap = the smallest positive double: every particle's ((1 - O) / s_o)^2 overflows, so every
  log-likelihood is -inf."""
  eng, nt = _predicted()
  before, mo = _np(eng.mcl_particles()), _np(eng.mcl_stage('motion'))
  ov, yaw = _obs(nt)
  with pytest.raises(OvnError, match='no particle has a finite log-weight'):
    eng.mcl_update(torch.as_tensor(ov).cuda(), torch.as_tensor(yaw).cuda(), nt, 5e-324, 0.3, 1.0)
  _held_as_after_predict(eng, before, mo)
  eng.close()


def test_a_retry_after_a_refusal_equals_the_valid_update_first():
  ov, yaw = None, None
  runs = []
  for refuse_first in (False, True):
    eng, nt = _predicted()
    ov, yaw = _obs(nt)
    if refuse_first:
      bad = ov.copy()
      bad[0] = np.nan
      with pytest.raises(OvnError):
        eng.mcl_update(torch.as_tensor(bad).cuda(), torch.as_tensor(yaw).cuda(), nt, 0.2, 0.3, 1.0)
      with pytest.raises(OvnError):
        eng.mcl_update(torch.as_tensor(ov).cuda(), torch.as_tensor(yaw).cuda(), nt, 5e-324, 0.3, 1.0)
    est = eng.mcl_update(torch.as_tensor(ov).cuda(), torch.as_tensor(yaw).cuda(), nt, 0.2, 0.3, 1.0)
    touched, nt2 = eng.mcl_predict((1.0, 0.0, 0.1), SIGMA)
    est2 = eng.mcl_update(torch.as_tensor(_obs(nt2)[0]).cuda(), torch.as_tensor(_obs(nt2)[1]).cuda(), nt2, 0.2, 0.3,
                          0.5)
    runs.append(([est, est2], _np(eng.mcl_particles()).view(np.uint64),
                 [_np(eng.mcl_stage(s)).view(np.uint64) for s in ('loglik', 'weights', 'scalars')]))
    eng.close()
  assert runs[0][0] == runs[1][0] and runs[0][0][0]['resampled']
  assert np.array_equal(runs[0][1], runs[1][1])
  for a, b in zip(runs[0][2], runs[1][2]):
    assert np.array_equal(a, b)


@pytest.mark.parametrize('precision', ['fp32', 'f16_tc'])
def test_step_volume_with_a_nan_query_is_refused(precision):
  """A query volume holding NaN: the tensor-core heads poison every touched overlap with NaN, and step_volume
  raises instead of returning a NaN estimate; the fp32 heads' ReLU (fmaxf) drops the NaN, so their overlaps and the
  estimate stay finite.  Either way no NaN reaches the particles, and the next valid step works."""
  import copy
  from overlapnet_b200 import synth
  from overlapnet_b200.infer import Infer
  cfg = {'pretrained_weightsfilename': '', 'use_depth': True, 'use_normals': True, 'use_class_probabilities': False,
         'use_class_probabilities_pca': False, 'use_intensity': False, 'data_root_folder': '', 'infer_seqs': '',
         'batch_size': 4, 'model': copy.deepcopy(MODEL)}
  infer = Infer(cfg, precision=precision)
  K = 6
  poses = np.tile(np.eye(4), (K, 1, 1))
  poses[:, 0, 3] = 2.0 * np.arange(K)
  clouds = [synth.kitti_like_cloud(900 + k, n_points=8000) for k in range(K)]
  m = mcl.OverlapMCL(infer, clouds, poses, max_distance=3.0)
  m.init_global(5000, 3, init_radius=2.0)
  q = m.encode(synth.kitti_like_cloud(77, n_points=8000))
  bad = q.clone()
  bad.view(-1)[::7] = float('nan')
  if precision == 'f16_tc':
    with pytest.raises(OvnError, match='overlap is not finite'):
      m.step_volume(bad, (0.5, 0.0, 0.0))
  else:
    est = m.step_volume(bad, (0.5, 0.0, 0.0))
    assert all(np.isfinite([est['x'], est['y'], est['theta'], est['ess']]))
  assert np.all(np.isfinite(m.particles()))
  est = m.step_volume(q, (0.5, 0.0, 0.0))
  assert est['n_touched'] > 0 and all(np.isfinite([est['x'], est['y'], est['theta'], est['ess']]))
  assert np.all(np.isfinite(m.particles()))
