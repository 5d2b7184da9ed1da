"""The Monte Carlo localization stage gates (oracle/mcl_stages.py) on the CPU: a NumPy restatement of every kernel in
its own order passes every gate, and each planted defect exceeds its gate on a stated share of the elements."""
import math

import numpy as np
import pytest

from oracle import mcl as om
from oracle import mcl_stages as M
from overlapnet_b200 import mcl

SEED = 77
ODOM = (1.2, -0.4, 0.15)
SIGMA = (0.3, 0.2, math.radians(3.0))
S_O, S_PSI = 0.2, math.radians(15)


def holey_map(K=40):
  rng = np.random.default_rng(5)
  kf = np.stack([rng.uniform(0, 60, K), rng.uniform(0, 40, K), rng.uniform(-np.pi, np.pi, K)], 1)
  idx = mcl.MapIndex(kf[:, :2], 0.5, 4.0)
  raster = idx.raster.copy()
  raster[10:30, 20:60] = -1
  return kf, raster, (idx.x0, idx.y0, idx.cell)


def run(n, mutant=None, rho=1.0, width=360):
  """One step of the restated filter: init, predict, update and resampling, with ``mutant`` planted."""
  kf, raster, geo = holey_map()
  p = M.restate_init_global(n, SEED, kf, 6.0, mutant)
  mo = np.stack(M.restate_motion(p[0], p[1], p[2], SEED, 1, ODOM, SIGMA, mutant))
  k = om.lookup(mo[0], mo[1], raster, *geo)
  ref_touched, _ = M.restate_compact(k, kf.shape[0])
  touched, slot = M.restate_compact(k, kf.shape[0], mutant)
  rng = np.random.default_rng(n)
  ov = rng.random(ref_touched.size).astype(np.float32)
  yaw = rng.integers(-180, 540, ref_touched.size).astype(np.int32)
  ll = M.restate_loglik(k, mo[2], kf[:, 2], slot, ov, yaw, width, S_O, S_PSI, mutant)
  up = M.restate_update(p[3], ll, mo[0], mo[1], mo[2], rho, SEED, 1, mutant)
  cdf = M.restate_prefix(up['w'], mutant)
  anc = M.restate_ancestors(cdf, up['u0'], mutant)
  return dict(kf=kf, p=p, mo=mo, k=k, touched=touched, ov=ov, yaw=yaw, ll=ll, up=up, cdf=cdf, anc=anc, n=n,
              width=width, rho=rho)


def gates(r):
  """Every gate of one restated step: the largest ratio of each bounded stage, the mismatches of the exact ones."""
  n, up = r['n'], r['up']
  out = {'init': M.check_init_global(n, SEED, r['kf'], 6.0, r['p']).max(),
         'motion': M.check_motion(r['p'][0], r['p'][1], r['p'][2], SEED, 1, ODOM, SIGMA, r['mo']).max(),
         'touched': M.check_touched(r['k'], r['kf'].shape[0], r['touched'], r['touched'].size),
         'loglik': M.check_loglik(r['k'], r['mo'][2], r['kf'][:, 2], M.restate_compact(r['k'], r['kf'].shape[0])[0],
                                  r['ov'], r['yaw'], r['width'], S_O, S_PSI, r['ll']).max()}
  scal = [up[key] for key in ('m', 'S', 'ess', 'x', 'y', 'theta', 'resampled', 'u0')]
  rep = M.check_update(r['p'][3], r['ll'], r['mo'][0], r['mo'][1], r['mo'][2], r['rho'] * n, scal, up['w'], up['lw'],
                       SEED, 1)
  out.update({key: float(np.max(rep[key])) for key in ('S', 'weights', 'lw', 'ess', 'x', 'y', 'theta')})
  out['exact'] = rep['exact']
  out['prefix'] = M.check_prefix(up['w'], r['cdf'])
  out['ancestors'] = M.check_ancestors(r['cdf'], up['u0'], r['anc'])
  return out, rep


def _passes(g):
  return all(g[key] == 0 for key in ('touched', 'exact', 'prefix', 'ancestors')) and all(
      g[key] <= 1 for key in ('init', 'motion', 'loglik', 'S', 'weights', 'lw', 'ess', 'x', 'y', 'theta'))


@pytest.fixture(scope='module')
def saturated():
  return run(262144)                                     # the reduction grid saturates at 1024 blocks


# ---- the restatement passes ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [1, 257, 2049])
@pytest.mark.parametrize('width', [360, 225, 405])
def test_restatement_passes_every_gate(n, width):
  g, _ = gates(run(n, width=width))
  print(n, width, g)
  assert _passes(g), g


def test_restatement_passes_at_the_saturated_grid(saturated):
  g, _ = gates(saturated)
  print(g)
  assert _passes(g), g
  assert g['S'] > 0 and g['weights'] > 0.05                # the restatement does round, and the bounds are tight


def test_kernel_sum_order():
  # N = 513 runs 3 blocks; element 512 is thread 0 of block 2, the only term the defect drops
  t = np.zeros(513)
  t[512] = 1.0
  assert M.kernel_sum(t)[0] == 1.0 and M.kernel_sum(t, 'drop_last')[0] == 0.0
  assert M.red_blocks(262144) == 1024 and M.red_blocks(262145) == 1024 and M.red_blocks(1) == 1


def test_wrap_pi_and_the_theta_gate_at_pi():
  assert M.wrap_pi(np.array([om.PI, -om.PI])).tolist() == [om.PI, om.PI]
  got = M.restate_init_pose(5, 1, (0.0, 0.0, math.pi), (1.0, 1.0, 0.0))
  assert np.all(got[2] == om.PI) and M.check_init_pose(5, 1, (0.0, 0.0, math.pi), (1.0, 1.0, 0.0), got).max() <= 1


# ---- planted defects exceed their gates ----------------------------------------------------------------------------
def share(bad, total):
  print('exceeds its gate on %d of %d (%.3g %%)' % (bad, total, 100.0 * bad / total))
  assert bad > 0


@pytest.mark.parametrize('mutant', ['drop_last', 'final_256'])
def test_reduction_defects_exceed_the_S_gate(saturated, mutant):
  r = run(262144, mutant)
  scal = [r['up'][key] for key in ('m', 'S', 'ess', 'x', 'y', 'theta', 'resampled', 'u0')]
  rep = M.check_update(saturated['p'][3], saturated['ll'], *saturated['mo'], 262144.0, scal, r['up']['w'])
  print(mutant, 'S error / bound %.3g' % rep['S'])
  share(int(rep['S'] > 1), 1)                               # the one scalar; the weights then follow the GPU's S


@pytest.mark.parametrize('mutant', ['scan_shift', 'offsets_inclusive'])
def test_prefix_defects_exceed_the_gate(saturated, mutant):
  cdf = M.restate_prefix(saturated['up']['w'], mutant)
  share(M.check_prefix(saturated['up']['w'], cdf), cdf.size)


def test_compact_warp_prefix_le_exceeds_the_gate():
  k = np.arange(3000) % 2500                                # 2500 keyframes, every one touched
  touched, _ = M.restate_compact(k, 2500, 'warp_le')
  share(M.check_touched(k, 2500, np.concatenate([touched, [-1]]), 2500), 2500)


@pytest.mark.parametrize('mutant', ['slot_plus_one', 'bin_trunc'])
def test_loglik_defects_exceed_the_gate(saturated, mutant):
  r = saturated
  _, slot = M.restate_compact(r['k'], r['kf'].shape[0], mutant)
  ll = M.restate_loglik(r['k'], r['mo'][2], r['kf'][:, 2], slot, r['ov'], r['yaw'], 360, S_O, S_PSI, mutant)
  ratio = M.check_loglik(r['k'], r['mo'][2], r['kf'][:, 2], r['touched'], r['ov'], r['yaw'], 360, S_O, S_PSI, ll)
  share(int(np.count_nonzero(ratio > 1)), ratio.size)


def test_wrap_pi_minus_pi_exceeds_the_gate():
  pose, sigma = (3.0, 4.0, math.pi), (1.0, 1.0, 0.0)
  got = M.restate_init_pose(2049, 3, pose, sigma, 'wrap_minus_pi')
  ratio = M.check_init_pose(2049, 3, pose, sigma, got)[2]
  share(int(np.count_nonzero(ratio > 1)), ratio.size)


@pytest.mark.parametrize('mutant', ['motion_new_theta', 'box_muller_swapped'])
def test_motion_defects_exceed_the_gate(saturated, mutant):
  p = saturated['p']
  got = np.stack(M.restate_motion(p[0], p[1], p[2], SEED, 1, ODOM, SIGMA, mutant))
  ratio = M.check_motion(p[0], p[1], p[2], SEED, 1, ODOM, SIGMA, got)
  share(int(np.count_nonzero((ratio > 1).any(0))), p.shape[1])
  if mutant == 'box_muller_swapped':
    got = M.restate_init_pose(2049, 3, (3.0, 4.0, 0.5), (1.0, 1.0, 0.2), mutant)
    share(int(np.count_nonzero((M.check_init_pose(2049, 3, (3.0, 4.0, 0.5), (1.0, 1.0, 0.2), got) > 1).any(0))), 2049)


def test_resample_ge_exceeds_the_gate():
  """u0 = 1/2 (the value u53 gives k = 0) and dyadic weights put thresholds exactly on steps of the prefix."""
  w = np.tile([0.125, 0.375, 0.25, 0.25], 512) / 512
  cdf = M.restate_prefix(w)
  anc = M.restate_ancestors(cdf, 0.5, 'resample_ge')
  share(M.check_ancestors(cdf, 0.5, anc), w.size)


@pytest.mark.parametrize('mutant', ['estimate_unnormalized', 'normalize_no_m'])
def test_update_defects_exceed_their_gates(saturated, mutant):
  r = saturated
  up = M.restate_update(r['p'][3], r['ll'], *r['mo'], 1.0, SEED, 1, mutant)
  scal = [up[key] for key in ('m', 'S', 'ess', 'x', 'y', 'theta', 'resampled', 'u0')]
  rep = M.check_update(r['p'][3], r['ll'], *r['mo'], 262144.0, scal, up['w'], up['lw'])
  print(mutant, {key: rep[key] for key in ('S', 'ess', 'x', 'y', 'theta')})
  if mutant == 'estimate_unnormalized':
    assert rep['ess'] > 1
  else:
    share(int(np.count_nonzero(rep['weights'] > 1)), 262144)
