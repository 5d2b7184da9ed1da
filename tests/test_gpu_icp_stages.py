"""Every stage of every ICP iteration on the GPU (k_icp_pairs through Engine.icp(..., want_stage=True)) against the
float64 stage model oracle/icp_stages.py: the association with zero unexplained pixels, the sums and the pose within
their derived bounds, the decisions, and the result fields, at the known transforms, the street pairs, every status,
the schedule's and the geometry's edges, and an exact known answer.  ``pytest -s`` prints each case's largest
error / bound and its ambiguous-pixel and near-tie counts."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from icp_cases import KITTI_TRANSFORMS, STREET_LEFT, STREET_RIGHT, kitti_pair, pixel_centre_image, rz, street_pair, \
    street_pose
from oracle import gt as G
from oracle import icp
from oracle import icp_stages as I
from overlapnet_b200 import gt, registration
from overlapnet_b200._cabi import ICP_STATUS, IcpParams, lib
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

GEOMETRIES = {'64x900': dict(proj_H=64, proj_W=900), '32x2048': dict(proj_H=32, proj_W=2048, fov_up=15.0, fov_down=-15.0),
              '128x1024': dict(proj_H=128, proj_W=1024, fov_up=2.0, fov_down=-24.9), '16x20': dict(proj_H=16, proj_W=20)}


def _engine(geometry='64x900'):
  return Engine(precision='fp32', max_batch_scans=16, max_batch_pairs=1, **GEOMETRIES[geometry])


def _geometry(eng):
  c = eng.cfg
  return icp.geometry(c.proj_H, c.proj_W, c.fov_up_deg, c.fov_down_deg, c.max_range)


def _params(params):
  p = IcpParams()
  lib().ovn_icp_default_params(C.byref(p))
  prm = {f: getattr(p, f) for f, _ in IcpParams._fields_}
  prm.update(params)
  return prm


def yaw_seed_of(T, Wf=360):
  return registration.seed_pose(gt.yaw_bin(np.eye(4), T, Wf), Wf)


def run(eng, vertex, normal, src, dst, init, want_stage=False, **params):
  out = eng.icp(vertex, normal, src, dst, init, params, want_stage)
  eng.check()
  return {k: v.cpu().numpy() for k, v in out.items()}


def tensors(eng, vertex, normal):
  return (torch.from_numpy(np.ascontiguousarray(vertex, np.float32)).to(eng.device),
          torch.from_numpy(np.ascontiguousarray(normal, np.float32)).to(eng.device))


def check_pairs(name, eng, vertex, normal, src, dst, init, ks=None, **params):
  """Run the pairs, then every iteration k in ``ks`` (all run by default) with iterations = k + 1 and check it from the
  pose after k iterations.  Returns the full run and the worst of each gate; asserts every gate."""
  g = _geometry(eng)
  prm = _params(params)
  V, Nm = vertex.cpu().numpy(), normal.cpu().numpy()
  src, dst = np.asarray(src), np.asarray(dst)
  init = np.asarray(init, np.float64).reshape(-1, 4, 4)
  full = run(eng, vertex, normal, src, dst, init, **params)
  ks = range(int(full['iterations'].max())) if ks is None else ks
  runs = {0: dict(pose=init)}

  def get(k):
    if k not in runs:
      runs[k] = run(eng, vertex, normal, src, dst, init, True, **dict(params, iterations=k))
    return runs[k]

  worst = dict(unexplained=0, ambiguous=0, sums=0.0, pose=0.0, decision=0, tie=0, fields=0, checked=0)
  for k in ks:
    before, step = get(k), get(k + 1)
    for i in range(src.size):
      if k >= full['iterations'][i]:
        continue
      stage = {key: step[key][i] for key in ('assoc', 'system', 'pose', 'status', 'iterations', 'inliers', 'rms',
                                             'valid')}
      rep = I.check_iteration(before['pose'][i], k, prm, g, V[src[i]], Nm[src[i]], V[dst[i]], Nm[dst[i]], stage)
      worst['checked'] += 1
      for key in ('unexplained', 'ambiguous', 'decision', 'tie', 'fields'):
        worst[key] += rep[key]
      worst['sums'] = max(worst['sums'], rep['sums'])
      worst['pose'] = max(worst['pose'], rep['pose'])
  print('%s: %d iterations checked; sums <= %.3g, pose <= %.3g of their bounds; %d unexplained and %d ambiguous '
        'pixels; %d decisions off the model, %d near ties; %d result fields off; statuses %s'
        % (name, worst['checked'], worst['sums'], worst['pose'], worst['unexplained'], worst['ambiguous'],
           worst['decision'], worst['tie'], worst['fields'], sorted(set(full['status'].tolist()))))
  assert worst['checked'] > 0
  assert worst['unexplained'] == 0 and worst['decision'] == 0 and worst['fields'] == 0
  assert worst['sums'] <= 1 and worst['pose'] <= 1
  return full, worst


def cases(geometry):
  if geometry == '64x900':
    return [kitti_pair(y, t) for y, t in KITTI_TRANSFORMS] + [street_pair(k) for k in range(len(STREET_RIGHT))]
  return [street_pair(0), street_pair(3), kitti_pair(30.0, (1.5, -1.0, 0.1)), kitti_pair(-30.0, (-1.2, 1.0, 0.0))]


def _cloud_pairs(eng, cs, init=None):
  vertex, normal = registration.images(eng, [c for L, R, _ in cs for c in (L, R)], list(range(2 * len(cs))))
  n = len(cs)
  init = np.stack([yaw_seed_of(T) for _, _, T in cs]) if init is None else init
  return vertex, normal, np.arange(n) * 2 + 1, np.arange(n) * 2, init


# ---- the known transforms and the street pairs, every iteration ----------------------------------------------------
@pytest.mark.parametrize('geometry', ['64x900', '32x2048', '128x1024'])
def test_every_iteration_of_the_registration_cases(geometry):
  eng = _engine(geometry)
  vertex, normal, src, dst, init = _cloud_pairs(eng, cases(geometry))
  full, worst = check_pairs(geometry, eng, vertex, normal, src, dst, init)
  assert np.count_nonzero(np.isin(full['status'], [ICP_STATUS['converged'], ICP_STATUS['max_iterations']])) >= 2
  assert worst['checked'] >= 20
  eng.close()


# ---- every status on the device ------------------------------------------------------------------------------------
def test_statuses_on_the_device():
  from overlapnet_b200.synth import street_scene_cloud
  eng = _engine()
  g = _geometry(eng)
  ground = [street_scene_cloud(street_pose(*STREET_LEFT), 7, ground_only=True),
            street_scene_cloud(street_pose(*STREET_RIGHT[0]), 7, ground_only=True)]
  L, R, T = street_pair(0)
  cv, cn = registration.images(eng, ground + [L, R], [0, 1, 2, 3])
  v5, n5 = pixel_centre_image(g, nz=False)
  fill_n = np.full_like(n5, -1.0)
  empty_v, empty_n = np.full_like(v5, -1.0), np.full_like(n5, -1.0)
  # scans: 0, 1 ground only; 2 LEFT, 3 RIGHT; 4 rank-5 planes; 5 empty; 6 the rank-5 vertices with fill normals
  V = np.concatenate([cv.cpu().numpy(), np.stack([v5, empty_v, v5])])
  Nm = np.concatenate([cn.cpu().numpy(), np.stack([n5, empty_n, fill_n])])
  vertex, normal = tensors(eng, V, Nm)
  seed = yaw_seed_of(T)
  S = ICP_STATUS
  full, _ = check_pairs('degenerate', eng, vertex, normal, [1, 4], [0, 4], [np.eye(4), np.eye(4)])
  assert full['status'].tolist() == [S['degenerate']] * 2 and full['iterations'].tolist() == [1, 1]
  full, _ = check_pairs('too few inliers', eng, vertex, normal, [3, 6], [5, 4], [seed, np.eye(4)])
  assert full['status'].tolist() == [S['too_few_inliers']] * 2 and full['inliers'].tolist() == [0, 0]
  assert full['valid'][0] > 0 and full['valid'][1] == 0
  full, _ = check_pairs('min_inliers above the count', eng, vertex, normal, [3], [2], [seed], min_inliers=10 ** 6)
  assert full['status'][0] == S['too_few_inliers'] and 0 < full['inliers'][0] < 10 ** 6
  # min_inliers = 0 with no inliers: H = 0, and the pivot test 0 > 1e-12 * 0 fails, so the pair is DEGENERATE
  full, _ = check_pairs('min_inliers 0, no inliers', eng, vertex, normal, [3, 6], [5, 4], [seed, np.eye(4)],
                        min_inliers=0)
  assert full['status'].tolist() == [S['degenerate']] * 2 and full['inliers'].tolist() == [0, 0]
  assert np.array_equal(full['pose'], np.stack([seed, np.eye(4)]))             # a degenerate pair keeps its pose
  eng.close()


# ---- the exact known answer ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('geometry', list(GEOMETRIES))
def test_pixel_centre_image_converges_at_once_to_the_identity(geometry):
  eng = _engine(geometry)
  g = _geometry(eng)
  v, n = pixel_centre_image(g)
  c = G.bin_candidates(*(v[..., k].reshape(-1).astype(np.float64) for k in range(3)), g)
  assert not np.any(c['amb_x'] | c['amb_y'])
  assert np.array_equal(c['by'] * g['W'] + c['bx'], np.arange(g['H'] * g['W']))     # each vertex bins to its pixel
  vertex, normal = tensors(eng, v[None], n[None])
  full, _ = check_pairs('known answer ' + geometry, eng, vertex, normal, [0], [0], [np.eye(4)], d_start=0.3,
                        d_end=0.3)
  step = run(eng, vertex, normal, [0], [0], [np.eye(4)], True, d_start=0.3, d_end=0.3)
  assert full['status'][0] == ICP_STATUS['converged'] and full['iterations'][0] == 1
  assert np.array_equal(full['pose'][0].view(np.uint64), np.eye(4).view(np.uint64))
  assert np.array_equal(step['assoc'][0].reshape(-1), np.arange(g['H'] * g['W']))
  assert np.all(step['system'][0][21:27] == 0) and step['system'][0][28] == 0 and full['rms'][0] == 0
  eng.close()


# ---- the schedule's edges ----------------------------------------------------------------------------------------
def test_schedule_edges():
  eng = _engine()
  vertex, normal, src, dst, init = _cloud_pairs(eng, [street_pair(1), kitti_pair(30.0, (1.5, -1.0, 0.1))])
  S = ICP_STATUS
  full, _ = check_pairs('gamma 1', eng, vertex, normal, src, dst, init, ks=[0, 1, 28, 29], gamma=1.0)
  assert np.all(full['status'] == S['max_iterations']) and np.all(full['iterations'] == 30)
  full, _ = check_pairs('eps 0', eng, vertex, normal, src, dst, init, ks=[0, 20, 29], eps_rot=0.0, eps_trans=0.0)
  assert np.all(full['status'] == S['max_iterations'])
  full, _ = check_pairs('1 iteration', eng, vertex, normal, src, dst, init, iterations=1)
  assert np.all(full['iterations'] == 1)
  full, _ = check_pairs('200 iterations', eng, vertex, normal, src, dst, init, ks=[0, 1, 100, 198, 199],
                        iterations=200, eps_rot=0.0, eps_trans=0.0)
  assert np.all(full['iterations'] == 200) and np.all(full['status'] == S['max_iterations'])
  loose, _ = check_pairs('cos_normal 0', eng, vertex, normal, src, dst, init, ks=[0, 1, 2], cos_normal=0.0)
  tight, _ = check_pairs('cos_normal 1', eng, vertex, normal, src, dst, init, ks=[0], cos_normal=1.0,
                         min_inliers=0)
  base = run(eng, vertex, normal, src, dst, init, True, iterations=1)
  one = run(eng, vertex, normal, src, dst, init, True, iterations=1, cos_normal=1.0, min_inliers=0)
  zero = run(eng, vertex, normal, src, dst, init, True, iterations=1, cos_normal=0.0)
  assert np.all(one['inliers'] <= base['inliers']) and np.all(base['inliers'] <= zero['inliers'])
  eng.close()


# ---- the geometry's edges ----------------------------------------------------------------------------------------
def test_geometry_edges():
  eng = _engine()
  L, R, T = kitti_pair(179.0, (1.0, 1.0, 0.0))
  # the half turn from a seed of exactly 180 degrees: associations cross the azimuth seam
  vertex, normal, src, dst, _ = _cloud_pairs(eng, [(L, R, T), (L, R, T)])
  init = np.stack([rz(math.pi), rz(0.0, (40.0, 0.0, 0.0))])                # and one that moves most points past 50 m
  full, worst = check_pairs('seam and max_range', eng, vertex, normal, src, dst, init)
  step = run(eng, vertex, normal, src[:1], dst[:1], init[:1], True, iterations=1)
  q = step['assoc'][0]
  W = eng.cfg.proj_W
  cols_dst = q[q >= 0] % W
  assert np.any(cols_dst <= 1) and np.any(cols_dst >= W - 2)          # targets on both sides of the seam
  first = run(eng, vertex, normal, src[1:], dst[1:], init[1:], True, iterations=1)
  assert first['inliers'][0] < 0.5 * first['valid'][0]
  eng.close()


def test_image_smaller_than_the_cta():
  eng = _engine('16x20')
  vertex, normal, src, dst, init = _cloud_pairs(eng, [street_pair(0), street_pair(1)])
  assert eng.cfg.proj_H * eng.cfg.proj_W < I.THREADS
  check_pairs('16x20', eng, vertex, normal, src, dst, init, min_inliers=10)
  eng.close()


# ---- a batch of every status --------------------------------------------------------------------------------------
def test_a_batch_of_every_status_has_each_pairs_bits_alone():
  from overlapnet_b200.synth import street_scene_cloud
  eng = _engine()
  g = _geometry(eng)
  L, R, T = street_pair(0)
  ground = [street_scene_cloud(street_pose(*STREET_LEFT), 7, ground_only=True),
            street_scene_cloud(street_pose(*STREET_RIGHT[0]), 7, ground_only=True)]
  cv, cn = registration.images(eng, [L, R] + ground, [0, 1, 2, 3])
  vk, nk = pixel_centre_image(g)
  V = np.concatenate([cv.cpu().numpy(), np.stack([vk, np.full_like(vk, -1.0)])])
  Nm = np.concatenate([cn.cpu().numpy(), np.stack([nk, np.full_like(nk, -1.0)])])
  vertex, normal = tensors(eng, V, Nm)
  # pairs: converged (the known answer at d_end), max iterations (eps 0 is a call parameter, so the street pair with
  # 3 iterations instead), degenerate (ground only), too few inliers (empty target)
  src, dst = [4, 1, 3, 1], [4, 0, 2, 5]
  init = np.stack([np.eye(4), yaw_seed_of(T), np.eye(4), yaw_seed_of(T)])
  prm = dict(d_start=0.3, d_end=0.3, iterations=3)
  batch = run(eng, vertex, normal, src, dst, init, True, **prm)
  S = ICP_STATUS
  assert batch['status'].tolist() == [S['converged'], S['max_iterations'], S['degenerate'], S['too_few_inliers']]
  for i in range(4):
    alone = run(eng, vertex, normal, src[i:i + 1], dst[i:i + 1], init[i:i + 1], True, **prm)
    for key, value in alone.items():
      assert np.array_equal(np.ascontiguousarray(value[0]).view(np.uint8),
                            np.ascontiguousarray(batch[key][i]).view(np.uint8)), (i, key)
  check_pairs('mixed batch', eng, vertex, normal, src, dst, init, **prm)
  eng.close()
