"""GPU parity of the ground-truth overlap / yaw generator (csrc/gt_overlap.cu through the C ABI)
against the golden vectors produced by the reference's ``com_overlap_yaw`` and against the oracle.

Tolerance: yaw bins and frame indices exact.  The range images are float64 arithmetic followed by a
float32 store.  The pose products (mat4_apply: separately rounded, left to right) and every step of the
bin but the device's atan2 / asin are restated bit for bit, so every pixel of a device image is
explained by oracle/gt.explain_range_image: the nearest certain point, or an ambiguous point
(bin_candidates) that may land there.  The overlaps then agree exactly except where an ambiguous
point may change a pixel, and the tolerance of a row is those pixels' share."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from make_golden_gt import gt_test_clouds  # noqa: E402
from oracle import gt as G  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
GEOMETRIES = {'64x900': dict(proj_H=64, proj_W=900), '32x2048': dict(proj_H=32, proj_W=2048, fov_up=15.0, fov_down=-15.0),
              '128x1024': dict(proj_H=128, proj_W=1024, fov_up=2.0, fov_down=-24.9)}


@pytest.fixture(scope='module')
def fixture():
  clouds, poses = gt_test_clouds(GOLDEN)
  return clouds, poses, np.load(os.path.join(GOLDEN, 'gt_overlap_yaw.npz'))


def moved_points(cloud, pose_ref=None, pose_cur_inv=None):
  """float64 (N, 4) points as ovn_gt_range_batch moves them: each 4x4 product a left-to-right sum of separately
  rounded products (se3.cuh mat4_apply)"""
  v = G.homogeneous_points(cloud)
  for M in (pose_ref, pose_cur_inv):
    if M is not None:
      v = ((v[:, 0:1] * M[:, 0] + v[:, 1:2] * M[:, 1]) + v[:, 2:3] * M[:, 2]) + v[:, 3:4] * M[:, 3]
  return v


def explain(got, clouds, poses_ref, cur_inv, g):
  """(unexplained pixels, ambiguous points, uncertain masks) of device images ``got`` [n, H, W]"""
  bad = amb = 0
  masks = []
  for r, c in enumerate(clouds):
    v = moved_points(c, None if poses_ref is None else poses_ref[r], cur_inv)
    b, a, m = G.explain_range_image(v, got[r], g)
    bad, amb = bad + b, amb + a
    masks.append(m)
  return bad, amb, masks


def edge_cloud(g, n=4000, seed=0):
  """float32 points on yaw and pitch bin edges, and on the azimuth seam (y = +-0, x < 0), at 3 .. 40 m"""
  rng = np.random.default_rng(seed)
  W, H = g['W'], g['H']
  down = abs(g['fov_down'] / 180.0 * np.pi)
  fov = down + abs(g['fov_up'] / 180.0 * np.pi)
  yaw = np.pi * (2.0 * rng.integers(0, W + 1, n) / W - 1.0)
  yaw[: n // 8] = np.pi * np.where(np.arange(n // 8) % 2, 1.0, -1.0)
  pitch = (1.0 - rng.integers(1, H, n) / H) * fov - down
  pitch[n // 2:] = rng.uniform(-down, fov - down, n - n // 2)
  d = rng.uniform(3.0, 40.0, n)
  pts = np.zeros((n, 4), np.float32)
  pts[:, 0] = d * np.cos(pitch) * np.cos(-yaw)
  pts[:, 1] = d * np.cos(pitch) * np.sin(-yaw)
  pts[:, 2] = d * np.sin(pitch)
  pts[: n // 8, 1] = np.where(np.arange(n // 8) % 3, 0.0, -0.0)
  return pts


def _geometry(eng):
  c = eng.cfg
  return G.geometry(c.proj_H, c.proj_W, c.fov_up_deg, c.fov_down_deg, c.max_range)


def _explain_fixture(eng, clouds, poses, name):
  """Explain every pixel of the fixture's images moved into frame 3 and of their own images; returns the images
  moved into frame 3 and their uncertain masks."""
  g = _geometry(eng)
  cur_inv = np.linalg.inv(poses[3])
  got = eng.gt_range(eng.upload_clouds(clouds), pose_ref=poses, pose_cur_inv=cur_inv).cpu().numpy()
  assert got.dtype == np.float32
  bad, amb, masks = explain(got, clouds, poses, cur_inv, g)
  own = eng.gt_range(eng.upload_clouds(clouds)).cpu().numpy()          # no transform (com_overlap_yaw.py:29-30)
  bad_own, amb_own, _ = explain(own, clouds, None, None, g)
  print('%s: %d + %d unexplained pixels, %d + %d ambiguous points of %d'
        % (name, bad, bad_own, amb, amb_own, 2 * sum(len(x) for x in clouds)))
  assert bad == 0 and bad_own == 0
  return got, masks


def test_gt_range_images_match_oracle(engine_fp32, fixture):
  clouds, poses, _ = fixture
  got, masks = _explain_fixture(engine_fp32, clouds, poses, '64x900')
  cur_inv = np.linalg.inv(poses[3])
  for r, cl in enumerate(clouds):                                    # the oracle's image differs only where an
    want = G.range_image_f64(moved_points(cl, poses[r], cur_inv))    # ambiguous point may change a pixel
    assert not np.any((got[r].view(np.uint32) != want.view(np.uint32)) & ~masks[r])


@pytest.mark.parametrize('geometry', list(GEOMETRIES))
def test_every_pixel_of_the_gt_range_images_is_explained(fixture, geometry):
  from overlapnet_b200.engine import Engine
  clouds, poses, _ = fixture
  eng = Engine(precision='fp32', max_batch_scans=8, max_batch_pairs=1, **GEOMETRIES[geometry])
  g = _geometry(eng)
  if geometry != '64x900':                                           # 64x900: test_gt_range_images_match_oracle
    _explain_fixture(eng, clouds, poses, geometry)
  edges = [edge_cloud(g, seed=s) for s in range(2)]
  got_e = eng.gt_range(eng.upload_clouds(edges)).cpu().numpy()
  bad_e, amb_e, _ = explain(got_e, edges, None, None, g)
  print('%s edge clouds: %d unexplained pixels, %d of %d points ambiguous'
        % (geometry, bad_e, amb_e, sum(len(x) for x in edges)))
  assert bad_e == 0
  assert amb_e > 0                                                   # the edge clouds do reach the ambiguity
  eng.close()


def test_gt_overlap_count_matches_numpy(engine_fp32):
  import torch
  rng = np.random.default_rng(5)
  ref = np.where(rng.random((4, 64, 900)) < 0.2, -1.0, rng.uniform(0, 50, (4, 64, 900))).astype(np.float32)
  cur = np.where(rng.random((64, 900)) < 0.2, -1.0, rng.uniform(0, 50, (64, 900))).astype(np.float32)
  ref[1] = cur                                     # identical image: every valid pixel counts
  got = engine_fp32.gt_overlap_count(torch.from_numpy(ref).cuda(), torch.from_numpy(cur).cuda()).cpu().numpy()
  want = [G.overlap_counts(cur, r) for r in ref] + [int(np.count_nonzero(cur > 0))]
  assert got.tolist() == want
  assert got[1] == got[4]


@pytest.mark.parametrize('frame', [0, 3])
def test_mapping_matches_reference_golden(fixture, frame):
  from overlapnet_b200.gt import overlap_yaw_from_clouds
  clouds, poses, gold = fixture
  rows = overlap_yaw_from_clouds(clouds, poses, frame, scans_per_launch=2)       # exercises the chunking
  want = gold['mapping_frame%d' % frame]
  assert rows.dtype == np.float64 and rows.shape == want.shape
  assert np.array_equal(rows[:, [0, 1, 3]], want[:, [0, 1, 3]])
  assert np.all(np.abs(rows[:, 2] - want[:, 2]) <= overlap_tolerance(clouds, poses, frame))


def overlap_tolerance(clouds, poses, frame):
  """Per row, how far a correct overlap may be from the reference's: c / v with c the pixels of ref > 0 and
  |ref - cur| < 1 and v the current image's valid pixels.  Only pixels an ambiguous point may change can differ
  (explain_range_image's uncertain mask): a count moves by at most the uncertain pixels of both images and v by the
  current image's, so |c'/v' - c/v| <= (A_ref + A_cur + (c/v) A_cur) / v'.  Zero where no point is ambiguous."""
  g = G.geometry(f32=False)
  cur = G.homogeneous_points(clouds[frame])
  cur_img = G.range_image_f64(cur)
  a_cur = np.count_nonzero(G.explain_range_image(cur, cur_img, g)[2])
  v = np.count_nonzero(cur_img > 0)
  inv = np.linalg.inv(poses[frame])
  tol = np.zeros(len(clouds))
  for r, c in enumerate(clouds):
    pts = inv.dot(poses[r].dot(G.homogeneous_points(c).T)).T
    img = G.range_image_f64(pts)
    a_ref = np.count_nonzero(G.explain_range_image(pts, img, g)[2])
    share = G.overlap_counts(cur_img, img) / v
    tol[r] = (a_ref + a_cur + share * a_cur) / max(v - a_cur, 1)
  return tol


def test_com_overlap_yaw_drop_in_reads_bin_files(fixture, tmp_path, capsys):
  from overlapnet_b200 import com_overlap_yaw
  clouds, poses, gold = fixture
  paths = []
  for i, c in enumerate(clouds):
    p = tmp_path / ('%06d.bin' % i)
    np.ascontiguousarray(c, np.float32).tofile(p)
    paths.append(str(p))
  rows = com_overlap_yaw(paths, poses, frame_idx=0)
  assert 'Finish generating ground_truth_mapping!' in capsys.readouterr().out       # the reference prints this
  want = gold['mapping_frame0']
  assert np.array_equal(rows[:, [0, 1, 3]], want[:, [0, 1, 3]])
  assert np.all(np.abs(rows[:, 2] - want[:, 2]) <= overlap_tolerance(clouds, poses, 0))
