"""The render's NumPy model (tests/render_oracle.py): pinned to the golden projections through identity entries, the
concatenation order and its ties, and the synthetic study behind the virtual map's default of 8 sources."""
import numpy as np
import pytest

import render_oracle as ro
from conftest import load_golden
from oracle import projection as oproj
from overlapnet_b200 import synth, virtual_map


@pytest.mark.parametrize('name', ['kitti_000000', 'kitti_000001'])
def test_identity_render_equals_the_golden_projection(name):
  """Identity entries of the two KITTI fixtures (neither holds a negative zero coordinate, so M = I moves no point)
  give the golden range, intensity and normal images bit for bit, and winners that are the golden filtered indices
  mapped back to the cloud."""
  g = load_golden(name)
  pts = g['points']
  assert not (np.signbit(pts[:, :3]) & (pts[:, :3] == 0)).any()
  rng, _, inten, winner, normal = ro.render([pts], [0], [np.eye(4)])
  assert np.array_equal(rng.view(np.uint32), g['range'].view(np.uint32))
  assert np.array_equal(inten.view(np.uint32), g['intensity'].view(np.uint32))
  assert np.array_equal(normal.view(np.uint32), g['normal'].view(np.uint32))
  valid = oproj.projection_bins(pts)[0]
  sel = np.flatnonzero(valid)
  assert np.array_equal(winner, np.where(g['idx'] >= 0, sel[np.maximum(g['idx'], 0)], -1))


def test_two_equal_entries_give_the_single_entry_image_with_entry_0_winning():
  pts = synth.kitti_like_cloud(21, n_points=20000)
  a = 0.4
  M = np.eye(4)
  M[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
  M[:3, 3] = (1.5, -0.5, 0.1)
  one = ro.render([pts], [0], [M])
  two = ro.render([pts], [0, 0], [M, M])
  for i in (0, 1, 2, 4):
    assert np.array_equal(one[i].view(np.uint32), two[i].view(np.uint32))
  assert np.array_equal(one[3], two[3]) and two[3].max() < pts.shape[0] and (two[3] >= 0).any()


def _pose(x, y, th, z=1.73):
  T = np.eye(4)
  T[:2, :2] = [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]
  T[:3, 3] = (x, y, z)
  return T


# The study of DESIGN.md section 7: keyframes every 4 m along y = 0 at heading 0.02 x, virtual frames at heading 0.
# Overlaps (M = 1, 2, 4, 8): (42, 0) 0.768 0.902 0.924 0.956; (42, 2) 0.699 0.871 0.912 0.945;
# (41, -3) 0.659 0.801 0.883 0.921; (40, 4.5) 0.593 0.728 0.850 0.904.
STUDY_POSES = [(42.0, 0.0), (42.0, 2.0), (41.0, -3.0), (40.0, 4.5)]


def test_rendering_more_sources_raises_the_overlap_with_the_real_scan():
  kp = np.stack([_pose(x, 0.0, 0.02 * x) for x in range(0, 81, 4)])
  clouds = [synth.street_scene_cloud(T, seed=5) for T in kp]
  for x, y in STUDY_POSES:
    Tv = _pose(x, y, 0.0)
    real = oproj.range_projection(synth.street_scene_cloud(Tv, seed=5))[0]
    ov = {}
    for m in (1, 8):
      _, ec, ep = virtual_map.entries(Tv[None], kp, m, 50.0)
      ov[m] = ro.overlap(ro.render(clouds, ec, ep)[0], real)
    assert ov[8] >= 0.9 and ov[8] > ov[1], ((x, y), ov)
