"""The virtual map's host side: the lattice and its entries, the filter on a lattice map with a sensor that knows the
true pose (oracle/mcl.py on the CPU), and the command line's virtual-map flags."""
import math

import numpy as np
import pytest

from oracle import mcl as om
from overlapnet_b200 import mcl, virtual_map


def poses4(p, z=0.0):
  """(n, 4, 4) poses of planar (n, 3) x, y, theta at height z."""
  p = np.asarray(p, np.float64).reshape(-1, 3)
  T = np.tile(np.eye(4), (p.shape[0], 1, 1))
  c, s = np.cos(p[:, 2]), np.sin(p[:, 2])
  T[:, 0, 0], T[:, 0, 1], T[:, 1, 0], T[:, 1, 1] = c, -s, s, c
  T[:, 0, 3], T[:, 1, 3], T[:, 2, 3] = p[:, 0], p[:, 1], z
  return T


@pytest.mark.parametrize('seed, g, md', [(0, 1.0, 3.0), (1, 0.7, 2.0), (2, 2.5, 0.0), (3, 1.0, 10.0)])
def test_lattice_keeps_exactly_the_points_within_reach(seed, g, md):
  rs = np.random.default_rng(seed)
  K = 25
  kf = np.stack([rs.uniform(-30, 30, K), rs.uniform(-20, 20, K), rs.uniform(-np.pi, np.pi, K)], 1)
  kp = poses4(kf)
  kp[:, 2, 3] = rs.uniform(1.0, 2.0, K)
  out = virtual_map.lattice(kp, g, md)
  # brute force over the keyframes' bounding box grown by md
  i = np.arange(math.floor((kf[:, 0].min() - md) / g) - 1, math.ceil((kf[:, 0].max() + md) / g) + 2)
  j = np.arange(math.floor((kf[:, 1].min() - md) / g) - 1, math.ceil((kf[:, 1].max() + md) / g) + 2)
  jj, ii = np.meshgrid(j, i, indexing='ij')
  pts = np.stack([ii.reshape(-1) * g, jj.reshape(-1) * g], 1)
  d2 = ((pts[:, None, :] - kf[None, :, :2]) ** 2).sum(-1)
  keep = d2.min(1) <= md * md
  assert np.array_equal(out[:, :2, 3], pts[keep])                # the same points, ordered by j then i
  near = np.argmin(d2[keep], 1)                                   # argmin: the lowest index among equal distances
  assert np.array_equal(out[:, :3, :3], kp[near, :3, :3]) and np.array_equal(out[:, 2, 3], kp[near, 2, 3])
  assert np.array_equal(out[:, 3], np.tile([0.0, 0.0, 0.0, 1.0], (out.shape[0], 1)))


def test_lattice_ties_go_to_the_lowest_keyframe():
  kp = poses4([(1.0, 0.0, 0.5), (-1.0, 0.0, -0.5), (0.0, 1.0, 1.5)])
  out = virtual_map.lattice(kp, 1.0, 0.0 + 1.0)
  at0 = out[(out[:, 0, 3] == 0.0) & (out[:, 1, 3] == 0.0)]
  assert at0.shape[0] == 1 and np.array_equal(at0[0, :3, :3], kp[0, :3, :3])   # three keyframes 1 m away
  with pytest.raises(ValueError):
    virtual_map.lattice(kp, 0.0, 1.0)
  with pytest.raises(ValueError):
    virtual_map.lattice(kp[:0], 1.0, 1.0)


def test_entries_order_radius_and_poses():
  rs = np.random.default_rng(7)
  kf = np.stack([rs.uniform(0, 40, 30), rs.uniform(-5, 5, 30), rs.uniform(-np.pi, np.pi, 30)], 1)
  kf[5, :2] = kf[3, :2]                                           # a tie at equal distance: 3 before 5
  kp = poses4(kf, 1.73)
  vp = poses4(np.stack([rs.uniform(0, 40, 12), rs.uniform(-5, 5, 12), rs.uniform(-np.pi, np.pi, 12)], 1), 1.7)
  vp[0, :2, 3] = kf[3, :2] + 0.1
  vp[11, :2, 3] = (500.0, 500.0)                                  # nothing within the radius
  m, radius = 4, 9.0
  eo, ec, ep = virtual_map.entries(vp, kp, m, radius)
  assert eo.dtype == np.int64 and ec.dtype == np.int32 and ep.shape == (ec.size, 4, 4) and eo[0] == 0
  for v in range(vp.shape[0]):
    d2 = ((kf[:, :2] - vp[v, :2, 3]) ** 2).sum(1)
    order = [k for k in np.lexsort((np.arange(kf.shape[0]), d2)) if d2[k] <= radius * radius][:m]
    assert list(ec[eo[v]:eo[v + 1]]) == order
    for e, k in zip(range(eo[v], eo[v + 1]), order):
      want = np.linalg.inv(vp[v]) @ kp[k]
      assert np.array_equal(ep[e, :3], want[:3]) and np.array_equal(ep[e, 3], [0.0, 0.0, 0.0, 1.0])
  assert eo[1] - eo[0] == m and list(ec[:2]) == [3, 5] and eo[12] == eo[11]


# ---- the filter on a lattice map with a sensor that knows the true pose ------------------------------------------
# oracle/mcl.py's filter at 10^4 particles on om.scenario() with keyframes every 4 m and the queries between them,
# seeds 0..4, 200 steps.  On the keyframe map (MapIndex within 3 m): seeds 0 and 3 never stay within 2 m, and the
# other seeds' mean position errors after step 50 are 0.96 to 1.67 m.  On a 1 m lattice within 3 m of the keyframes
# (18 809 frames, MapIndex within 1 m): every seed within 2 m from step 17 on; after step 50 the largest position
# error was 0.071 m and the largest yaw error 0.17 bins.  The gates below (and test_gpu_render's) sit on those numbers.
LATTICE = dict(spacing=1.0, max_distance=3.0, cell=0.5, sigma_overlap=0.05, sigma_yaw=math.radians(10.0),
               motion_sigma=(0.1, 0.1, math.radians(1.0)))
GATE_CONVERGED_BY = 50
GATE_POSITION_M = 0.25
GATE_YAW_BINS = 1.0


def lattice_scenario():
  """(lattice planar frames, MapIndex of them, true query poses, odometry) of the scenario above."""
  poses = om.scenario()
  kfi, qi = mcl.split_sequence(len(poses), 4)
  kf, truth = poses[kfi], poses[qi]
  frames = mcl.planar(virtual_map.lattice(poses4(kf), LATTICE['spacing'], LATTICE['max_distance']))
  idx = mcl.MapIndex(frames[:, :2], LATTICE['cell'], LATTICE['spacing'])
  return frames, idx, truth, mcl.odometry(truth), kf


def test_cpu_filter_localizes_to_the_lattice_with_a_true_sensor():
  frames, idx, truth, odom, kf = lattice_scenario()
  T = 120
  for name, fr, ix in (('lattice', frames, idx), ('keyframes', kf, mcl.MapIndex(kf[:, :2], 0.5, 3.0))):
    f = om.Filter(fr, ix.raster, ix.x0, ix.y0, ix.cell)
    f.init_global(10000, 2, 1.0)
    pos, yaw = np.zeros(T), np.zeros(T)
    for t in range(T):
      e = f.step(odom[t], LATTICE['motion_sigma'], om.fake_sensor(truth[t], fr), LATTICE['sigma_overlap'],
                 LATTICE['sigma_yaw'])
      pos[t] = math.hypot(e['x'] - truth[t, 0], e['y'] - truth[t, 1])
      yaw[t] = abs(mcl.wrap_pi(e['theta'] - truth[t, 2])) / (2 * math.pi / 360)
    if name == 'lattice':
      assert 0 <= mcl.convergence_step(pos, 2.0) <= GATE_CONVERGED_BY
      assert pos[50:].max() < GATE_POSITION_M and yaw[50:].max() < GATE_YAW_BINS
    else:
      assert pos[50:].mean() > 0.5                                 # 0.96 m: the keyframe spacing limits this map


def test_cli_virtual_map_flags():
  a = mcl.parse_args([])
  assert a.virtual_spacing is None and a.render_sources == 8 and a.render_radius is None
  assert mcl.virtual_args(a) == {}
  a = mcl.parse_args(['--virtual-spacing', '1.5', '--render-sources', '64', '--render-radius', '30'])
  assert (a.virtual_spacing, a.render_sources, a.render_radius) == (1.5, 64, 30.0)
  assert mcl.virtual_args(a) == dict(virtual_spacing=1.5, render_sources=64, render_radius=30.0)
  for bad in (['--virtual-spacing', '0'], ['--virtual-spacing', '-1'], ['--virtual-spacing', 'inf'],
              ['--render-sources', '0'], ['--render-sources', '65'], ['--render-radius', '0'],
              ['--render-radius', 'nan']):
    with pytest.raises(SystemExit):
      mcl.parse_args(bad)
