"""The surfel render's NumPy model (tests/surfel_oracle.py) on the CPU: the pixel rays, single disks against a
brute-force angular test, the max_splat cut, ties, the kernel's window against the full box, the synthetic study
behind the defaults (DESIGN.md section 7, "Surfel renders"), and the parameters, flags and symbols around it."""
import math

import numpy as np
import pytest

import render_oracle as ro
import surfel_oracle as so
from oracle import projection as oproj
from overlapnet_b200 import _cabi, mcl, synth, virtual_map

H, W = 64, 900


@pytest.mark.parametrize('h,w,fu,fd', [(64, 900, 3.0, -25.0), (32, 1024, 15.0, -15.0)])
def test_every_pixel_ray_lands_in_its_own_pixel(h, w, fu, fd):
  u = virtual_map.pixel_rays(h, w, fu, fd)
  assert np.allclose(np.linalg.norm(u, axis=2), 1.0, rtol=0, atol=1e-15)
  pts = np.zeros((h * w, 4), np.float32)
  pts[:, :3] = (10.0 * u.reshape(-1, 3)).astype(np.float32)
  valid, _, py, px = oproj.projection_bins(pts, fu, fd, h, w)
  yy, xx = np.divmod(np.arange(h * w), w)
  assert valid.all() and np.array_equal(py, yy) and np.array_equal(px, xx)


def _facing_disk(q, r, slot=0):
  """A bank holding one disk at q that faces the sensor (n = -q / |q|)."""
  q = np.asarray(q, np.float64)
  bank = np.zeros((H * W, 8), np.float32)
  bank[slot] = (*q, r, *(-q / np.linalg.norm(q)), 0.5)
  return bank.reshape(H, W, 8)


def _angular(bank, rays, slot=0):
  """Brute force for a sensor-facing disk: the ray u is drawn when its angle to q is below atan(r / |q|), except
  where the two agree to 1e-9 rad (undecided).  Returns (drawn, undecided) [H, W] masks."""
  s = bank.reshape(-1, 8)[slot].astype(np.float64)
  q, r = s[:3], s[3]
  qh = q / np.linalg.norm(q)
  ang = np.arccos(np.clip(rays @ qh, -1, 1))
  lim = math.atan(r / np.linalg.norm(q))
  return ang < lim, np.abs(ang - lim) < 1e-9


@pytest.mark.parametrize('q,r', [((8.0, 3.0, -0.6), 0.5), ((-7.0, 0.0, -0.4), 0.6), ((-7.0, -0.01, 0.2), 0.3),
                                 ((3.0, -2.0, -1.0), 0.2)])
def test_a_sensor_facing_disk_matches_the_angular_brute_force(q, r):
  """Disks away from the seam and across it (x < 0, y = 0 and y slightly below), drawn with a window that does not
  cut them."""
  bank = _facing_disk(q, r)
  rays = virtual_map.pixel_rays(H, W, 3.0, -25.0)
  drawn, undecided = _angular(bank, rays)
  got = so.render([bank], [0], [np.eye(4)], rays, max_splat=32)[3] >= 0
  assert drawn.sum() > 4 and not undecided.any()
  assert np.array_equal(got, drawn)
  if q[0] < 0 and abs(q[1]) < 0.1:
    assert got[:, 0].any() and got[:, W - 1].any()


@pytest.mark.parametrize('S', [0, 1, 3, 8])
def test_a_wide_disk_is_cut_exactly_at_the_window(S):
  bank = _facing_disk((2.0, -0.3, -0.4), 0.8)
  rays = virtual_map.pixel_rays(H, W, 3.0, -25.0)
  drawn, undecided = _angular(bank, rays)
  assert not undecided.any()
  pts = np.zeros((1, 4), np.float32)
  pts[0, :3] = bank.reshape(-1, 8)[0, :3]
  _, _, cy, cx = oproj.projection_bins(pts)
  yy, xx = np.mgrid[:H, :W]
  dx = np.abs((xx - cx[0] + W // 2) % W - W // 2)
  box = (np.abs(yy - cy[0]) <= S) & (dx <= S)
  assert (drawn & ~box).any()                                      # the true footprint exceeds the window
  got = so.render([bank], [0], [np.eye(4)], rays, max_splat=S)[3] >= 0
  assert np.array_equal(got, drawn & box)


def test_two_equal_entries_give_the_single_entry_image_with_entry_0_winning():
  bank = so.surfels(synth.kitti_like_cloud(21, n_points=20000))
  rays = virtual_map.pixel_rays(H, W, 3.0, -25.0)
  a = 0.4
  M = np.eye(4)
  M[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
  M[:3, 3] = (1.5, -0.5, 0.1)
  one = so.render([bank], [0], [M], rays)
  two = so.render([bank, bank], [0, 1], [M, M], rays)
  for i in (0, 1, 2, 4):
    assert np.array_equal(one[i].view(np.uint32), two[i].view(np.uint32))
  assert np.array_equal(one[3], two[3]) and two[3].max() < H * W and (two[3] >= 0).any()


def test_the_kernel_window_never_drops_a_drawable_pixel():
  """The window (surfel_window) against the full (2 S + 1)^2 box: a KITTI-like bank seen from a pose that brings
  many surfels close to the sensor, and a pose past the maximum range."""
  bank = so.surfels(synth.kitti_like_cloud(5, n_points=30000))
  sub = bank.copy().reshape(-1, 8)
  sub[np.arange(sub.shape[0]) % 5 != 0] = 0                         # a fifth of the slots keeps the full box fast
  sub = sub.reshape(H, W, 8)
  rays = virtual_map.pixel_rays(H, W, 3.0, -25.0)
  for t in ((0.0, 0.0, 0.0), (4.0, -2.0, 0.5), (45.0, 0.0, 0.0)):
    M = np.eye(4)
    M[:3, 3] = t
    for S in (4, 8):
      win = so.render([sub], [0], [M], rays, max_splat=S)
      full = so.render([sub], [0], [M], rays, max_splat=S, full_window=True)
      for i in range(5):
        assert np.array_equal(win[i].view(np.uint32), full[i].view(np.uint32)), (t, S, i)


def _pose(x, y, th, z=1.73):
  T = np.eye(4)
  T[:2, :2] = [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]
  T[:3, 3] = (x, y, z)
  return T


# The study of DESIGN.md section 7 ("Surfel renders"): keyframes every 4 m along y = 0 at heading 0.02 x, seed 5,
# virtual frames at heading 0; the overlap of the point render and of the surfel render with the real scan.
STUDY_POSES = [(42.0, 0.0), (42.0, 2.0), (41.0, -3.0), (40.0, 4.5)]


def test_surfels_raise_the_overlap_of_the_study_poses():
  kp = np.stack([_pose(x, 0.0, 0.02 * x) for x in range(0, 81, 4)])
  clouds = [synth.street_scene_cloud(T, seed=5) for T in kp]
  banks = {k: [so.surfels(c, kappa=k) for c in clouds] for k in (1.0, 2.0)}
  rays = virtual_map.pixel_rays(H, W, 3.0, -25.0)
  for x, y in STUDY_POSES:
    Tv = _pose(x, y, 0.0)
    real = oproj.range_projection(synth.street_scene_cloud(Tv, seed=5))[0]
    ov = {}
    for m, kappa in ((8, 1.0), (1, 2.0)):
      _, ec, ep = virtual_map.entries(Tv[None], kp, m, 50.0)
      ov['points', m] = ro.overlap(ro.render(clouds, ec, ep)[0], real)
      ov['surfels', m] = ro.overlap(so.render(banks[kappa], ec, ep, rays)[0], real)
    assert ov['surfels', 8] >= max(ov['points', 8], 0.95), ((x, y), ov)
    assert ov['surfels', 1] >= ov['points', 1] + 0.05, ((x, y), ov)


# ---- parameters, flags, symbols ----------------------------------------------------------------------------------
def test_the_cli_flags_parse_and_bad_values_are_refused():
  base = ['demo.yml', '--virtual-spacing', '1']
  a = mcl.parse_args(base)
  assert a.render == 'points' and mcl.virtual_args(a) == dict(virtual_spacing=1.0, render_sources=8,
                                                              render_radius=None)
  a = mcl.parse_args(base + ['--render', 'surfels'])
  assert mcl.virtual_args(a)['render'] == 'surfels' and mcl.virtual_args(a)['surfel_params'] == {}
  a = mcl.parse_args(base + ['--render', 'surfels', '--surfel-kappa', '2', '--max-splat', '5'])
  assert mcl.virtual_args(a)['surfel_params'] == {'kappa': 2.0, 'max_splat': 5}
  assert mcl.parse_args(base + ['--render', 'surfels', '--max-splat', '0']).max_splat == 0
  assert mcl.parse_args(base + ['--render', 'surfels', '--max-splat', '32']).max_splat == 32
  for bad in (['demo.yml', '--render', 'surfels'], base + ['--render', 'mesh'],
              base + ['--surfel-kappa', '2'], base + ['--max-splat', '4'],
              base + ['--render', 'surfels', '--surfel-kappa', '0'],
              base + ['--render', 'surfels', '--surfel-kappa', 'nan'],
              base + ['--render', 'surfels', '--max-splat', '-1'],
              base + ['--render', 'surfels', '--max-splat', '33']):
    with pytest.raises(SystemExit):
      mcl.parse_args(bad)
  assert mcl.virtual_args(mcl.parse_args(['demo.yml'])) == {}


def test_the_surfel_bank_is_counted_in_the_bank_bytes():
  class E:
    Wf, H, W, precision = 360, 64, 900, 'fp32'
  assert virtual_map.bank_bytes(E, 10) == 10 * 360 * 128 * 4
  assert virtual_map.bank_bytes(E, 10, 3) == 10 * 360 * 128 * 4 + 3 * 64 * 900 * 32
  assert 64 * 900 * 32 == 1843200                                   # 1.84 MB per keyframe


def test_the_c_abi_exports_the_surfel_symbols():
  names = ('ovn_surfel_default_params', 'ovn_surfels_batch', 'ovn_render_surfels_batch',
           'ovn_render_surfels_preprocess_batch')
  assert set(names) <= set(_cabi.SYMBOLS)
  L = _cabi.lib()
  for n in names:
    getattr(L, n)
  p = _cabi.SurfelParams()
  L.ovn_surfel_default_params(p)
  assert (p.kappa, p.c_min, p.max_splat) == (1.0, 0.5, 8) == tuple(so.DEFAULTS.values())
