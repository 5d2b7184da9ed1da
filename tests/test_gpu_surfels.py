"""Surfel renders on the GPU (ovn_surfels_batch, ovn_render_surfels_batch, ovn_render_surfels_preprocess_batch):
every bank and image against tests/surfel_oracle.py bit for bit, the refusals, the point render left as it was, and
the virtual map under the Monte Carlo localization filter."""
import ctypes as C
import functools
import math

import numpy as np
import pytest
import torch

import surfel_oracle as so
from conftest import GOLDEN_CASES, load_golden
from oracle import projection as oproj
from overlapnet_b200 import mcl, synth, virtual_map
from overlapnet_b200._cabi import OvnError, SurfelParams, lib
from test_gpu_render import MODEL, _bits, _engine, _infer, _street, random_entries
from test_virtual_map import poses4

pytestmark = pytest.mark.gpu

STUDY_POSES = [(42.0, 0.0), (42.0, 2.0), (41.0, -3.0), (40.0, 4.5)]


def _pose(x, y, th, z=1.73):
  T = np.eye(4)
  T[:2, :2] = [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]
  T[:3, 3] = (x, y, z)
  return T


def _rays(H, W, fu, fd):
  return virtual_map.pixel_rays(H, W, float(np.float32(fu)), float(np.float32(fd)))


def check_render(eng, banks, dev_banks, eo, ec, ep, H=64, W=900, fu=3.0, fd=-25.0, max_splat=8):
  """The device's images, normals and packed input against the oracle, bit for bit."""
  prm = {'max_splat': max_splat}
  got = eng.render_surfels(dev_banks, eo, ec, ep, prm)
  x = eng.render_surfels_preprocess(dev_banks, eo, ec, ep, prm)
  nrm = eng.normals(got['range'], got['vertex'])
  rays = _rays(H, W, fu, fd)
  for v in range(len(eo) - 1):
    rng, vert, inten, winner, normal = so.render(banks, ec[eo[v]:eo[v + 1]], ep[eo[v]:eo[v + 1]], rays, H, W, fu, fd,
                                                 max_splat=max_splat)
    assert np.array_equal(_bits(got['range'])[v], rng.view(np.uint32)), v
    assert np.array_equal(_bits(got['vertex'])[v], vert.view(np.uint32)), v
    assert np.array_equal(_bits(got['intensity'])[v], inten.view(np.uint32)), v
    assert np.array_equal(_bits(got['winner'])[v], winner), v
    assert np.array_equal(_bits(nrm)[v], normal.view(np.uint32)), v
    assert np.array_equal(_bits(x)[v], oproj.pack_input(rng, normal).view(np.uint32)), v
  return got


@pytest.mark.parametrize('name', GOLDEN_CASES)
def test_surfel_banks_equal_the_oracle(name):
  pts = load_golden(name)['points']
  eng = _engine()
  got = eng.surfels(eng.upload_clouds([pts, pts[:5000]]))
  assert np.array_equal(_bits(got)[0], so.surfels(pts).view(np.uint32))
  assert np.array_equal(_bits(got)[1], so.surfels(pts[:5000]).view(np.uint32))
  k = eng.surfels(eng.upload_clouds([pts]), {'kappa': 1.41, 'c_min': 0.3})
  assert np.array_equal(_bits(k)[0], so.surfels(pts, kappa=1.41, c_min=0.3).view(np.uint32))
  eng.close()


@functools.lru_cache(maxsize=None)
def _study():
  kp = np.stack([_pose(x, 0.0, 0.02 * x) for x in range(0, 81, 4)])
  clouds = [synth.street_scene_cloud(T, seed=5) for T in kp]
  return kp, clouds, [so.surfels(c) for c in clouds]


@pytest.mark.parametrize('m', [1, 8])
def test_the_study_poses_equal_the_oracle(m):
  kp, clouds, banks = _study()
  eng = _engine()
  dev = eng.surfels(eng.upload_clouds(clouds))
  assert np.array_equal(_bits(dev), np.stack(banks).view(np.uint32))
  eo, ec, ep = virtual_map.entries(np.stack([_pose(x, y, 0.0) for x, y in STUDY_POSES]), kp, m, 50.0)
  check_render(eng, banks, dev, eo, ec, ep)
  eng.close()


def test_ragged_images_with_an_empty_one_equal_the_oracle():
  clouds = [synth.kitti_like_cloud(60 + s, n_points=20000) for s in range(3)]
  eng = _engine()
  dev = eng.surfels(eng.upload_clouds(clouds))
  banks = [so.surfels(c) for c in clouds]
  eo, ec, ep = random_entries(11, 8, len(clouds))
  assert eo[2] == eo[1] and len(set(np.diff(eo))) > 1
  got = check_render(eng, banks, dev, eo, ec, ep)
  assert (_bits(got['winner'])[1] == -1).all() and (_bits(got['winner']) >= 0).any()
  eng.close()


def _disk_bank(H, W, centres, normals, radii, slots):
  bank = np.zeros((H * W, 8), np.float32)
  for c, n, r, s in zip(centres, normals, radii, slots):
    bank[s] = (*c, r, *n, 0.25)
  return bank.reshape(H, W, 8)


def test_a_footprint_across_the_azimuth_seam_and_near_disks_cut_at_the_window():
  """A disk behind the sensor straddles columns 0 and W - 1; disks 1 m away, wider than the window, are cut at
  max_splat rows and columns; an identity entry and a rotated one."""
  H, W = 64, 900
  seam = ((-6.0, 0.0, -0.5), (1.0, 0.0, 0.0), 0.4, 7)
  near = ((1.0, 0.3, -0.2), (-1.0, 0.0, 0.0), 0.6, 900 * 20 + 3)
  up = ((0.4, -0.9, 0.05), (0.0, 1.0, 0.0), 0.9, 64 * 900 - 1)
  bank = _disk_bank(H, W, *zip(seam, near, up))
  eng = _engine()
  dev = torch.as_tensor(bank[None]).cuda().contiguous()
  R = _pose(0.1, -0.05, 0.3, 0.0)
  eo, ec, ep = np.array([0, 1, 2], np.int64), np.zeros(2, np.int32), np.stack([np.eye(4), R])
  for S in (0, 2, 8, 32):
    got = check_render(eng, [bank], dev, eo, ec, ep, max_splat=S)
    ok = _bits(got['winner'])[0] >= 0
    if S >= 2:
      assert ok[:, 0].any() and ok[:, W - 1].any()                # the seam disk reaches both edge columns
  full = so.render([bank], [0], [np.eye(4)], _rays(H, W, 3.0, -25.0), max_splat=32, full_window=True)
  assert np.array_equal(_bits(eng.render_surfels(dev, eo[:2], ec[:1], ep[:1], {'max_splat': 32})['range'])[0],
                        full[0].view(np.uint32))
  eng.close()


def test_a_32x1024_handle_equals_the_oracle():
  H, W, fu, fd = 32, 1024, 15.0, -15.0
  clouds = [synth.kitti_like_cloud(70 + s, n_points=15000) for s in range(3)]
  eng = _engine(H, W, fu, fd)
  dev = eng.surfels(eng.upload_clouds(clouds))
  banks = [so.surfels(c, H, W, fu, fd) for c in clouds]
  assert np.array_equal(_bits(dev), np.stack(banks).view(np.uint32))
  eo, ec, ep = random_entries(13, 5, len(clouds))
  check_render(eng, banks, dev, eo, ec, ep, H, W, fu, fd)
  eng.close()


# ---- refusals ---------------------------------------------------------------------------------------------------
def test_refusals_and_the_point_render_is_unchanged():
  clouds = [synth.kitti_like_cloud(80 + s, n_points=20000) for s in range(3)]
  eng = _engine()
  batch = eng.upload_clouds(clouds)
  eo, ec, ep = random_entries(9, 3, len(clouds))
  before = {k: _bits(v) for k, v in eng.render(batch, eo, ec, ep).items()}
  xb = _bits(eng.render_preprocess(batch, eo, ec, ep))
  dev = eng.surfels(batch)
  want = _bits(eng.render_surfels(dev, eo, ec, ep)['range'])
  rays = eng.pixel_rays()
  out = torch.full((9, 64, 900), 7.0, device='cuda')
  hp = lambda a: a.ctypes.data_as(C.c_void_p)
  L = lib()

  def raw(eo_=eo, ec_=ec, ep_=ep, prm=None, n_clouds=3, rays_=rays, n_virtual=None):
    p = eng.surfel_params()
    for k, v in (prm or {}).items():
      setattr(p, k, v)
    e, c, q = (np.ascontiguousarray(eo_, np.int64), np.ascontiguousarray(ec_, np.int32),
               np.ascontiguousarray(ep_, np.float64).reshape(-1, 16))
    nv = e.size - 1 if n_virtual is None else n_virtual
    return L.ovn_render_surfels_batch(eng._h, C.c_void_p(dev.data_ptr()), n_clouds,
                                      C.c_void_p(rays_.data_ptr()) if rays_ is not None else None, nv, hp(e), hp(c),
                                      hp(q), C.byref(p), C.c_float(-1.0), C.c_void_p(out.data_ptr()), None, None, None,
                                      eng._stream())

  def refused(status, **kw):
    st = raw(**kw)
    assert st == status, (kw, st, L.ovn_last_error(eng._h))
    torch.cuda.synchronize()
    assert (out == 7.0).all()

  for prm in ({'kappa': 0.0}, {'kappa': -1.0}, {'kappa': float('nan')}, {'kappa': float('inf')},
              {'c_min': 0.0}, {'c_min': 1.0 + 1e-9}, {'c_min': float('nan')}, {'max_splat': -1}, {'max_splat': 33}):
    refused(-1, prm=prm)
    b = eng.surfel_params()
    for k, v in prm.items():
      setattr(b, k, v)
    assert L.ovn_surfels_batch(eng._h, C.c_void_p(batch.points.data_ptr()), C.c_void_p(batch.offsets.data_ptr()), 3,
                               int(batch.offsets_host[-1]), C.byref(b), C.c_void_p(out.data_ptr()),
                               eng._stream()) == -1
  refused(-1, eo_=np.array([0, 2, 1, eo[-1]]))                       # decreasing entry offsets
  refused(-1, eo_=eo + 1, ec_=np.concatenate([[0], ec]), ep_=np.concatenate([[np.eye(4)], ep]))
  for c in (-1, 3):
    e = ec.copy()
    e[-1] = c
    refused(-1, ec_=e)
  p = ep.copy()
  p[1, 0, 3] = float('nan')
  refused(-1, ep_=p)
  p = ep.copy()
  p.reshape(-1, 16)[0, 14] = -0.5
  refused(-1, ep_=p)
  k = -(-(1 << 32) // (64 * 900))                                   # an image of 2^32 / (H W) entries
  refused(-1, eo_=np.array([0, k], np.int64), ec_=np.zeros(k, np.int32), ep_=np.tile(np.eye(4), (k, 1, 1)))
  refused(-1, rays_=None)
  refused(-6, eo_=np.arange(10, dtype=np.int64), ec_=np.zeros(9, np.int32), ep_=np.tile(np.eye(4), (9, 1, 1)))
  with pytest.raises(OvnError, match='OVN_ERR_CAPACITY'):
    L2 = eng.surfel_params()
    big = eng.upload_clouds(clouds * 3)
    from overlapnet_b200._cabi import check
    check(eng._h, L.ovn_surfels_batch(eng._h, C.c_void_p(big.points.data_ptr()), C.c_void_p(big.offsets.data_ptr()),
                                      9, int(big.offsets_host[-1]), C.byref(L2), C.c_void_p(out.data_ptr()),
                                      eng._stream()), 'ovn_surfels_batch')
  assert np.array_equal(_bits(eng.render_surfels(dev, eo, ec, ep)['range']), want)   # the handle still renders
  after = {k: _bits(v) for k, v in eng.render(batch, eo, ec, ep).items()}
  for k in before:
    assert np.array_equal(before[k], after[k]), k
  assert np.array_equal(xb, _bits(eng.render_preprocess(batch, eo, ec, ep)))
  eng.close()
  sem = _engine(use={'use_class_probabilities': True})
  sdev = sem.surfels(sem.upload_clouds(clouds))
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG'):
    sem.render_surfels_preprocess(sdev, eo, ec, ep)
  assert np.array_equal(_bits(sem.render_surfels(sdev, eo, ec, ep)['range']), want)
  sem.close()


# ---- the virtual map under the filter ----------------------------------------------------------------------------
def test_surfel_virtual_map_step_equals_surfels_render_leg_bank_and_step_observed():
  """OverlapMCL(virtual_spacing=..., render='surfels') is plumbing: its bank is surfels + render_surfels_preprocess +
  leg of the lattice frames' entries, and its steps are heads_1vsN on that bank + step_observed, bit for bit."""
  infer = _infer()
  eng = infer._engine
  poses, clouds = _street(6)
  spacing, md, m_src, radius = 1.0, 2.0, 3, 30.0
  prm = {'kappa': 1.41, 'max_splat': 6}
  m = mcl.OverlapMCL(infer, clouds, poses, max_distance=md, virtual_spacing=spacing, render_sources=m_src,
                     render_radius=radius, render='surfels', surfel_params=prm)
  assert m.surfel_params == {'kappa': 1.41, 'c_min': 0.5, 'max_splat': 6}
  query = synth.street_scene_cloud(poses4([(7.2, 0.4, 0.3)], 1.73)[0], seed=9, n_azimuth=900)
  odoms = [(0.0, 0.0, 0.0), (1.0, 0.1, 0.05), (1.5, -0.2, 0.1)]
  m.init_global(5000, 3, init_radius=2.0)
  direct = [m.step(query, o) for o in odoms]
  frames = virtual_map.lattice(poses, spacing, md)
  eo, ec, ep = virtual_map.entries(frames, poses, m_src, radius)
  banks = eng.surfels(eng.upload_clouds(clouds), prm)
  x = eng.render_surfels_preprocess(banks, eo, ec, ep, prm)
  bank = torch.cat([eng.leg(x[v0:v0 + eng.max_batch_scans]) for v0 in range(0, len(frames), eng.max_batch_scans)])
  assert np.array_equal(_bits(bank), _bits(m.bank))
  m.init_global(5000, 3, init_radius=2.0)
  composed = []
  for o in odoms:
    q = infer.encode_clouds([query])[0]
    composed.append(m.step_observed(o, lambda ids: eng.heads_1vsN(m.bank, q, cand_idx=ids)[:2]))
  assert direct == composed and any(e['n_touched'] > 0 for e in direct)
  with pytest.raises(ValueError):
    mcl.OverlapMCL(infer, clouds, poses, render='surfels')
