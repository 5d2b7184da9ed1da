"""The render on the GPU (ovn_render_batch / ovn_render_preprocess_batch): every image against tests/render_oracle.py
bit for bit, identity entries against the projection, determinism, the refusals, and the virtual map under the Monte
Carlo localization filter."""
import copy
import ctypes as C
import functools
import json
import math

import numpy as np
import pytest
import torch

import render_oracle as ro
from oracle import mcl as om
from oracle import projection as oproj
from overlapnet_b200 import mcl, synth, virtual_map
from overlapnet_b200._cabi import OvnError, lib
from overlapnet_b200.engine import Engine
from test_virtual_map import GATE_CONVERGED_BY, GATE_POSITION_M, GATE_YAW_BINS, LATTICE, lattice_scenario, poses4

pytestmark = pytest.mark.gpu

MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
         'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
         'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
         'additional_unsymmetric_layer3a': True}
GEOMETRIES = [(64, 900, 3.0, -25.0), (32, 2048, 15.0, -15.0), (128, 1024, 2.0, -24.9)]
MAX_BATCH = 8


def _engine(H=64, W=900, fu=3.0, fd=-25.0, use=None, max_batch_scans=MAX_BATCH):
  return Engine(use=use, model=MODEL, precision='fp32', max_batch_scans=max_batch_scans, max_batch_pairs=1, proj_H=H,
                proj_W=W, fov_up=fu, fov_down=fd)


@functools.lru_cache(maxsize=None)
def _clouds():
  """Seeded clouds: three KITTI-like ones with zero points, an empty one and a one-point one."""
  clouds = [synth.kitti_like_cloud(40 + s, n_points=n, zero_points=z) for s, (n, z) in
            enumerate([(30000, 5), (12000, 0), (20000, 3)])]
  clouds.insert(1, np.zeros((0, 4), np.float32))
  clouds.append(np.array([[2.0, 1.0, -0.2, 0.7]], np.float32))
  return clouds


def _pose(rs, yaw=None):
  a = rs.uniform(-np.pi, np.pi) if yaw is None else yaw
  T = np.eye(4)
  T[:2, :2] = [[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]]
  b = rs.uniform(-0.05, 0.05)                                     # a small roll
  R = np.array([[1, 0, 0], [0, math.cos(b), -math.sin(b)], [0, math.sin(b), math.cos(b)]])
  T[:3, :3] = T[:3, :3] @ R
  T[:3, 3] = rs.uniform(-6, 6, 3) * (1, 1, 0.1)
  return T


def random_entries(seed, n_virtual, n_clouds):
  """Entry tables of n_virtual images with 0..3 entries each (image 1 has none when there are several images),
  random poses, the first at yaw 179 degrees."""
  rs = np.random.default_rng(seed)
  counts = rs.integers(1, 4, n_virtual)
  if n_virtual > 1:
    counts[1] = 0
  eo = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
  ec = rs.integers(0, n_clouds, int(eo[-1])).astype(np.int32)
  ep = np.stack([_pose(rs, math.radians(179.0) if e == 0 else None) for e in range(int(eo[-1]))]) \
      if eo[-1] else np.zeros((0, 4, 4))
  return eo, ec, ep


def oracle_images(clouds, eo, ec, ep, H, W, fu, fd, max_range=50.0):
  out = [ro.render(clouds, ec[eo[v]:eo[v + 1]], ep[eo[v]:eo[v + 1]], H, W, fu, fd, max_range)
         for v in range(eo.size - 1)]
  return [np.stack([o[i] for o in out]) for i in range(5)]


def _bits(t):
  a = t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
  return a.view(np.uint32) if a.dtype == np.float32 else a


@pytest.mark.parametrize('n_virtual', [1, 7, MAX_BATCH])
@pytest.mark.parametrize('H,W,fu,fd', GEOMETRIES)
def test_render_equals_the_oracle(H, W, fu, fd, n_virtual):
  clouds = _clouds()
  eng = _engine(H, W, fu, fd)
  batch = eng.upload_clouds(clouds)
  eo, ec, ep = random_entries(H + W + n_virtual, n_virtual, len(clouds))
  got = eng.render(batch, eo, ec, ep)
  x = eng.render_preprocess(batch, eo, ec, ep)
  nrm = eng.normals(got['range'], got['vertex'])
  rng, vert, inten, winner, normal = oracle_images(clouds, eo, ec, ep, H, W, fu, fd)
  assert np.array_equal(_bits(got['range']), rng.view(np.uint32))
  assert np.array_equal(_bits(got['vertex']), vert.view(np.uint32))
  assert np.array_equal(_bits(got['intensity']), inten.view(np.uint32))
  assert np.array_equal(_bits(got['winner']), winner)
  assert np.array_equal(_bits(nrm), normal.view(np.uint32))
  packed = np.stack([oproj.pack_input(rng[v], normal[v]) for v in range(n_virtual)])
  assert np.array_equal(_bits(x), packed.view(np.uint32))
  if n_virtual > 1:
    assert (_bits(got['winner'])[1] == -1).all() and (_bits(got['range'])[1] == np.float32(-1).view(np.uint32)).all()
  assert (_bits(got['winner']) >= 0).any()
  eng.close()


@pytest.mark.parametrize('H,W,fu,fd', GEOMETRIES)
def test_identity_entries_equal_the_projection(H, W, fu, fd):
  """One identity entry per image equals ovn_project_batch / ovn_preprocess_batch of that cloud, for the seeded
  clouds above: none of them holds a negative zero coordinate, which M = I would turn into +0."""
  clouds = _clouds()
  for c in clouds:
    assert not (np.signbit(c[:, :3]) & (c[:, :3] == 0)).any()
  eng = _engine(H, W, fu, fd)
  batch = eng.upload_clouds(clouds)
  n = len(clouds)
  eo, ec, ep = np.arange(n + 1, dtype=np.int64), np.arange(n, dtype=np.int32), np.tile(np.eye(4), (n, 1, 1))
  got = eng.render(batch, eo, ec, ep)
  ref = eng.project(batch)
  for k in ('range', 'vertex', 'intensity'):
    assert np.array_equal(_bits(got[k]), _bits(ref[k])), k
  idx = _bits(ref['idx'])
  for i, c in enumerate(clouds):
    valid = oproj.projection_bins(c, fu, fd, H, W)[0]
    sel = np.flatnonzero(valid)
    want = np.where(idx[i] >= 0, sel[np.maximum(idx[i], 0)] if sel.size else -1, -1)
    assert np.array_equal(_bits(got['winner'])[i], want)
  assert np.array_equal(_bits(eng.render_preprocess(batch, eo, ec, ep)), _bits(eng.preprocess(batch)))
  eng.close()


def test_a_frame_has_the_same_bits_alone_in_a_batch_on_another_handle_and_again():
  clouds = _clouds()
  eo, ec, ep = random_entries(5, MAX_BATCH, len(clouds))
  results = []
  for _ in range(2):
    eng = _engine()
    batch = eng.upload_clouds(clouds)
    full = eng.render(batch, eo, ec, ep)
    again = eng.render(batch, eo, ec, ep)
    x = eng.render_preprocess(batch, eo, ec, ep)
    for v in (0, 4, MAX_BATCH - 1):
      alone = eng.render(batch, [0, eo[v + 1] - eo[v]], ec[eo[v]:eo[v + 1]], ep[eo[v]:eo[v + 1]])
      x1 = eng.render_preprocess(batch, [0, eo[v + 1] - eo[v]], ec[eo[v]:eo[v + 1]], ep[eo[v]:eo[v + 1]])
      for k in full:
        assert np.array_equal(_bits(alone[k])[0], _bits(full[k])[v]), (v, k)
      assert np.array_equal(_bits(x1)[0], _bits(x)[v])
    for k in full:
      assert np.array_equal(_bits(again[k]), _bits(full[k]))
    results.append({k: _bits(v) for k, v in full.items()})
    eng.close()
  for k in results[0]:
    assert np.array_equal(results[0][k], results[1][k])


# ---- refusals -------------------------------------------------------------------------------------------------
def _raw(eng, batch, offs, n_clouds, eo, ec, ep, n_virtual=None, out=None, preprocess=False):
  """ovn_render_batch / ovn_render_preprocess_batch on host tables as given (no Python checks)."""
  offs = np.ascontiguousarray(offs, np.int64)
  eo = np.ascontiguousarray(eo, np.int64)
  ec = np.ascontiguousarray(ec, np.int32)
  ep = np.ascontiguousarray(ep, np.float64).reshape(-1, 16)
  n_virtual = eo.size - 1 if n_virtual is None else n_virtual
  hp = lambda a: a.ctypes.data_as(C.c_void_p)
  L = lib()
  if preprocess:
    return L.ovn_render_preprocess_batch(eng._h, C.c_void_p(batch.points.data_ptr()), hp(offs), n_clouds, n_virtual,
                                         hp(eo), hp(ec), hp(ep), C.c_void_p(out.data_ptr()), eng._stream())
  return L.ovn_render_batch(eng._h, C.c_void_p(batch.points.data_ptr()), hp(offs), n_clouds, n_virtual, hp(eo),
                            hp(ec), hp(ep), C.c_float(-1.0), C.c_void_p(out.data_ptr()), None, None, None,
                            eng._stream())


def test_refusals_launch_nothing_and_the_handle_stays_usable():
  clouds = _clouds()
  eng = _engine()
  batch = eng.upload_clouds(clouds)
  offs = batch.offsets_host
  eo, ec, ep = random_entries(9, 3, len(clouds))
  want = _bits(eng.render(batch, eo, ec, ep)['range'])
  out = torch.full((MAX_BATCH + 1, 64, 900), 7.0, device='cuda')
  x = torch.full((MAX_BATCH + 1, 64, 900, eng.C), 7.0, device='cuda')
  n = len(clouds)

  def refused(status, **kw):
    args = dict(offs=offs, n_clouds=n, eo=eo, ec=ec, ep=ep)
    args.update(kw)
    st = _raw(eng, batch, args['offs'], args['n_clouds'], args['eo'], args['ec'], args['ep'], out=out)
    assert st == status, (kw, st, lib().ovn_last_error(eng._h))
    torch.cuda.synchronize()
    assert (out == 7.0).all()                                     # nothing launched, nothing written

  bad = offs.copy()
  bad[2] = bad[3] + 1
  refused(-1, offs=bad)                                           # decreasing cloud offsets
  bad = offs.copy()
  bad[0] = -1
  refused(-1, offs=bad)
  refused(-1, eo=np.array([0, 2, 1, eo[-1]]))                     # decreasing entry offsets
  refused(-1, eo=eo + 1, ec=np.concatenate([[0], ec]), ep=np.concatenate([[np.eye(4)], ep]))   # not from 0
  for c in (-1, n):                                               # a cloud index outside [0, n_clouds)
    e = ec.copy()
    e[-1] = c
    refused(-1, ec=e)
  for v in (float('nan'), float('inf')):                          # a pose that is not finite
    p = ep.copy()
    p[1, 0, 3] = v
    refused(-1, ep=p)
  for i, v in ((12, 1e-300), (14, -0.5), (15, 1.0 + 2 ** -52)):   # a bottom row that is not 0 0 0 1
    p = ep.copy()
    p.reshape(-1, 16)[0, i] = v
    refused(-1, ep=p)
  # an image concatenating 2^32 points: 2^32 / 30000 entries of the 30000-point cloud
  k = -(-(1 << 32) // clouds[0].shape[0])
  refused(-1, eo=np.array([0, k], np.int64), ec=np.zeros(k, np.int32), ep=np.tile(np.eye(4), (k, 1, 1)))
  # more images than max_batch_scans (Engine.render cuts its calls into chunks, so only a direct call gets here)
  refused(-6, eo=np.arange(MAX_BATCH + 2, dtype=np.int64), ec=np.zeros(MAX_BATCH + 1, np.int32),
          ep=np.tile(np.eye(4), (MAX_BATCH + 1, 1, 1)))
  assert np.array_equal(_bits(eng.render(batch, eo, ec, ep)['range']), want)   # the handle still renders
  eng.close()
  # renders carry no class probabilities: a semantic handle refuses the packed input, and still renders images
  sem = _engine(use={'use_class_probabilities': True})
  batch = sem.upload_clouds(clouds)
  xs = torch.empty((3, 64, 900, sem.C), device='cuda')
  assert _raw(sem, batch, offs, n, eo, ec, ep, out=xs, preprocess=True) == -2
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG'):
    sem.render_preprocess(batch, eo, ec, ep)
  assert np.array_equal(_bits(sem.render(batch, eo, ec, ep)['range']), want)
  sem.close()


# ---- the virtual map under the filter ----------------------------------------------------------------------------
def _infer():
  from overlapnet_b200.infer import Infer
  cfg = {'pretrained_weightsfilename': '', 'use_depth': True, 'use_normals': True, 'use_class_probabilities': False,
         'use_class_probabilities_pca': False, 'use_intensity': False, 'data_root_folder': '', 'infer_seqs': '',
         'batch_size': 4, 'model': copy.deepcopy(MODEL)}
  return Infer(cfg)


def _street(K, step=3.0):
  poses = np.stack([poses4([(step * k, 0.3 * math.sin(k), 0.05 * k)], 1.73)[0] for k in range(K)])
  return poses, [synth.street_scene_cloud(T, seed=9, n_azimuth=900) for T in poses]


def test_virtual_map_step_equals_render_leg_bank_and_step_observed():
  """OverlapMCL(virtual_spacing=...) is plumbing: its bank is render_preprocess + leg of the lattice frames' entries,
  its map is mcl_set_map of the lattice, and its steps are heads_1vsN on that bank + step_observed, bit for bit."""
  infer = _infer()
  eng = infer._engine
  poses, clouds = _street(6)
  spacing, md, m_src, radius = 1.0, 2.0, 3, 30.0
  m = mcl.OverlapMCL(infer, clouds, poses, max_distance=md, virtual_spacing=spacing, render_sources=m_src,
                     render_radius=radius)
  query = synth.street_scene_cloud(poses4([(7.2, 0.4, 0.3)], 1.73)[0], seed=9, n_azimuth=900)
  odoms = [(0.0, 0.0, 0.0), (1.0, 0.1, 0.05), (1.5, -0.2, 0.1)]
  m.init_global(5000, 3, init_radius=2.0)
  direct = [m.step(query, o) for o in odoms]
  p_direct = m.particles()
  # the composition
  frames = virtual_map.lattice(poses, spacing, md)
  eo, ec, ep = virtual_map.entries(frames, poses, m_src, radius)
  x = eng.render_preprocess(eng.upload_clouds(clouds), eo, ec, ep)
  bank = torch.cat([eng.leg(x[v0:v0 + eng.max_batch_scans]) for v0 in range(0, len(frames), eng.max_batch_scans)])
  assert np.array_equal(_bits(bank), _bits(m.bank))
  planar = mcl.planar(frames)
  assert np.array_equal(planar, m.keyframes)
  idx = mcl.MapIndex(planar[:, :2], m.index.cell, spacing)
  eng.mcl_set_map(planar, idx.raster, idx.x0, idx.y0, idx.cell)
  m.init_global(5000, 3, init_radius=2.0)
  composed = []
  for o in odoms:
    q = infer.encode_clouds([query])[0]
    composed.append(m.step_observed(o, lambda ids: eng.heads_1vsN(m.bank, q, cand_idx=ids)[:2]))
  assert direct == composed and any(e['n_touched'] > 0 for e in direct)
  assert np.array_equal(p_direct.view(np.uint64), m.particles().view(np.uint64))


@pytest.mark.parametrize('seed', range(5))
def test_filter_converges_on_the_lattice_with_a_true_sensor(seed):
  frames, idx, truth, odom, _ = lattice_scenario()
  eng = _engine(max_batch_scans=1)
  eng.mcl_set_map(frames, idx.raster, idx.x0, idx.y0, idx.cell)
  eng.mcl_init('global', 10 ** 4, seed, init_radius=1.0)
  T = 200
  pos, yaw = np.zeros(T), np.zeros(T)
  for t in range(T):
    touched, nt = eng.mcl_predict(odom[t], LATTICE['motion_sigma'])
    ov, yw = om.fake_sensor(truth[t], frames)(touched[:nt].cpu().numpy())
    e = eng.mcl_update(torch.as_tensor(ov).cuda(), torch.as_tensor(yw).cuda(), nt, LATTICE['sigma_overlap'],
                       LATTICE['sigma_yaw'], 0.5)
    pos[t] = math.hypot(e['x'] - truth[t, 0], e['y'] - truth[t, 1])
    yaw[t] = abs(mcl.wrap_pi(e['theta'] - truth[t, 2])) / (2 * math.pi / 360)
  c = mcl.convergence_step(pos, 2.0)
  print('seed %d: converged at step %d, largest errors after step 50: %.3f m, %.2f bins'
        % (seed, c, pos[50:].max(), yaw[50:].max()))
  assert 0 <= c <= GATE_CONVERGED_BY and pos[50:].max() < GATE_POSITION_M and yaw[50:].max() < GATE_YAW_BINS
  eng.close()


def test_cli_runs_a_virtual_map_end_to_end(tmp_path):
  import yaml
  n = 10
  scans = tmp_path / 'velodyne'
  scans.mkdir()
  poses, clouds = _street(n, step=1.5)
  lines = []
  for i in range(n):
    clouds[i].tofile(str(scans / ('%06d.bin' % i)))
    lines.append(' '.join('%.9f' % v for v in poses[i, :3].reshape(-1)))
  (tmp_path / 'poses.txt').write_text('\n'.join(lines) + '\n')
  (tmp_path / 'calib.txt').write_text('Tr: 1 0 0 0 0 1 0 0 0 0 1 0\n')
  net = {'pretrained_weightsfilename': '', 'use_depth': True, 'use_normals': True, 'use_class_probabilities': False,
         'use_intensity': False, 'batch_size': 4, 'model': copy.deepcopy(MODEL),
         'experiments_path': str(tmp_path / 'exp'), 'testname': 'mcl_virtual'}
  (tmp_path / 'net.yml').write_text(yaml.safe_dump(net))
  demo = {'Demo3': {'network_config': str(tmp_path / 'net.yml'), 'scan_folder': str(scans),
                    'poses_file': str(tmp_path / 'poses.txt'), 'calib_file': str(tmp_path / 'calib.txt')}}
  (tmp_path / 'demo.yml').write_text(yaml.safe_dump(demo))
  s = mcl.main([str(tmp_path / 'demo.yml'), '--keyframe-stride', '2', '--particles', '2000', '--runs', '2',
                '--max-distance', '2', '--virtual-spacing', '1', '--render-sources', '4'])
  out = tmp_path / 'exp' / 'mcl_virtual'
  assert json.loads((out / 'mcl_summary.json').read_text()) == json.loads(json.dumps(s))
  r = np.load(str(out / 'mcl_results.npz'))
  kf = poses[::2]
  frames = mcl.planar(virtual_map.lattice(kf, 1.0, 2.0))
  assert s['virtual_spacing'] == 1.0 and s['render_sources'] == 4 and s['render_radius'] == 50.0
  assert s['map_frames'] == frames.shape[0] and np.allclose(r['map_frames'], frames, atol=1e-6)   # poses via text
  assert s['keyframes'] == 5 and s['queries'] == 5 and r['estimate'].shape == (2, 5, 3)
  s0 = mcl.main([str(tmp_path / 'demo.yml'), '--keyframe-stride', '2', '--particles', '2000', '--runs', '1',
                 '--max-distance', '2'])
  assert not {'virtual_spacing', 'render_sources', 'render_radius', 'map_frames'} & set(s0)
  assert 'map_frames' not in np.load(str(out / 'mcl_results.npz')).files
