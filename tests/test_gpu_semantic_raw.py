"""Semantic configs from raw scans: ``preprocess_cues`` (ovn_preprocess_cues_batch) against the reference's four cue
files -- depth, normals and intensity at max_range, the class probabilities at max_range = inf with the
filtered-index gather of gen_semantic_data.py:36-46 -- bit for bit, and the host entry points and ``Infer`` built
on it."""
import copy
import ctypes as C
import functools
import hashlib
import os
import shutil

import numpy as np
import pytest
import torch

from conftest import GOLDEN_CASES, load_golden
from oracle import projection as P
from overlapnet_b200 import synth
from overlapnet_b200._cabi import OvnError, lib
from overlapnet_b200.engine import Engine
from test_geometry import MODEL
from test_gpu_geometry import PROJ_GEOMETRIES, _clouds

pytestmark = pytest.mark.gpu

SEM24 = {'use_class_probabilities': True}
SEM25 = {'use_class_probabilities': True, 'use_intensity': True}
SEM_PCA = {'use_class_probabilities': True, 'use_class_probabilities_pca': True, 'use_intensity': True}
INFER_MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
               'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
               'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
               'additional_unsymmetric_layer3a': True}


def bits(a):
  a = np.ascontiguousarray(a)
  return a.view(np.uint32) if a.dtype == np.float32 else a


def sha(a):
  return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def far_tied_cloud(seed, n=40000):
  """A KITTI-shaped cloud of which a third lies between 50 and 150 m, with exact-depth ties on both sides of
  max_range (duplicated points, the copy later in the cloud with another intensity), points at exactly 50 m, and
  NaN / inf points that neither filter keeps."""
  c = synth.kitti_like_cloud(seed, n_points=n, zero_points=5)
  rng = np.random.default_rng(seed)
  far = c[rng.choice(n, n // 3, replace=False)].copy()
  far[:, :3] *= rng.uniform(50.0, 150.0, (len(far), 1)).astype(np.float32) / np.maximum(
      P.point_depth(far)[:, None], np.float32(1e-3))
  dup = np.concatenate([c[rng.choice(n, 2000, replace=False)], far[:2000]])
  dup[:, 3] = rng.uniform(0, 1, len(dup)).astype(np.float32)
  at50 = c[:300].copy()
  at50[:, :3] *= np.float32(50.0) / np.maximum(P.point_depth(at50)[:, None], np.float32(1e-3))
  bad = np.array([[np.nan, 1, 1, 0.5], [1, np.nan, 0, 0.5], [np.inf, 0, 0, 0.5], [0, -np.inf, 1, 0.5]], np.float32)
  pts = np.concatenate([c[:n // 2], far, at50, dup[:1000], bad, c[n // 2:], dup])
  return np.ascontiguousarray(pts, np.float32)


@functools.lru_cache(maxsize=None)
def _cue_clouds():
  clouds, probs = _clouds()
  extra = [far_tied_cloud(70), far_tied_cloud(71, n=3000)]
  clouds = list(clouds) + extra
  probs = list(probs) + [synth.random_probs(400 + i, c.shape[0]) for i, c in enumerate(extra)]
  return clouds, probs


def reference_cue_files(cloud, probs, H=64, W=900, fu=3.0, fd=-25.0):
  """The reference's four cue images of a scan: gen_depth / normal / semantic / intensity_data.py."""
  rng, vert, inten, _ = P.range_projection(cloud, fu, fd, H, W)
  return rng, P.gen_normal_map(rng, vert, H, W), P.gen_semantic_image(cloud, probs, H, W, fu, fd), inten


def packed(cues, use, n_prob=20):
  """pack_input of the cue files a config reads (prepareOneInput)."""
  rng, nrm, sem, inten = cues
  return P.pack_input(rng, nrm, sem[..., :n_prob], inten if use.get('use_intensity') else None)


def five_calls(eng, batch, probs_dev, intensity):
  """The device route without the fused mode: project at max_range, normals, project at inf for the index,
  semantic gather, pack."""
  out = eng.project(batch, want=('range', 'vertex', 'intensity'))
  nrm = eng.normals(out['range'], out['vertex'])
  idx_inf = eng.project(batch, max_range=float('inf'), want=('idx',))['idx']
  sem = eng.semantic(idx_inf, probs_dev, batch.offsets)
  return eng.pack_input(out['range'], nrm, sem, out['intensity'] if intensity else None)


def _engine(H=64, W=900, fu=3.0, fd=-25.0, use=None, precision='fp32', **kw):
  kw.setdefault('max_batch_scans', 8)
  kw.setdefault('max_batch_pairs', 1)
  return Engine(use=use, model=MODEL, precision=precision, proj_H=H, proj_W=W, fov_up=fu, fov_down=fd, **kw)


@pytest.mark.parametrize('H,W,fu,fd', PROJ_GEOMETRIES)
def test_cues_match_reference_cue_files_at_geometry(H, W, fu, fd):
  clouds, probs20 = _cue_clouds()
  ref = [reference_cue_files(c, p, H, W, fu, fd) for c, p in zip(clouds, probs20)]
  for use, n_prob, C_in in ((SEM24, 20, 24), (SEM25, 20, 25), (SEM_PCA, 3, 8)):
    eng = _engine(H, W, fu, fd, use)
    assert eng.C == C_in and eng.n_prob == n_prob
    batch = eng.upload_clouds(clouds)                       # 9 clouds > max_batch_scans = 8: two calls
    prob_dev = torch.from_numpy(np.concatenate([p[:, :n_prob] for p in probs20])).to(eng.device).contiguous()
    x = eng.preprocess_cues(batch, prob_dev).cpu().numpy()
    y = five_calls(eng, batch, prob_dev, 'use_intensity' in use).cpu().numpy()
    eng.check()
    eng.close()
    for i in range(len(clouds)):
      want = packed(ref[i], use, n_prob)
      assert np.array_equal(bits(x[i]), bits(want)), (use, i)
      assert np.array_equal(bits(y[i]), bits(want)), (use, i)


def test_far_points_and_ties_reach_the_second_key_image():
  """On the far / tied clouds the semantic cue's winners and ranks differ from the configured range's, so a
  single key image could not give the reference's probabilities; ovn_preprocess_batch (one range) differs."""
  clouds, probs = _cue_clouds()
  for c, pr in zip(clouds[-2:], probs[-2:]):
    _, _, _, idx_a = P.range_projection(c)
    _, _, _, idx_b = P.range_projection(c, max_range=np.inf)
    only_b = (idx_a < 0) & (idx_b >= 0)
    rank_moved = (idx_a >= 0) & (idx_b >= 0) & (idx_a != idx_b)
    assert only_b.sum() > 0 and rank_moved.sum() > 100, (only_b.sum(), rank_moved.sum())
    valid_b = np.isfinite(P.point_depth(c)) & (P.point_depth(c) > 0)
    sel = np.nonzero(valid_b)[0]
    d = P.point_depth(c)[sel]
    _, first = np.unique(d, return_index=True)
    assert len(d) - len(first) >= 1000                      # exact-depth ties among the points B keeps
    eng = _engine(use=SEM25)
    batch = eng.upload_clouds([c])
    p = torch.from_numpy(pr).to(eng.device)
    cues = eng.preprocess_cues(batch, p).cpu().numpy()[0]
    one_range = eng.preprocess(batch, p).cpu().numpy()[0]
    eng.close()
    assert np.array_equal(bits(cues), bits(packed(reference_cue_files(c, pr), SEM25)))
    assert not np.array_equal(bits(cues[..., 4:24]), bits(one_range[..., 4:24]))
    assert np.array_equal(bits(cues[..., :4]), bits(one_range[..., :4]))
    assert np.array_equal(bits(cues[..., 24]), bits(one_range[..., 24]))


def test_golden_scans(manifest):
  """The reference-generated goldens: depth, normals and intensity as shipped, the semantic cue with the
  manifest's SHA of gen_semantic_data's image for the seeded probabilities."""
  gs = [load_golden(c) for c in GOLDEN_CASES]
  probs = [synth.random_probs(manifest[c]['probs_seed'], g['points'].shape[0]) for c, g in zip(GOLDEN_CASES, gs)]
  eng = _engine(use=SEM25)
  x = eng.preprocess_cues(eng.upload_clouds([g['points'] for g in gs]),
                          torch.from_numpy(np.concatenate(probs)).to(eng.device)).cpu().numpy()
  eng.close()
  for i, (case, g) in enumerate(zip(GOLDEN_CASES, gs)):
    assert np.array_equal(bits(x[i, ..., 0]), bits(g['range'])), case
    assert np.array_equal(bits(x[i, ..., 1:4]), bits(g['normal'])), case
    assert sha(x[i, ..., 4:24]) == manifest[case]['semantic_sha_synthetic_probs'], case
    assert np.array_equal(bits(x[i, 24:28, :, 4:24]), bits(g['semantic_rows'])), case
    assert np.array_equal(bits(x[i, ..., 24]), bits(g['intensity'])), case


def test_geometric_handle_runs_the_one_range_path():
  clouds, _ = _cue_clouds()
  eng = _engine()
  batch = eng.upload_clouds(clouds)
  assert torch.equal(eng.preprocess_cues(batch), eng.preprocess(batch))
  eng.close()


def _weights(C_in, seed):
  from oracle import network as N
  return N.glorot_weights(C_in, MODEL, seed=seed)


@pytest.mark.parametrize('prec', ['fp32', 'f16_tc'])
def test_host_entry_points_match_device_stages(prec):
  clouds, probs = _cue_clouds()
  clouds, probs = clouds[-2:] + clouds[:2], probs[-2:] + probs[:2]
  eng = _engine(use=SEM25, precision=prec, max_batch_scans=3, max_batch_pairs=64)
  eng.load_weights(_weights(25, 8))
  batch = eng.upload_clouds(clouds)
  x = eng.preprocess_cues(batch, torch.from_numpy(np.concatenate(probs)).to(eng.device))
  fv = eng.leg(x).cpu().numpy()                            # 4 scans, max_batch_scans = 3: chunks of 3 and 1
  fv_host = eng.encode_clouds_host(clouds, probs)
  assert np.array_equal(bits(fv_host), bits(fv))
  bank = torch.from_numpy(synth.feature_volumes(5, 40)[:, 0]).to(eng.device)
  bank[:4] = torch.from_numpy(fv).to(eng.device)
  if prec == 'f16_tc':
    eng.bank_prepare(bank)
  q, q_probs = clouds[0], probs[0]
  xq = eng.preprocess_cues(eng.upload_clouds([q]), torch.from_numpy(q_probs).to(eng.device))
  fq = eng.leg(xq)[0]
  cand = np.array([3, 0, 39, 17, 2, 2], np.int32)
  for kw, dev_kw in (({'n_cand': 40}, {'n_cand': 40}),
                     ({'cand_idx_host': cand}, {'cand_idx': torch.from_numpy(cand)})):
    ov_d, yaw_d, _ = eng.heads_1vsN(bank, fq, **dev_kw)
    # the host entry points run on the handle's own stream and share its workspaces: the work queued on the
    # current stream (the bank's rows, the heads call above) finishes first
    ov_d, yaw_d, fq_h = ov_d.cpu().numpy(), yaw_d.cpu().numpy(), fq.cpu().numpy()
    qfv = np.empty((360, 128), np.float32)
    ov, yaw = eng.query_cloud_vs_bank_host(q, bank, out_query_fv=qfv, probs=q_probs, **kw)
    assert np.array_equal(bits(qfv), bits(fq_h))
    assert np.array_equal(bits(ov), bits(ov_d)), kw
    assert np.array_equal(yaw, yaw_d), kw
  eng.check()
  eng.close()


def test_refusals():
  clouds, probs = _cue_clouds()
  c, p = clouds[1], probs[1]
  L = lib()
  sem = _engine(use=SEM25, max_batch_pairs=4)
  sem.load_weights(_weights(25, 9))
  batch = sem.upload_clouds([c])
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    sem.preprocess_cues(batch)                             # missing probabilities
  offs = np.array([0, c.shape[0]], np.int64)
  fv = np.empty((1, 360, 128), np.float32)
  vp = lambda a: a.ctypes.data_as(C.c_void_p)
  assert L.ovn_status_string(L.ovn_encode_clouds_probs_host(sem._h, vp(c), vp(offs), 1, None, vp(fv))) == \
      b'OVN_ERR_INVALID_ARG'
  bank = torch.zeros((4, 360, 128), device=sem.device)
  ov, yaw = np.empty(4, np.float32), np.empty(4, np.int32)
  st = L.ovn_query_cloud_probs_vs_bank_host(sem._h, vp(c), c.shape[0], None, C.c_void_p(bank.data_ptr()), 4, None,
                                            4, vp(ov), vp(yaw), None)
  assert L.ovn_status_string(st) == b'OVN_ERR_INVALID_ARG'
  # a probability array of the wrong length, refused before the device
  for bad in (p[:-1], p[:, :19], np.concatenate([p, p[:1]])):
    with pytest.raises(ValueError, match='one row of 20 per point'):
      sem.preprocess_cues(batch, torch.from_numpy(bad))
    with pytest.raises(ValueError, match='one row of 20 per point'):
      sem.encode_clouds_host([c], [bad])
    with pytest.raises(ValueError, match='one row of 20 per point'):
      sem.query_cloud_vs_bank_host(c, bank, n_cand=4, probs=bad)
  # the entry points without probabilities keep their refusal of semantic handles
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG.*semantic channels need per-point probabilities'):
    sem.encode_clouds_host([c])
  with pytest.raises(OvnError, match='OVN_ERR_BAD_CONFIG.*semantic channels are not supported here'):
    sem.query_cloud_vs_bank_host(c, bank, n_cand=4)
  sem.close()
  geo = _engine(max_batch_pairs=4)
  geo.load_weights(_weights(4, 9))
  gbatch = geo.upload_clouds([c])
  with pytest.raises(ValueError, match='no probability channels'):
    geo.preprocess_cues(gbatch, torch.from_numpy(p))
  with pytest.raises(ValueError, match='no probability channels'):
    geo.encode_clouds_host([c], [p])
  with pytest.raises(ValueError, match='no probability channels'):
    geo.query_cloud_vs_bank_host(c, bank, n_cand=4, probs=p)
  pd = torch.from_numpy(p).to(geo.device)
  x = torch.empty((1, 64, 900, 4), device=geo.device)
  st = L.ovn_preprocess_cues_batch(geo._h, C.c_void_p(gbatch.points.data_ptr()), C.c_void_p(gbatch.offsets.data_ptr()),
                                   1, c.shape[0], C.c_void_p(pd.data_ptr()), C.c_void_p(x.data_ptr()), None)
  assert L.ovn_status_string(st) == b'OVN_ERR_INVALID_ARG'
  assert L.ovn_status_string(L.ovn_encode_clouds_probs_host(geo._h, vp(c), vp(offs), 1, vp(p), vp(fv))) == \
      b'OVN_ERR_INVALID_ARG'
  # without probabilities the new host entry point is the old one on a geometric handle
  assert L.ovn_encode_clouds_probs_host(geo._h, vp(c), vp(offs), 1, None, vp(fv)) == 0
  assert np.array_equal(bits(fv), bits(geo.encode_clouds_host([c])))
  geo.close()


def test_infer_raw_scans_equal_reference_cue_files(tmp_path):
  """The reference's flow for a semantic config -- gen_depth / normal / semantic / intensity_data.py write .npy cue
  files, the feeder reads probability/ (ImagePairOverlapOrientationSequence.py:166-191) -- against
  Infer.encode_clouds / infer_one_raw on the .bin and .label files."""
  from overlapnet_b200 import preprocess as pp
  from overlapnet_b200.infer import Infer
  scans, labels, seq = tmp_path / 'velodyne', tmp_path / 'labels', tmp_path / 'data' / '07'
  scans.mkdir()
  labels.mkdir()
  seq.mkdir(parents=True)
  clouds = [far_tied_cloud(80), synth.kitti_like_cloud(81, n_points=90000), far_tied_cloud(82, n=20000)]
  probs = [synth.random_probs(500 + i, c.shape[0]) for i, c in enumerate(clouds)]
  for i, (c, p) in enumerate(zip(clouds, probs)):
    c.tofile(str(scans / ('%06d.bin' % i)))
    p.tofile(str(labels / ('%06d.label' % i)))
  pp.gen_depth_data(str(scans), str(seq))
  pp.gen_normal_data(str(scans), str(seq))
  pp.gen_intensity_data(str(scans), str(seq))
  pp.gen_semantic_data(str(labels), str(scans), str(seq))
  shutil.copytree(str(seq / 'semantic'), str(seq / 'probability'))     # what Infer reads
  cfg = {'pretrained_weightsfilename': '', 'use_depth': True, 'use_normals': True, 'use_class_probabilities': True,
         'use_class_probabilities_pca': False, 'use_intensity': True, 'data_root_folder': str(tmp_path / 'data'),
         'infer_seqs': '07', 'batch_size': 4, 'model': copy.deepcopy(INFER_MODEL)}
  inf = Infer(cfg)
  names = ['000000', '000001', '000002']
  fv_files = inf.create_feature_volumes(names)
  fv_raw = inf.encode_clouds(clouds, probs).cpu().numpy()
  assert np.array_equal(bits(fv_raw), bits(fv_files[:, 0]))
  b = lambda i: str(scans / ('%06d.bin' % i))
  lab = lambda i: str(labels / ('%06d.label' % i))
  ov_raw, yaw_raw = inf.infer_one_raw(b(0), b(2), lab(0), lab(2))
  ov_npy, yaw_npy = inf.infer_one(b(0), b(2))
  assert np.array_equal(ov_raw, ov_npy) and np.array_equal(yaw_raw, yaw_npy)
  with pytest.raises(Exception, match='need per-point class scores'):
    inf.encode_clouds(clouds)
  with pytest.raises(Exception, match='one row of 20 per point'):
    inf.encode_clouds(clouds, [probs[0], probs[1][:-3], probs[2]])
  with pytest.raises(Exception, match='.label files of both scans'):
    inf.infer_one_raw(b(0), b(2), lab(0))
  assert os.path.isdir(str(seq / 'semantic'))
