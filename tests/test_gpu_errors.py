"""Deferred device errors at the C ABI (VERDICT r1 "silent failure mode", ADVICE r1): a malformed
index or a pipeline-barrier time-out must come back as OVN_ERR_*, never as OVN_OK with garbage,
and must not take the handle down."""
import os

import numpy as np
import pytest
import torch

from oracle import network as N
from overlapnet_b200 import synth
from overlapnet_b200._cabi import OvnError
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}


@pytest.fixture(scope='module')
def bank_np():
  return synth.feature_volumes(9, 6)[:, 0]


@pytest.mark.parametrize('prec', ['f16_tc', 'fp32'])
def test_out_of_range_index_is_reported_not_read(bank_np, prec):
  eng = Engine(model=MODEL, precision=prec, max_batch_scans=1, max_batch_pairs=8)
  eng.load_weights(N.glorot_weights(4, MODEL, seed=0))
  bank = torch.from_numpy(bank_np).to(eng.device)
  good_l = torch.tensor([0, 1, 2], dtype=torch.int32)
  good_r = torch.tensor([3, 4, 5], dtype=torch.int32)
  ov_good, yaw_good, _ = eng.heads(bank, good_l, good_r)
  eng.check()
  for bad in (torch.tensor([0, 6, 2], dtype=torch.int32), torch.tensor([0, -1, 2], dtype=torch.int32),
              torch.tensor([0, 2 ** 30, 2], dtype=torch.int32)):
    ov, yaw, _ = eng.heads(bank, bad, good_r)
    with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG.*outside'):
      eng.check()
    if prec == 'f16_tc':                                       # outputs of the flagged call are poisoned
      assert torch.isnan(ov).all() and (yaw == -2 ** 31).all()
    ov, yaw, _ = eng.heads(bank, good_l, bad)                  # RIGHT list is checked too
    with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
      eng.check()
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.heads_1vsN(bank, bank[0], cand_idx=torch.tensor([5, 6], dtype=torch.int32))
    eng.check()
  with pytest.raises(OvnError, match='n_cand exceeds bank_size'):
    eng.heads_1vsN(bank, bank[0], n_cand=7)
  # the flag is cleared when reported: the handle keeps working and gives the same answer as before
  ov2, yaw2, _ = eng.heads(bank, good_l, good_r)
  eng.check()
  assert torch.equal(ov2, ov_good) and torch.equal(yaw2, yaw_good)
  eng.close()


def test_resident_bank_rows_must_be_prepared(bank_np):
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=8)
  eng.load_weights(N.glorot_weights(4, MODEL, seed=0))
  bank = torch.from_numpy(bank_np).to(eng.device)
  eng.bank_prepare(bank, 0, 4)                                 # rows 4, 5 exist in the tensor but were never prepared
  ov, yaw, _ = eng.heads_1vsN(bank, bank[0], cand_idx=torch.tensor([0, 3], dtype=torch.int32))
  eng.check()
  ov, yaw, _ = eng.heads_1vsN(bank, bank[0], cand_idx=torch.tensor([0, 4], dtype=torch.int32))
  with pytest.raises(OvnError, match='never passed to ovn_bank_prepare'):
    eng.check()
  eng.bank_prepare(bank, 4, 2)
  ov, yaw, _ = eng.heads_1vsN(bank, bank[0], cand_idx=torch.tensor([0, 4], dtype=torch.int32))
  eng.check()
  assert torch.isfinite(ov).all()
  eng.close()


def test_host_entry_point_reports_bad_candidates(bank_np):
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=8)
  eng.load_weights(N.glorot_weights(4, MODEL, seed=0))
  bank = torch.from_numpy(bank_np).to(eng.device)
  cloud = synth.kitti_like_cloud(3, n_points=20000)
  ov, yaw = eng.query_cloud_vs_bank_host(cloud, bank, n_cand=6)
  assert np.isfinite(ov).all()
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG'):
    eng.query_cloud_vs_bank_host(cloud, bank, cand_idx_host=np.array([1, 99], np.int32))
  ov2, yaw2 = eng.query_cloud_vs_bank_host(cloud, bank, n_cand=6)
  assert np.array_equal(ov, ov2) and np.array_equal(yaw, yaw2)
  eng.close()


def test_pipeline_failure_is_reported(bank_np):
  """OVN_DEBUG_FAULT makes k_conv2_wgmma skip its work and raise the pipeline-failure flag: the finalize
  kernels poison the outputs and the next synchronising call returns OVN_ERR_CUDA, naming the fault."""
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=8)
  eng.load_weights(N.glorot_weights(4, MODEL, seed=0))
  bank = torch.from_numpy(bank_np).to(eng.device)
  ov_good, yaw_good, _ = eng.heads_1vsN(bank, bank[0], n_cand=6)
  eng.check()
  os.environ['OVN_DEBUG_FAULT'] = '1'
  try:
    ov, yaw, _ = eng.heads_1vsN(bank, bank[0], n_cand=6)
    with pytest.raises(OvnError, match='OVN_ERR_CUDA.*pipeline failed: k_conv2_wgmma: fault injected.*code 501'):
      eng.check()
    assert torch.isnan(ov).all() and (yaw == -2 ** 31).all()
  finally:
    del os.environ['OVN_DEBUG_FAULT']
  ov2, yaw2, _ = eng.heads_1vsN(bank, bank[0], n_cand=6)
  eng.check()
  assert torch.equal(ov2, ov_good) and torch.equal(yaw2, yaw_good)
  eng.close()


@pytest.mark.parametrize('n', [1, 3])
@pytest.mark.parametrize('what', ['nan pixel', 'inf pixel', '-inf pixel', 'activation above 65504'])
def test_tensor_core_leg_reports_what_its_fp16_planes_cannot_hold(what, n):
  """The tensor-core leg hands each layer's activations to the next as hi / lo fp16 planes.  A NaN or infinite
  input pixel, or an activation above 65504 (hi = inf, lo = -inf, NaN in the next layer's MMAs, which its ReLU
  turns into 0), used to come back as an ordinary finite volume with OVN_OK.  The kernel that writes the planes
  now raises the deferred error: one scan (k_leg_layer1_small, k_leg_splitk_reduce) and a batch of 3
  (k_leg_layer1_direct, k_leg_mma's own epilogue).  The fp32 leg has no fp16 planes and propagates the value."""
  w = N.glorot_weights(4, MODEL, seed=0)
  x = synth.range_like_images(1234, n, 4)
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=n, max_batch_pairs=1)
  eng.load_weights(w)
  good = eng.leg(torch.from_numpy(x).to(eng.device)).clone()
  eng.check()
  if what == 'activation above 65504':               # s_conv5's activations reach 2.9 with these weights: x 2^15
    f = np.float32(2.0 ** 15)
    eng.load_weights(dict(w, s_conv5=(w['s_conv5'][0] * f, w['s_conv5'][1] * f)))
    bad = x
  else:
    bad = x.copy()
    bad[n - 1, 40, 451, 0] = {'nan pixel': np.nan, 'inf pixel': np.inf, '-inf pixel': -np.inf}[what]
  fv = eng.leg(torch.from_numpy(bad).to(eng.device))
  with pytest.raises(OvnError, match='OVN_ERR_INVALID_ARG.*tensor-core leg'):
    eng.check()
  eng.load_weights(w)                                  # the flag is cleared when reported: the handle keeps working
  assert torch.equal(eng.leg(torch.from_numpy(x).to(eng.device)), good)
  eng.check()
  eng.close()


def test_failed_workspace_allocation_leaves_handle_usable():
  """A projection whose rank workspace is larger than the device is refused by cudaMalloc before any kernel
  runs.  The handle reports OVN_ERR_CUDA once, then projects like a fresh handle: the workspace, which held
  this cloud's capacity before the failed grow, was left empty rather than with that stale capacity, and the
  next call does not report the old error again."""
  from overlapnet_b200._cabi import lib
  from overlapnet_b200.engine import _ptr
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=8)
  batch = eng.upload_clouds([synth.kitti_like_cloud(0, n_points=30000)])
  eng.project(batch)                                        # the rank workspace now has room for this cloud
  eng.check()
  idx = torch.empty((1, eng.H, eng.W), dtype=torch.int32, device=eng.device)
  n_huge = 16 * torch.cuda.mem_get_info(eng.device)[1]     # validity bitmask: 4 B per 32 points, > 2x the device
  st = lib().ovn_project_batch(eng._h, _ptr(batch.points), _ptr(batch.offsets), 1, n_huge, -1.0, None, None, None,
                               _ptr(idx), eng._stream())
  assert lib().ovn_status_string(st) == b'OVN_ERR_CUDA'
  assert b'cudaMalloc' in lib().ovn_last_error(eng._h)
  out = eng.project(batch)
  eng.check()
  fresh = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=8)
  ref = fresh.project(batch)
  fresh.check()
  for k in ('range', 'vertex', 'intensity', 'idx'):
    assert torch.equal(out[k].view(torch.int32), ref[k].view(torch.int32)), k
  eng.close()
  fresh.close()


def test_engine_on_non_current_device():
  """ADVICE r1: a handle is bound to its device; calls work whatever the caller's current device is."""
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  torch.cuda.set_device(0)
  eng = Engine(model=MODEL, precision='f16_tc', device=1, max_batch_scans=1, max_batch_pairs=4)
  eng.load_weights(N.glorot_weights(4, MODEL, seed=0))
  bank = torch.from_numpy(synth.feature_volumes(9, 3)[:, 0]).to(eng.device)
  assert torch.cuda.current_device() == 0
  ov, yaw, _ = eng.heads_1vsN(bank, bank[0], n_cand=3)
  eng.check()
  assert torch.isfinite(ov).all() and int(yaw[0]) == 0
  eng.close()


def test_empty_and_degenerate_calls(bank_np):
  """Empty candidate lists, empty row ranges and no-op calls return OVN_OK without launching work that
  could fault (SURVEY 8b: infer_multiple with [] returns None; infer_multiple_vs_multiple with [] too)."""
  for prec in ('f16_tc', 'fp32'):
    eng = Engine(model=MODEL, precision=prec, max_batch_scans=1, max_batch_pairs=8)
    eng.load_weights(N.glorot_weights(4, MODEL, seed=0))
    bank = torch.from_numpy(bank_np).to(eng.device)
    empty = torch.zeros((0,), dtype=torch.int32)
    ov, yaw, _ = eng.heads(bank, empty, empty)
    assert ov.numel() == 0 and yaw.numel() == 0
    ov, yaw, _ = eng.heads_1vsN(bank, bank[0], cand_idx=empty)
    assert ov.numel() == 0
    ov, yaw = eng.heads_rows_vs_bank(bank, 3, 3)
    assert ov.shape == (0, 6)
    fv = eng.leg(torch.zeros((0, 64, 900, 4), device=eng.device))
    assert fv.shape == (0, 360, 128)
    eng.calibrate(bank[1])                                   # no-op for fp32, explicit calibration for f16_tc
    mu, is_set = eng.get_feature_center()
    assert is_set == (prec == 'f16_tc')
    eng.peer_signal([], 1)
    eng.check()
    ov, yaw, _ = eng.heads_1vsN(bank, bank[2], n_cand=6)     # the handle is fully usable afterwards
    eng.check()
    assert int(yaw[2]) == 0 and torch.isfinite(ov).all()
    eng.close()


def test_sharded_infer_without_process_group_is_infer(tmp_path):
  """ShardedInfer with world size 1 (no process group) is the plain Infer: same numbers, same shapes."""
  import copy
  from overlapnet_b200 import weights as W
  from overlapnet_b200.infer import Infer
  from overlapnet_b200.sharded_infer import ShardedInfer
  model = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs', 'overlap_head': 'DeltaLayerConv1NetworkHead',
           'orientation_head': 'CorrelationHead', 'inputShape': [64, 900], 'leg_output_width': 360,
           'strides_layer1': [2, 2], 'additional_unsymmetric_layer3a': True}
  seq = tmp_path / '07'
  (seq / 'depth').mkdir(parents=True)
  (seq / 'normal').mkdir()
  x = synth.range_like_images(3, 4, 4)
  for i in range(4):
    np.save(str(seq / 'depth' / ('%06d.npy' % i)), x[i, :, :, 0])
    np.save(str(seq / 'normal' / ('%06d.npy' % i)), x[i, :, :, 1:4])
  wpath = str(tmp_path / 'w.npz')
  W.save_npz(wpath, N.glorot_weights(4, model, seed=2))
  cfg = {'pretrained_weightsfilename': wpath, 'use_depth': True, 'use_normals': True, 'use_class_probabilities': False,
         'use_class_probabilities_pca': False, 'use_intensity': False, 'data_root_folder': str(tmp_path),
         'infer_seqs': '07', 'batch_size': 16, 'model': model}
  a, b = Infer(copy.deepcopy(cfg)), ShardedInfer(copy.deepcopy(cfg))
  for inf in (a, b):
    assert inf.infer_multiple(0, []) is None and inf.infer_multiple(1, []) is None
  ra, rb = a.infer_multiple(2, [0, 1]), b.infer_multiple(2, [0, 1])
  assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1]) and ra[0].shape == rb[0].shape == (2,)
  ra, rb = a.infer_multiple(3, [1]), b.infer_multiple(3, [1])
  assert ra[0].shape == rb[0].shape == () and float(ra[0]) == float(rb[0])
  assert b.local_frames == [0, 1, 2, 3]
