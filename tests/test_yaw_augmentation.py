"""CPU checks of yaw augmentation (overlapnet_b200.augment, ``yaw_augmentation: True``): the NumPy oracle of the
augmented image against the projection of the rotated cloud, the moved label against the ground-truth yaw bin of
the rotated pose and against the correlation head's argmax, the shift sampler, and the training configs."""
import os

import numpy as np
import pytest
import torch

from oracle import gt as G
from oracle import network as N
from oracle import projection as P
from overlapnet_b200 import augment, training, training_leg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')

# (W, Wf, column pitch, label step in bins)
PITCHES = [(900, 360, 5, 2), (900, 225, 4, 1), (900, 405, 20, 9)]


def augment_oracle(images, rows, shifts, rot, c_normal):
  """NumPy statement of ovn_gather_images: images[rows[i]] rolled by shifts[i] columns, the normal channels at
  c_normal (None: no normals) rotated by rot[i] = (cos, sin) in float32 unless they hold the (-1, -1, -1) fill."""
  out = np.stack([np.roll(images[r], int(s), axis=1) for r, s in zip(rows, shifts)]).astype(np.float32)
  if rot is None or c_normal is None:
    return out
  for i in range(len(rows)):
    c, s = np.float32(rot[i][0]), np.float32(rot[i][1])
    nx, ny = out[i, ..., c_normal].copy(), out[i, ..., c_normal + 1].copy()
    keep = ~np.all(out[i, ..., c_normal:c_normal + 3] == -1, axis=-1)
    out[i, ..., c_normal][keep] = (c * nx - s * ny)[keep]
    out[i, ..., c_normal + 1][keep] = (s * nx + c * ny)[keep]
  return out


def rotate_cloud(points, theta):
  """The float32 cloud rotated about z by theta (in float64, rounded to float32 like a stored scan)."""
  R = np.array([[np.cos(theta), -np.sin(theta)], [np.sin(theta), np.cos(theta)]])
  out = points.copy()
  out[:, :2] = (points[:, :2].astype(np.float64) @ R.T).astype(np.float32)
  return out


def _edge_points(points, pixels, tol=2e-3):
  """True where some point of the cloud that falls into one of ``pixels`` ((y, x) list) lies within tol of a row
  or column edge of the projection: a pixel such a point decides can change under float32 rounding."""
  _, py, px = P.projection_prefloor(points)
  valid, _, iy, ix = P.projection_bins(points)
  near = (np.abs(px - np.round(px)) < tol) | (np.abs(py - np.round(py)) < tol)
  return [bool(np.any(valid & near & (iy == y) & (ix == x))) for y, x in pixels]


@pytest.mark.parametrize('case', ['kitti_000000', 'synth_3'])
def test_rotated_cloud_projects_to_the_augmented_image(case):
  """For every nonzero multiple of 5 columns at 64 x 900, the projection of the rotated cloud equals the
  augmented image of the unrotated one: same valid and normal-fill masks, depth and normals within float32
  rounding of the rotated points except at a few bin-edge pixels.  A plain roll fails the normal bound."""
  pts = np.load(os.path.join(GOLDEN, case + '.npz'))['points']
  rng, vert, _, _ = P.range_projection(pts)
  x = P.pack_input(rng, P.gen_normal_map(rng, vert))
  worst = {'depth': 0, 'normal': 0, 'mask': 0}
  plain_fails = False
  for s in range(5, 900, 5):
    q = rotate_cloud(pts, -2 * np.pi * s / 900)
    r2, v2, _, _ = P.range_projection(q)
    want = P.pack_input(r2, P.gen_normal_map(r2, v2))
    got = augment_oracle(x[None], [0], [s], augment.rotation([s], 900), 1)[0]
    valid_diff = np.argwhere((want[..., 0] > 0) != (got[..., 0] > 0))
    fill_w, fill_g = np.all(want[..., 1:] == -1, -1), np.all(got[..., 1:] == -1, -1)
    fill_diff = np.argwhere(fill_w != fill_g)
    # synth_3 at s = 815: one point 6.47 m away sits on a column edge and changes pixel under the rotation's
    # float32 rounding, which changes that pixel's validity and the normals of it and its two upper / left
    # neighbours.  Every mask difference must be such a pixel; on kitti_000000 there is none.
    for y, xx in valid_diff:
      assert any(_edge_points(q, [(y, xx)]) + _edge_points(pts, [(y, (xx - s) % 900)])), (case, s, y, xx)
    near = {(int(y), int(xx)) for y, xx in valid_diff}
    for y, xx in fill_diff:
      assert {(y, xx), (y, (xx + 1) % 900), (y + 1, xx)} & near, (case, s, y, xx)
    worst['mask'] = max(worst['mask'], len(valid_diff))
    m = (want[..., 0] > 0) & (got[..., 0] > 0)
    d_depth = int(np.sum(np.abs(want[..., 0][m] - got[..., 0][m]) > 1e-6 * np.abs(got[..., 0][m])))
    ok = ~fill_w & ~fill_g
    d_normal = int(np.sum(np.any(np.abs(want[..., 1:] - got[..., 1:]) > 1e-3, -1) & ok))
    worst['depth'] = max(worst['depth'], d_depth)
    worst['normal'] = max(worst['normal'], d_normal)
    plain = np.roll(x, s, axis=1)
    plain_fails |= int(np.sum(np.any(np.abs(want[..., 1:] - plain[..., 1:]) > 1e-3, -1) & ok)) > 50
  print(case, 'worst over 179 shifts:', worst)
  if case == 'kitti_000000':
    assert worst['mask'] == 0
  assert worst['mask'] <= 2
  assert worst['depth'] <= 10
  assert worst['normal'] <= 50
  assert plain_fails


def _rz(theta):
  R = np.eye(4)
  R[:2, :2] = [[np.cos(theta), -np.sin(theta)], [np.sin(theta), np.cos(theta)]]
  return R


def _near_edge(yaw, Wf, tol=1e-9):
  k = np.round(-yaw * Wf / (2 * np.pi))
  return abs(yaw + 2 * np.pi * k / Wf) < tol


@pytest.mark.parametrize('W,Wf,p,step', PITCHES)
def test_moved_label_is_the_ground_truth_bin_of_the_rotated_pose(W, Wf, p, step):
  """Rotating RIGHT (the reference frame) by theta replaces pose_ref with pose_ref . Rz(-theta): the yaw bin of
  cur_inv . pose_ref . Rz(-theta) (com_overlap_yaw.py:49-54) is move_labels of the original bin, for every pose
  pair of the golden sequence and every multiple of the pitch.

  The reference's yaw is the Z angle of a ZYX Euler decomposition (utils.py:189-216), and a rotation about the
  scan's own z axis moves it by exactly -theta only when the relative pose has no roll or pitch.  The golden
  poses tilt by up to 1.3 degrees, and the Euler yaw then moves by -theta within 2.5e-4 rad (second order in the
  tilt), which is checked first.  Bins are compared where neither yaw lies within 5e-4 rad of a bin edge.  The
  reference's bin of a yaw of exactly -pi is Wf; the label is taken mod Wf like the circular correlation."""
  poses = np.load(os.path.join(GOLDEN, 'gt_overlap_yaw.npz'))['poses']
  tilt_bound = 5e-4
  checked = skipped = 0
  for f in range(len(poses)):
    cur_inv = np.linalg.inv(poses[f])
    for r in range(len(poses)):
      rel = cur_inv.dot(poses[r])
      yaw0 = G.yaw_from_rotation(rel[:3, :3])
      label0 = G.yaw_bin(yaw0, Wf)
      for s in range(0, W, p):
        yaw = G.yaw_from_rotation(rel.dot(_rz(2 * np.pi * s / W))[:3, :3])
        moved = (yaw - yaw0 - 2 * np.pi * s / W + np.pi) % (2 * np.pi) - np.pi
        assert abs(moved) <= tilt_bound, (f, r, s, moved)
        if _near_edge(yaw0, Wf, tilt_bound) or _near_edge(yaw, Wf, tilt_bound):
          skipped += 1
          continue
        assert G.yaw_bin(yaw, Wf) % Wf == augment.move_labels(label0, s, W, Wf), (f, r, s)
        checked += 1
  print('checked %d, skipped %d (bin edges)' % (checked, skipped))
  # the golden poses differ by whole-degree yaws (10, 93, -140 ...), which are bin edges at Wf = 360: 1440 of the
  # 4500 cases are compared there, 900 to 4500 at the other widths
  assert checked >= 900
  assert augment.move_labels(np.array([0, 1, Wf - 1]), np.array([p, p, 0]), W, Wf).tolist() == \
      [(-step) % Wf, (1 - step) % Wf, Wf - 1]


@pytest.mark.parametrize('W,Wf,p,step', PITCHES)
def test_correlation_argmax_moves_with_the_label(W, Wf, p, step):
  """The correlation head's argmax on RIGHT = roll(L, d) is (-d - Wf//2) mod Wf (tests/test_geometry.py): rolling
  the RIGHT features by d = s Wf / W more moves it exactly like move_labels."""
  rng = np.random.default_rng(Wf)
  L = np.abs(rng.standard_normal((1, 1, Wf, 16))).astype(np.float32)
  R0 = np.roll(L, 17, axis=2)
  label0 = int(np.argmax(N.correlation_head(L, R0)[0]))
  for s in range(0, W, p):
    R = np.roll(R0, s * Wf // W, axis=2)
    assert int(np.argmax(N.correlation_head(L, R)[0])) == augment.move_labels(label0, s, W, Wf), s


@pytest.mark.parametrize('W,Wf,p,step', PITCHES)
def test_sample_shifts_are_reproducible_multiples_of_the_pitch(W, Wf, p, step):
  assert augment.column_pitch(W, Wf) == p and p * Wf // W == step
  np.random.seed(4)
  a = augment.sample_shifts(2000, W, Wf)
  np.random.seed(4)
  b = augment.sample_shifts(2000, W, Wf)
  assert a.dtype == np.int32 and np.array_equal(a, b)
  assert np.all(a % p == 0) and a.min() >= 0 and a.max() < W
  assert len(set(a.tolist())) == W // p              # 2000 draws reach every multiple
  with pytest.raises(ValueError, match='pitch'):
    augment.move_labels(np.zeros(2, np.int64), np.array([0, p + 1]), W, Wf)


def test_rotation_is_minus_two_pi_shift_over_width():
  r = augment.rotation(np.array([0, 225, 450, 5]), 900)
  assert r.dtype == np.float32 and r.shape == (4, 2)
  assert np.allclose(r[:3], [[1, 0], [0, -1], [-1, 0]], atol=1e-7)
  assert np.array_equal(r[3], np.array([np.cos(-np.pi / 90), np.sin(-np.pi / 90)], np.float32))
  t = augment.move_labels(torch.tensor([0, 100], dtype=torch.int32), torch.tensor([5, 450], dtype=torch.int32),
                          900, 360)
  assert t.dtype == torch.int32 and t.tolist() == [358, 280]


# ---- training configs --------------------------------------------------------------------------------------
def _config(tmp_path, legs, **kw):
  cfg = {'experiments_path': str(tmp_path), 'testname': 't', 'pretrained_weightsfilename': '',
         'traindata_npzfile': 'x', 'validationdata_npzfile': 'y', 'batch_size': 2, 'no_batches_in_epoch': 1,
         'no_epochs': 1, 'no_test_pairs': 1, 'learning_rate': 1e-3,
         'model': {'modelType': 'SiameseNetworkTemplate', 'legsType': legs,
                   'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
                   'inputShape': [64, 900], 'leg_output_width': 360}}
  cfg.update(kw)
  return cfg


FLOWS = [('360OutputkLegsFixed', training), ('360OutputkLegs', training_leg)]


@pytest.mark.parametrize('legs,module', FLOWS)
def test_both_flows_accept_the_key(tmp_path, legs, module):
  module.check_config(_config(tmp_path, legs, yaw_augmentation=True))
  module.check_config(_config(tmp_path, legs, yaw_augmentation=False))


@pytest.mark.parametrize('legs,module', FLOWS)
def test_a_width_without_whole_bin_rotations_is_refused(tmp_path, legs, module):
  cfg = _config(tmp_path, legs, yaw_augmentation=True)
  cfg['model']['inputShape'] = [32, 457]
  with pytest.raises(Exception, match='W = 457.*Wf = 360'):
    module.check_config(cfg)
  with pytest.raises(Exception, match='W = 457'):
    module.train(cfg)                               # refused before any file or device is touched
  assert not os.path.exists(os.path.join(str(tmp_path), 't'))
  cfg['yaw_augmentation'] = False
  module.check_config(cfg)


@pytest.mark.parametrize('legs,module', FLOWS)
def test_reference_rotation_key_stays_refused(tmp_path, legs, module):
  with pytest.raises(Exception, match='rotate_training_data'):
    module.check_config(_config(tmp_path, legs, yaw_augmentation=True, rotate_training_data=1))


class _Engine:
  device = torch.device('cpu')
  W = 900

  def get_weights(self):
    return {}

  def check(self):
    pass


class _Infer:
  def __init__(self, cfg, precision, device, max_batch_pairs):
    self._engine = _Engine()
    self.network_output_size = cfg['model']['leg_output_width']


class _Flow:
  """Records what the loop hands to each step."""
  calls = []

  def __init__(self, infer, keys, rotate_keys=None):
    self.rows = {k: i for i, k in enumerate(sorted(keys))}
    self.image_rows = {k: 100 + i for i, k in enumerate(sorted(rotate_keys or ()))}
    _Flow.instance = self
    _Flow.calls.append(('init', rotate_keys))

  def step(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, lr, rotate=None):
    _Flow.calls.append(('step', left.clone(), right.clone(), gt_orientation.clone(), rotate))
    return (1.0, 0.5, 0.5)

  def evaluate(self, left, right):
    return torch.zeros(left.numel()), torch.full((left.numel(),), 180, dtype=torch.int32)


def _train_on_fakes(tmp_path, monkeypatch, **kw):
  """training._train on a 12-pair training file and a 3-pair validation file, with a fake handle and flow."""
  table = np.array([[i, (i + 1 + i // 6) % 6, 0.5, (37 * i) % 360] for i in range(12)], float)
  np.savez(os.path.join(str(tmp_path), 'train.npz'), overlaps=table, seq=np.array([['00', '00']] * 12))
  np.savez(os.path.join(str(tmp_path), 'val.npz'), overlaps=table[:3], seq=np.array([['00', '00']] * 3))
  cfg = _config(tmp_path, '360OutputkLegs', traindata_npzfile=os.path.join(str(tmp_path), 'train.npz'),
                validationdata_npzfile=os.path.join(str(tmp_path), 'val.npz'), batch_size=5, no_batches_in_epoch=3,
                no_epochs=2, no_test_pairs=3, **kw)
  monkeypatch.setattr(training, 'save_weights', lambda path, w: None)
  _Flow.calls = []
  training._train(cfg, cfg['model'], '', str(tmp_path), None, _Infer, _Flow)
  return table


@pytest.mark.parametrize('on', [False, True])
def test_train_loop_draws_and_hands_over_the_rotation(tmp_path, monkeypatch, caplog, on):
  """Key off: the loop draws exactly what it drew before (the npz shuffle, one batch permutation per epoch) and
  hands no rotation to the steps.  Key on: one shift per training pair at the start of each epoch as well, and
  each step gets the RIGHT image rows, the shifts, their rotation and the labels moved by them."""
  import logging
  caplog.set_level(logging.INFO, logger='overlapnet_b200.training')
  np.random.seed(7)
  table = _train_on_fakes(tmp_path, monkeypatch, **({'yaw_augmentation': True} if on else {}))
  after = np.random.get_state()[1].copy()
  np.random.seed(7)
  np.random.permutation(12)
  want_shifts = []
  for _ in range(2):
    if on:
      want_shifts.append(np.random.randint(0, 180, 12) * 5)
    np.random.permutation(3)
  assert np.array_equal(np.random.get_state()[1], after)
  assert ('rotation of training data: RIGHT images by a random multiple of 5 columns (2 bins), labels moved'
          in caplog.text) == on
  assert ('NO rotation of training data' in caplog.text) == (not on)
  steps = [c for c in _Flow.calls if c[0] == 'step']
  assert len(steps) == 6
  rotate_keys = _Flow.calls[0][1]
  assert (rotate_keys is not None) == on
  if on:                                             # the RIGHT scans of the training pairs
    assert rotate_keys == {('00', '%06d' % k) for k in table[:, 1].astype(int)}
  keys = sorted({('00', '%06d' % k) for k in table[:, :2].ravel().astype(int)})
  inv = dict(enumerate(keys))
  label = {('%06d' % a, '%06d' % b): o for a, b, _, o in table.astype(int)}
  for i, (_, left, right, gt_or, rotate) in enumerate(steps):
    assert (rotate is not None) == on
    orig = np.array([label[(inv[int(l)][1], inv[int(r)][1])] for l, r in zip(left, right)])
    if not on:
      assert gt_or.tolist() == orig.tolist()
      continue
    rows, shifts, rot = rotate
    assert rows.tolist() == [_Flow.instance.image_rows[inv[int(r)]] for r in right]
    epoch_shifts = want_shifts[i // 3]
    assert set(shifts.tolist()) <= set(epoch_shifts.tolist())
    assert gt_or.tolist() == ((orig - shifts.numpy() * 360 // 900) % 360).tolist()
    assert np.array_equal(rot.numpy(), augment.rotation(shifts.numpy(), 900))
  if on:   # the pair order of an epoch is the shuffled file order; its shifts are drawn in that order
    all_shifts = np.concatenate([s[4][1].numpy() for s in steps[:3]])
    assert sorted(all_shifts.tolist()) == sorted(want_shifts[0].tolist())
