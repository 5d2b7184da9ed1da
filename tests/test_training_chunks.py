"""``gradient_chunks`` without a GPU: the chunk bounds and each rank's chunk range, the refusals of the key, the
checkpoint fingerprint, the sizes the image bank plans for, and the batch loss summed in chunk order."""
import numpy as np
import pytest

from overlapnet_b200 import data_parallel, image_bank, training


def _covers(n, k, world):
  """Every pair of an n-pair batch once, contiguously and in order, over the chunks and over the ranks' ranges."""
  seen = []
  for rank in range(world):
    bounds, weights, (c0, c1), (a, b) = data_parallel.chunk_plan(n, k, world, rank)
    assert len(bounds) == k and bounds[0][0] == 0 and bounds[-1][1] == n
    assert all(bounds[c][1] == bounds[c + 1][0] for c in range(k - 1))
    assert all(hi - lo in (n // k, n // k + 1) for lo, hi in bounds)
    assert weights == [(hi - lo) / float(n) for lo, hi in bounds]
    assert c1 > c0 and (a, b) == (bounds[c0][0], bounds[c1 - 1][1])
    seen.append((c0, c1, a, b))
  assert seen[0][0] == 0 and seen[-1][1] == k and seen[0][2] == 0 and seen[-1][3] == n
  for (_, c1, _, b), (c0, _, a, _) in zip(seen, seen[1:]):
    assert c1 == c0 and b == a
  return seen


@pytest.mark.parametrize('n', [1, 2, 5, 16, 37])
def test_chunks_and_rank_ranges_cover_every_pair_once(n):
  for k in range(1, 9):
    for world in range(1, k + 1):
      _covers(n, k, world)


def test_short_last_batch_and_unequal_ranges():
  # batch 16 into K = 3 chunks of 6, 5, 5: on two ranks rank 0 trains 11 pairs
  assert [r[2:] for r in _covers(16, 3, 2)] == [(0, 11), (11, 16)]
  assert image_bank.share_pairs(16, 2, 3) == 11 and image_bank.share_pairs(16, 2) == 8
  # a last batch of 2 pairs into K = 4: chunks 1, 1, 0, 0; on three ranks the last rank's range is empty
  bounds, weights, _, _ = data_parallel.chunk_plan(2, 4, 3, 0)
  assert bounds == [(0, 1), (1, 2), (2, 2), (2, 2)] and weights == [0.5, 0.5, 0.0, 0.0]
  assert [r[:2] for r in _covers(2, 4, 3)] == [(0, 2), (2, 3), (3, 4)]
  assert data_parallel.chunk_plan(2, 4, 3, 2)[3] == (2, 2)
  # a full batch has the largest ranges
  for n in range(1, 17):
    assert max(b - a for _, _, a, b in _covers(n, 3, 2)) <= image_bank.share_pairs(16, 2, 3)
  assert data_parallel.chunk_rows(4, 3) == 2 and data_parallel.chunk_rows(4, 1) == 4


class _Eng:
  def gradient_size(self, whole_network):
    return 100 if whole_network else 10


def test_parts_bytes():
  assert image_bank.parts_bytes(_Eng(), True, 1) == 0
  assert image_bank.parts_bytes(_Eng(), True, 1, 4) == 4 * 100 * 4
  assert image_bank.parts_bytes(_Eng(), False, 3, 4) == (3 * 2 + 2) * 10 * 4


@pytest.mark.parametrize('value,world,match', [(0, 1, 'not an integer >= 1'), (-2, 1, 'not an integer >= 1'),
                                               (2.0, 1, 'not an integer >= 1'), ('4', 1, 'not an integer >= 1'),
                                               (True, 1, 'not an integer >= 1'), (None, 1, 'not an integer >= 1'),
                                               (65, 1, 'exceeds 64'), (17, 1, 'exceeds batch_size 16'),
                                               (2, 3, 'below the world size 3')])
def test_refusals(value, world, match):
  with pytest.raises(Exception, match=match):
    training.check_gradient_chunks({'batch_size': 16, 'gradient_chunks': value}, world)


def test_accepted_values():
  assert training.check_gradient_chunks({'batch_size': 16}) is None
  assert training.check_gradient_chunks({'batch_size': 16, 'gradient_chunks': 1}) == 1
  assert training.check_gradient_chunks({'batch_size': 16, 'gradient_chunks': np.int64(16)}, 16) == 16
  assert training.check_gradient_chunks({'batch_size': 64, 'gradient_chunks': 64}, 8) == 64


def _base_config():
  return {'model': {'legsType': '360OutputkLegs'}, 'batch_size': 16, 'no_batches_in_epoch': 10,
          'learning_rate': 1e-3, 'training_seqs': '00'}


def test_fingerprint_has_the_key_only_when_set():
  plain = training.trajectory_fingerprint(_base_config())
  assert 'gradient_chunks' not in plain
  assert sorted(plain) == ['batch_size', 'data_root_folder', 'learning_rate', 'lr_alpha', 'min_overlap_for_angle',
                           'model', 'no_batches_in_epoch', 'traindata_npzfile', 'training_seqs', 'use_class_probabilities',
                           'use_class_probabilities_pca', 'use_depth', 'use_intensity', 'use_normals',
                           'yaw_augmentation']
  chunked = training.trajectory_fingerprint(dict(_base_config(), gradient_chunks=4))
  assert chunked == dict(plain, gradient_chunks=4)
  assert training.trajectory_fingerprint(dict(_base_config(), gradient_chunks=2)) != chunked


class _Steps:
  """A flow whose chunked gradients are fixed numbers per pair, recording what the step asked for."""
  whole_network = False

  def __init__(self):
    self.calls = []

  def gradients(self, left, right, gt_overlap, gt_orientation, min_overlap, rotate=None, chunks=None):
    offsets, parts = chunks
    self.calls.append((left.tolist(), list(offsets)))
    out = []
    for c in range(len(offsets) - 1):
      pairs = left[offsets[c]:offsets[c + 1]].double()
      parts[c] = float(pairs.sum()) if len(pairs) else 0.0
      out.append((float(pairs.mean()) if len(pairs) else 0.0, 0.1, 0.2))
    return out


class _StepEng:
  def __init__(self):
    self.steps = []

  def adagrad_step_sum(self, parts, weights, lr, whole_network):
    self.steps.append((parts.clone(), list(weights)))


def test_one_process_step_sums_the_chunks_in_order():
  import torch
  steps, eng = _Steps(), _StepEng()
  left = torch.arange(100, 116, dtype=torch.int32)
  parts = torch.full((3, 2), -1.0)
  loss = training._step(None, steps, eng, data_parallel.step_plan(16, 1, 0, 3), parts, parts, 0, left, left, left, left,
                        0.7, 1e-3, None)
  assert steps.calls == [(list(range(100, 116)), [0, 6, 11, 16])]
  (got, weights), = eng.steps
  assert weights == [6 / 16, 5 / 16, 5 / 16]
  assert got[:, 0].tolist() == [sum(range(100, 106)), sum(range(106, 111)), sum(range(111, 116))]
  means = [np.mean(range(100, 106)), np.mean(range(106, 111)), np.mean(range(111, 116))]
  expect = float(sum(w * np.float64(m) for w, m in zip(weights, means)))
  assert loss[0] == expect and loss[1] == float(sum(w * 0.1 for w in weights))
  # a short last batch: chunks of 1, 1, 0; the empty chunk has weight 0
  eng.steps.clear()
  training._step(None, steps, eng, data_parallel.step_plan(2, 1, 0, 3), parts, parts, 16,
                 torch.arange(18, dtype=torch.int32), left, left, left, 0.7, 1e-3, None)
  assert steps.calls[-1] == ([16, 17], [0, 1, 2, 2]) and eng.steps[0][1] == [0.5, 0.5, 0.0]
