"""The host-side logic of a training image bank in host memory (overlapnet_b200.image_bank), without a GPU: the
step planner, the placement rule and the refusal of a failed pin."""
import numpy as np
import pytest

from overlapnet_b200 import image_bank


@pytest.mark.parametrize('seed', range(20))
def test_plan_stages_every_row_a_step_reads(seed):
  """Random batches with repeated scans, LEFT = RIGHT pairs and yaw rows (the RIGHT rows again, or other rows of
  an image bank of RIGHT scans): the slot filled with bank[rows] gives bank[row] at every local index, in the
  order of first appearance, and never holds more than 2 B rows."""
  rng = np.random.default_rng(seed)
  n_bank, B = int(rng.integers(1, 40)), int(rng.integers(1, 17))
  bank = rng.standard_normal((n_bank, 3)).astype(np.float32)
  n = int(rng.integers(1, B + 1))
  left = rng.integers(0, n_bank, n)
  right = np.where(rng.random(n) < 0.3, left, rng.integers(0, n_bank, n))
  for lists in ((left, right), (left, right.copy()), (right,), (left,)):
    rows, local = image_bank.plan_rows(*lists)
    assert rows.dtype == np.int64 and len(local) == len(lists)
    assert rows.size == np.unique(np.concatenate(lists)).size <= 2 * B
    slot = bank[rows]                                          # what the ring's copies put into a slot
    for src, loc in zip(lists, local):
      assert loc.dtype == np.int32 and loc.shape == src.shape
      assert np.array_equal(slot[loc], bank[src])
    seen = []
    for r in np.concatenate(lists):                            # the fixed order: first appearance
      if r not in seen:
        seen.append(int(r))
    assert rows.tolist() == seen


def test_plan_of_nothing_and_of_one_repeated_row():
  rows, (a,) = image_bank.plan_rows(np.zeros(0, np.int64))
  assert rows.size == 0 and a.size == 0
  rows, (a, b) = image_bank.plan_rows([7, 7, 7], [7])
  assert rows.tolist() == [7] and a.tolist() == [0, 0, 0] and b.tolist() == [0]


@pytest.mark.parametrize('bank,free,ws,want', [
    (10, 100, 90, 'device'),          # fits exactly
    (11, 100, 90, 'host'),
    (0, 0, 0, 'device'),
    (1, 100, 200, 'host'),            # the working set alone exceeds the free memory
    (74_300_000_000, 76_000_000_000, 3_000_000_000, 'host'),
    (11_900_000_000, 79_000_000_000, 3_000_000_000, 'device'),
])
def test_placement_rule(bank, free, ws, want):
  got, budget = image_bank.choose_placement(bank, free, ws)
  assert got == want and budget == free - ws


def test_share_pairs():
  assert image_bank.share_pairs(16, 1) == 16
  assert image_bank.share_pairs(16, 3) == 6
  assert image_bank.share_pairs(2, 4) == 1


class _Engine:
  H, W, C = 4, 9, 5

  def __init__(self, fail):
    self.fail, self.pinned = fail, []

  def host_register(self, array):
    if self.fail:
      raise RuntimeError('cudaHostRegister failed: out of memory')
    self.pinned.append(array)

  def host_unregister(self, array):
    self.pinned.remove(array)


def test_failed_pin_names_the_bytes_it_needed():
  with pytest.raises(Exception, match=r'could not pin 5040 bytes \(0\.00 GB\) for 7 images of 4 x 9 x 5 float32: '
                                      r'cudaHostRegister failed: out of memory'):
    image_bank.HostBank(_Engine(True), 7)


def test_host_bank_is_one_block_released_on_close():
  eng = _Engine(False)
  bank = image_bank.HostBank(eng, 7)
  assert bank.images.shape == (7, 4, 9, 5) and bank.images.dtype == np.float32 and bank.images.flags['C_CONTIGUOUS']
  assert bank.nbytes == 5040 and eng.pinned == [bank.images]
  bank.close()
  bank.close()
  assert eng.pinned == []


def test_unknown_placement_is_refused():
  class Infer:
    _engine = _Engine(False)
  with pytest.raises(ValueError, match="image_bank 'gpu'"):
    image_bank.open_bank(Infer(), {('00', 'a')}, 'gpu', 1, True, 0, 1, 'Image bank')
