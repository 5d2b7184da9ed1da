"""The host-side logic of a training image bank sharded over the GPUs of a node (overlapnet_b200.image_bank),
without a GPU: the placement rule over several ranks and the shard plan."""
import pytest

from overlapnet_b200 import _cabi, image_bank
from overlapnet_b200.image_bank import bank_rows


@pytest.mark.parametrize('bank,budget', [(10, 100), (10, 10), (11, 10), (0, 0), (100, 1)])
def test_one_rank_is_never_sharded(bank, budget):
  """One rank keeps today's rule whatever a shard would need: the bank on the device or in host memory."""
  got, b = image_bank.choose_rank_placement(bank, 0, [budget], ['a'])
  assert got == ('device' if bank <= budget else 'host') and b == budget
  assert got == image_bank.choose_placement(bank, budget + 7, 7)[0]


@pytest.mark.parametrize('bank,shard,budgets,want', [
    (100, 50, [100, 120], 'device'),        # the bank = the smallest budget
    (101, 51, [100, 120], 'sharded'),
    (101, 100, [100, 120], 'sharded'),      # ceil(n / world) images = the smallest budget
    (201, 101, [100, 300], 'host'),         # one shard past the smallest budget
    (101, 51, [300, 100, 300], 'sharded'),  # the smallest budget decides, whichever rank has it
    (301, 101, [300, 100, 300], 'host'),
    (100, 50, [120, 99], 'sharded'),        # the bank fits one rank but not the other
    (10, 5, [-3, 40], 'host'),              # a working set above one rank's free memory
])
def test_the_smallest_budget_decides(bank, shard, budgets, want):
  got, b = image_bank.choose_rank_placement(bank, shard, budgets, ['node0'] * len(budgets))
  assert got == want and b == min(budgets)


def test_ranks_on_different_hosts_never_shard():
  assert image_bank.choose_rank_placement(101, 51, [100, 100], ['node0', 'node1']) == ('host', 100)
  assert image_bank.choose_rank_placement(100, 51, [100, 100], ['node0', 'node1']) == ('device', 100)
  assert image_bank.choose_rank_placement(101, 51, [100] * 4, ['n0', 'n0', 'n1', 'n1'])[0] == 'host'


@pytest.mark.parametrize('n', [1, 5, 11])
@pytest.mark.parametrize('world', [1, 2, 3, 4])
def test_shard_plan(n, world):
  """Contiguous blocks in rank order that cover every row once and differ by at most one row; row -> (rank, local
  row) and back is the identity; each rank's keys are exactly its block of bank_rows."""
  first = image_bank.shard_plan(n, world)
  assert len(first) == world + 1 and first[0] == 0 and first[-1] == n
  sizes = [first[r + 1] - first[r] for r in range(world)]
  assert min(sizes) >= 0 and max(sizes) - min(sizes) <= 1 and sum(sizes) == n
  assert max(sizes) == -(-n // world)
  seen = []
  for row in range(n):
    r, local = image_bank.shard_of(first, row)
    assert 0 <= local < sizes[r] and first[r] + local == row
    seen.append((r, local))
  assert seen == sorted(seen) and len(set(seen)) == n
  keys = {('%02d' % (i % 2), '%06d' % i) for i in range(n)}
  rows = bank_rows(keys)
  mine = [set(k for k, row in rows.items() if first[r] <= row < first[r + 1]) for r in range(world)]
  assert set().union(*mine) == set(keys) and sum(len(m) for m in mine) == n
  for r in range(world):
    assert sorted(rows[k] for k in mine[r]) == list(range(first[r], first[r + 1]))


def test_shard_symbols_are_declared():
  for name in ('ovn_shard_create', 'ovn_shard_open', 'ovn_shard_close', 'ovn_gather_rows'):
    assert name in _cabi.SYMBOLS
  assert _cabi.IPC_HANDLE_BYTES == 64
  assert image_bank.PLACEMENTS == ('device', 'host', 'sharded')
