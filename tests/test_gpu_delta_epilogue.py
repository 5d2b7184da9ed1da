"""k_delta_conv1_wgmma writes o1 through a shared-memory staging buffer that a bulk copy stores while the consumers
compute the next unit.  A race on that buffer, or a kernel that ends before its stores complete, gives o1 bits that
depend on the call: here o1 and x3 (read back through Engine.heads_stage) must be bit-identical between two identical
calls, between the full call and calls over its first candidates (other work shares and staging reuse), between
query mode and pair mode on the same pairs, and between two copies of a pair whose units cross a 128-row o1 block at
different rows.  Each comparison follows a call on other data, so a store that never lands leaves bits that differ."""
import numpy as np
import pytest
import torch

from oracle import network as N
from overlapnet_b200 import synth
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
N_CAND = 1101
Q, Q_OTHER = 17, 23


def stages(eng):
  """o1 and x3 of the last call as int16 bit patterns (both are stored in fp16, so the conversion is exact)"""
  return tuple(eng.heads_stage(s).half().view(torch.int16) for s in ('o1', 'x3'))


def assert_bits_equal(a, b, what):
  for x, y, name in zip(a, b, ('o1', 'x3')):
    assert x.shape == y.shape, (what, name)
    if not torch.equal(x, y):
      raise AssertionError('%s: %s differs in %d values' % (what, name, int((x != y).sum())))


@pytest.fixture(scope='module')
def setup():
  w = N.glorot_weights(4, MODEL, seed=0)
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=N_CAND)
  bank_np = synth.feature_volumes(11, N_CAND)[:, 0] * np.float32(0.2)
  sel = np.arange(16)
  right_np = np.repeat(bank_np[Q][None, None], len(sel), 0)
  _, _, _, z0 = N.heads_forward(bank_np[sel][:, None], right_np, w, MODEL, return_logit=True)
  eng.load_weights(N.spread_dense(w, z0, target_std=1.5))
  bank = torch.from_numpy(bank_np).to(eng.device)
  yield eng, bank
  eng.close()


def other_call(eng, bank, n):
  """a call on another query, so that o1 and x3 of the first n pairs hold other values before the next call"""
  eng.heads_1vsN(bank, bank[Q_OTHER], n_cand=n)


def test_repeated_full_call(setup):
  eng, bank = setup
  eng.heads_1vsN(bank, bank[Q], n_cand=N_CAND)
  first = stages(eng)
  other_call(eng, bank, N_CAND)
  eng.heads_1vsN(bank, bank[Q], n_cand=N_CAND)
  assert_bits_equal(stages(eng), first, 'second 1 x %d call' % N_CAND)
  eng.check()


@pytest.mark.parametrize('n', [1, 37, 300])
def test_first_candidates_match_the_full_call(setup, n):
  eng, bank = setup
  eng.heads_1vsN(bank, bank[Q], n_cand=N_CAND)
  full = [s[:n].clone() for s in stages(eng)]
  other_call(eng, bank, N_CAND)
  eng.heads_1vsN(bank, bank[Q], n_cand=n)
  assert_bits_equal(stages(eng), full, 'first %d of %d candidates' % (n, N_CAND))
  eng.check()


def test_pair_mode_matches_query_mode(setup):
  eng, bank = setup
  n = 300
  eng.heads_1vsN(bank, bank[Q], n_cand=n)
  query = stages(eng)
  other_call(eng, bank, n)
  left = torch.arange(n, dtype=torch.int32)
  eng.heads(bank, left, torch.full((n,), Q, dtype=torch.int32))
  assert_bits_equal(stages(eng), query, 'pair mode against query mode, %d pairs' % n)
  eng.check()


def test_units_across_an_o1_block(setup):
  """Row m = pair * 576 + jb * 24 + ib of o1 lies in 128-row block m // 128, and 576 = 4.5 x 128: the units of
  pair 0 cross a block at jb = 5, 10, 21, those of pair 1 at jb = 2, 13, 18.  Two copies of one pair in pair mode
  give the same o1 and x3 at both places, and the query-mode values."""
  crossing = [[jb for jb in range(24) if (p * 576 + jb * 24) // 128 != (p * 576 + jb * 24 + 23) // 128]
              for p in (0, 1)]
  assert crossing == [[5, 10, 21], [2, 13, 18]]
  eng, bank = setup
  a = 5
  eng.heads_1vsN(bank, bank[Q], n_cand=a + 1)
  single = [s[a:a + 1] for s in stages(eng)]
  other_call(eng, bank, 4)
  eng.heads(bank, torch.full((2,), a, dtype=torch.int32), torch.full((2,), Q, dtype=torch.int32))
  both = stages(eng)
  assert_bits_equal([s[0:1] for s in both], single, 'pair 0 (o1 rows 0 .. 575)')
  assert_bits_equal([s[1:2] for s in both], single, 'pair 1 (o1 rows 576 .. 1151)')
  eng.check()
