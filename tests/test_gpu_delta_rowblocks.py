"""In query mode (every pair meets the same RIGHT volume) k_delta_conv1_wgmma packs the flat LEFT rows
g = pair * 360 + i into blocks of 384 rows that may straddle two pairs; pair mode keeps one pair per block.  Where a
row sits in a wgmma tile does not change its bits, so o1, x3, the overlaps, the yaws and the correlation curves of a
1-vs-N call must equal those of the same pairs in pair mode bit for bit: for small and large n, for blocks that
start at every row offset i0 = 384 b mod 360 of a pair, for a partial last block, for work shares that start and end
inside a block (restated from the device's SM count) and for a resident bank read through a permuted index list.
Each call follows a call on another query, so a store that never lands leaves bits that differ."""
import numpy as np
import pytest
import torch

from oracle import network as N
from overlapnet_b200 import synth
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
N_BANK = 1101
Q, Q_OTHER = 17, 23
WF, NB, BLOCK = 360, 24, 384
NS = [2, 3, 15, 16, 17, 37, 1101]


def sm_count():
  return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def blocks(n):
  """[(g0, rows)] of the query-mode blocks of a call of n pairs"""
  return [(g0, min(BLOCK, n * WF - g0)) for g0 in range(0, n * WF, BLOCK)]


def share_starts(n, sms):
  """first (block, jb) unit of every CTA's contiguous share but the first"""
  units = NB * len(blocks(n))
  parts = min(units, sms)
  return [units * k // parts for k in range(1, parts)]


def straddles(n, b):
  g0, rows = blocks(n)[b]
  return g0 // WF != (g0 + rows - 1) // WF


def test_the_cases_cover_every_block_kind():
  i0 = {g0 % WF for n in NS for g0, _ in blocks(n)}
  assert i0 == set(range(0, WF, NB)), sorted(i0)
  assert any(blocks(n)[-1][1] < BLOCK for n in NS)
  inside = [(n, u) for n in NS for u in share_starts(n, sm_count()) if u % NB and straddles(n, u // NB)]
  assert inside, 'no work share starts inside a block that straddles two pairs'


def stages(eng):
  """o1 and x3 of the last call as int16 bit patterns (both are stored in fp16, so the conversion is exact)"""
  return tuple(eng.heads_stage(s).half().view(torch.int16) for s in ('o1', 'x3'))


def assert_same(a, b, what):
  for x, y, name in zip(a, b, ('o1', 'x3', 'overlap', 'yaw', 'corr')):
    assert x.shape == y.shape, (what, name)
    if not torch.equal(x, y):
      raise AssertionError('%s: %s differs in %d values' % (what, name, int((x != y).sum())))


@pytest.fixture(scope='module')
def setup():
  w = N.glorot_weights(4, MODEL, seed=0)
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=N_BANK)
  bank_np = synth.feature_volumes(11, N_BANK)[:, 0] * np.float32(0.2)
  sel = np.arange(16)
  right_np = np.repeat(bank_np[Q][None, None], len(sel), 0)
  _, _, _, z0 = N.heads_forward(bank_np[sel][:, None], right_np, w, MODEL, return_logit=True)
  eng.load_weights(N.spread_dense(w, z0, target_std=1.5))
  bank = torch.from_numpy(bank_np).to(eng.device)
  yield eng, bank
  eng.close()


def query_and_pair_mode(eng, bank, left):
  """(o1, x3, overlap, yaw, corr) of LEFT = bank[left] against bank[Q], in query mode and in pair mode"""
  n = left.numel()
  out = []
  eng.heads_1vsN(bank, bank[Q_OTHER], cand_idx=left)
  ov, yaw, corr = eng.heads_1vsN(bank, bank[Q], cand_idx=left, want_corr=True)
  out.append(stages(eng) + (ov.clone(), yaw.clone(), corr.clone()))
  eng.heads_1vsN(bank, bank[Q_OTHER], cand_idx=left)
  ov, yaw, corr = eng.heads(bank, left, torch.full((n,), Q, dtype=torch.int32), want_corr=True)
  out.append(stages(eng) + (ov, yaw, corr))
  eng.check()
  return out


@pytest.mark.parametrize('n', NS)
def test_query_mode_matches_pair_mode(setup, n):
  eng, bank = setup
  query, pair = query_and_pair_mode(eng, bank, torch.arange(n, dtype=torch.int32))
  assert_same(query, pair, 'query mode against pair mode, %d pairs' % n)


@pytest.mark.parametrize('n', [37, 1101])
def test_resident_bank_with_permuted_rows(setup, n):
  """LEFT rows come from the resident operand copies through a permuted index list, so the two bulk copies of a
  straddling block read volumes that are not adjacent in the bank"""
  eng, bank = setup
  left = torch.from_numpy(np.random.default_rng(n).permutation(N_BANK)[:n].astype(np.int32))
  assert (left[1:] != left[:-1] + 1).any()
  eng.bank_prepare(bank)
  try:
    query, pair = query_and_pair_mode(eng, bank, left)
  finally:
    eng.bank_release(bank)
  assert_same(query, pair, 'resident bank, permuted rows, %d pairs' % n)
