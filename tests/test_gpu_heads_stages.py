"""Every stage of the tensor-core heads against the float64 stage model (oracle/tc_heads.py), at the pairs where
the persistent kernels' work shares start and end.

k_delta_conv1_wgmma, k_conv2_wgmma, k_conv3_wgmma and k_corr_wgmma each give a CTA a contiguous share of work
units, and a share may start or end inside a pair.  For each case the pairs that hold a share boundary of any of the
four kernels are restated from the device's SM count; the first pair, the last pair and up to 22 boundary pairs are
checked at every stage: o1, x3, b2eff / b3eff, the Dense partials, the overlap and the correlation, each from the
GPU's own input to that stage (Engine.heads_stage).  `pytest -s` prints the largest error-to-bound ratio of each
stage."""
import math

import numpy as np
import pytest
import torch

from oracle import network as N
from oracle import tc_heads as T
from overlapnet_b200 import synth
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
MAX_CHECKED = 24
INT32_MIN = -2 ** 31


@pytest.fixture(scope='module')
def weights():
  return N.glorot_weights(4, MODEL, seed=0)


@pytest.fixture(scope='module')
def bank_np(weights):
  """40 synthetic volumes, 6 rolled copies of them and two real leg outputs."""
  v = synth.feature_volumes(11, 40)[:, 0] * np.float32(0.2)
  rolled = np.stack([np.roll(v[k], s, axis=0) for k, s in zip(range(6), (1, 37, -120, 180, 15, -1))])
  legs = N.leg_forward(synth.range_like_images(1234, 2, 4), weights, MODEL)[:, 0]
  return np.ascontiguousarray(np.concatenate([v, rolled, legs]), np.float32)


def sm_count():
  return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def boundary_pairs(n, sms):
  """Pairs that hold a work-share boundary of one of the four persistent kernels of a call of n pairs."""
  rows = 576 * n
  tiles = math.ceil(rows / 256)
  out = set()

  def shares(units, parts):
    return [units * k // parts for k in range(1, parts)]

  for u in shares(24 * n, min(24 * n, sms)):                   # delta: (pair, jb) units
    out.update({u // 24, (u - 1) // 24})
  for t in shares(tiles, min(tiles, sms)):                     # c_conv2: 256-row tiles
    out.update({256 * t // 576, (256 * t - 1) // 576})
  for u in shares(2 * tiles, min(2 * tiles, sms)):             # c_conv3: (tile, channel half) units
    t = u // 2
    out.update({256 * t // 576, (min(256 * t + 255, rows - 1)) // 576, (256 * t - 1) // 576})
  for u in shares(6 * n, min(6 * n, sms // 3)):                # correlation: (pair, LEFT tile) units
    out.update({u // 6, (u - 1) // 6})
  return sorted(p for p in out if 0 <= p < n)


def checked_pairs(n):
  b = [p for p in boundary_pairs(n, sm_count()) if p not in (0, n - 1)]
  if len(b) > MAX_CHECKED - 2:
    b = [b[i] for i in np.linspace(0, len(b) - 1, MAX_CHECKED - 2).round().astype(int)]
  return sorted(set([0, n - 1] + b))


def ratio(gpu, model, tol):
  return float((np.abs(np.asarray(gpu, np.float64) - model) / tol).max())


def check_stages(eng, w, lefts, rights, sel, ov, yaw, corr, label):
  """lefts / rights: {pair: float32 volume}.  Asserts every stage of the pairs in sel within its bound."""
  assert eng.heads_stage_pairs() == len(ov)
  # one pair per copy: the read-back stays small (o1 is 2.2 MB per pair)
  o1, x3, dense = ([eng.heads_stage(st, p, 1)[0].cpu().numpy() for p in sel] for st in ('o1', 'x3', 'dense'))
  cen = eng.heads_stage('centres').cpu().numpy()
  ov, yaw, corr = ov.cpu().numpy(), yaw.cpu().numpy(), corr.cpu().numpy()
  mu, is_set = eng.get_feature_center()
  assert is_set
  mu_o1, mu_x3, b2eff, b3eff = cen[:64], cen[64:192], cen[192:320], cen[320:]
  r = {}
  m, t = T.b2eff_model(w, mu_o1)
  r['b2eff'] = ratio(b2eff, m, t)
  m, t = T.b3eff_model(w, mu_x3)
  r['b3eff'] = ratio(b3eff, m, t)
  kink = 0
  for k, p in enumerate(sel):
    l, rt = lefts[p], rights[p]
    m, t = T.o1_stage(l, rt, mu, w['c_conv1'][0], mu_o1)
    r['o1'] = max(r.get('o1', 0), ratio(o1[k], m, t))
    m, t, nk = T.x3_stage(o1[k], w['c_conv2'][0], b2eff, mu_x3)
    kink += nk
    r['x3'] = max(r.get('x3', 0), ratio(x3[k], m, t))
    m, t = T.dense_stage(x3[k], w['c_conv3'][0], b3eff, w['overlap_output'][0])
    valid = t > 0
    assert (dense[k][~valid] == 0).all(), (label, p)                # rows c_conv3 does not produce
    r['dense'] = max(r.get('dense', 0), ratio(dense[k][valid], m[valid], t[valid]))
    m, t = T.overlap_stage(dense[k], w['overlap_output'][1])
    r['overlap'] = max(r.get('overlap', 0), abs(float(ov[p]) - m) / t)
    exact, bound = T.corr_stage(l, rt)
    r['corr'] = max(r.get('corr', 0), ratio(corr[p], exact, bound))
    best = int(np.argmax(corr[p]))                                  # first maximum, as k_corr_finalize
    assert int(yaw[p]) == 180 - best, (label, p)
    want = int(np.argmax(exact))
    assert best == want or exact[want] - exact[best] <= bound[want] + bound[best], (label, p, best, want)
  print('\n[stages] %-28s %3d of %4d pairs checked, error / bound: %s; x3 within its bound of the ReLU kink: %d'
        % (label, len(sel), len(ov), ', '.join('%s %.3f' % kv for kv in r.items()), kink))
  for stage, v in r.items():
    assert v <= 1.0, (label, stage, v)
  return r


def engine(w, n, calib):
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=n)
  eng.load_weights(w)
  eng.calibrate(calib)
  return eng


def pairs(n, n_bank, seed):
  rng = np.random.default_rng(seed)
  left = rng.integers(0, n_bank, n).astype(np.int32)
  right = rng.integers(0, n_bank, n).astype(np.int32)
  left[0], right[-1] = n_bank - 1, n_bank - 2                       # the two leg outputs
  return left, right


@pytest.mark.parametrize('n', [1, 5, 6, 37, 300])
def test_pair_mode(weights, bank_np, n):
  eng = engine(weights, n, torch.from_numpy(bank_np[0]))
  bank = torch.from_numpy(bank_np).to(eng.device)
  left, right = pairs(n, len(bank_np), n)
  ov, yaw, corr = eng.heads(bank, torch.from_numpy(left), torch.from_numpy(right), want_corr=True)
  sel = checked_pairs(n)
  check_stages(eng, weights, {p: bank_np[left[p]] for p in sel}, {p: bank_np[right[p]] for p in sel}, sel,
               ov, yaw, corr, 'pair mode, n = %d' % n)
  eng.check()
  eng.close()


@pytest.mark.parametrize('n', [7, 1101])
def test_query_mode(weights, bank_np, n):
  eng = engine(weights, n, torch.from_numpy(bank_np[3]))
  bank = torch.from_numpy(bank_np).to(eng.device)
  cand = np.random.default_rng(n).integers(0, len(bank_np), n).astype(np.int32)
  q = len(bank_np) - 1
  ov, yaw, corr = eng.heads_1vsN(bank, bank[q], cand_idx=torch.from_numpy(cand), want_corr=True)
  sel = checked_pairs(n)
  check_stages(eng, weights, {p: bank_np[cand[p]] for p in sel}, {p: bank_np[q] for p in sel}, sel,
               ov, yaw, corr, 'query mode, n = %d' % n)
  eng.check()
  eng.close()


def test_resident_bank_pair_mode(weights, bank_np):
  """LEFT from the resident operand copies (ovn_bank_prepare): a permutation of the bank with repeats, and some
  pairs with LEFT == RIGHT."""
  n = 37
  eng = engine(weights, n, torch.from_numpy(bank_np[0]))
  bank = torch.from_numpy(bank_np).to(eng.device)
  eng.bank_prepare(bank)
  rng = np.random.default_rng(7)
  left = np.concatenate([rng.permutation(len(bank_np))[:30], [5, 5, 47, 47, 12, 0, 0]]).astype(np.int32)
  right = rng.integers(0, len(bank_np), n).astype(np.int32)
  right[[3, 17, 31, 36]] = left[[3, 17, 31, 36]]
  ov, yaw, corr = eng.heads(bank, torch.from_numpy(left), torch.from_numpy(right), want_corr=True)
  sel = sorted(set(checked_pairs(n)) | {3, 17, 31})[:MAX_CHECKED]
  check_stages(eng, weights, {p: bank_np[left[p]] for p in sel}, {p: bank_np[right[p]] for p in sel}, sel,
               ov, yaw, corr, 'resident bank, n = %d' % n)
  for p in (3, 17, 31, 36):
    assert int(yaw[p]) == 0
  eng.check()
  eng.bank_release(bank)
  eng.close()


def test_stale_buffers_do_not_reach_a_smaller_call(weights, bank_np):
  """A handle that scored 300 pairs, then 37, gives the stages and outputs of a fresh handle on the 37 pairs, bit for
  bit: nothing of the larger call's o1, x3 or partials is read."""
  calib = torch.from_numpy(bank_np[2])
  big = engine(weights, 300, calib)
  bank = torch.from_numpy(bank_np).to(big.device)
  l3, r3 = pairs(300, len(bank_np), 11)
  big.heads(bank, torch.from_numpy(l3), torch.from_numpy(r3))
  left, right = pairs(37, len(bank_np), 12)
  outs = []
  engines = (big, engine(weights, 37, calib))
  for eng in engines:
    res = eng.heads(bank, torch.from_numpy(left), torch.from_numpy(right), want_corr=True)
    outs.append(list(res) + [eng.heads_stage(s) for s in ('o1', 'x3', 'dense', 'centres')])
    eng.check()
  for a, b, name in zip(*outs, ('overlap', 'yaw', 'corr', 'o1', 'x3', 'dense', 'centres')):
    assert torch.equal(a, b), name
  for eng in engines:
    eng.close()


@pytest.mark.parametrize('scale', [2.0 ** -12, 2.0 ** 6])
def test_subnormal_and_large_operands(weights, bank_np, scale):
  """Volumes x 2^-12 (|l - r| and the correlation's lo halves subnormal in fp16) and x 2^6, with W1 scaled by the
  inverse: the model gates only (fp16 rounds differently at each scale)."""
  w = dict(weights)
  w['c_conv1'] = ((weights['c_conv1'][0].astype(np.float64) / scale).astype(np.float32), weights['c_conv1'][1])
  b = np.ascontiguousarray(bank_np[:40] * np.float32(scale))
  n = 6
  eng = engine(w, n, torch.from_numpy(b[0]))
  bank = torch.from_numpy(b).to(eng.device)
  left, right = pairs(n, len(b), 20)
  ov, yaw, corr = eng.heads(bank, torch.from_numpy(left), torch.from_numpy(right), want_corr=True)
  sel = list(range(n))
  check_stages(eng, w, {p: b[left[p]] for p in sel}, {p: b[right[p]] for p in sel}, sel, ov, yaw, corr,
               'volumes x 2^%d' % round(math.log2(scale)))
  eng.check()
  eng.close()


@pytest.mark.parametrize('bad', [7e4, float('nan')])
def test_values_outside_fp16_poison_the_outputs(weights, bank_np, bad):
  """A volume value fp16 cannot hold (beyond 65504, NaN) must not give a plausible overlap or yaw: as a LEFT or a
  RIGHT operand, both outputs are poisoned and check() raises; the handle then works again."""
  eng = engine(weights, 2, torch.from_numpy(bank_np[0]))
  b = bank_np[:4].copy()
  b[1, 100, 7] = bad
  bank = torch.from_numpy(b).to(eng.device)
  clean = torch.from_numpy(bank_np[:4]).to(eng.device)
  for left, right in (([1, 0], [2, 3]), ([0, 2], [3, 1])):
    left, right = torch.tensor(left, dtype=torch.int32), torch.tensor(right, dtype=torch.int32)
    ov, yaw, _ = eng.heads(bank, left, right)
    assert torch.isnan(ov).all() and (yaw == INT32_MIN).all(), (ov, yaw)
    with pytest.raises(Exception, match='not finite'):
      eng.check()
    ov, yaw, _ = eng.heads(clean, left, right)
    eng.check()
    assert torch.isfinite(ov).all() and (yaw != INT32_MIN).all()
  eng.close()


@pytest.mark.parametrize('bad', [7e4, float('nan')])
def test_resident_row_outside_fp16_poisons_every_call_that_reads_it(weights, bank_np, bad):
  """A resident bank row with a value fp16 cannot hold is marked by bank_prepare: every heads call that reads it (as
  LEFT, through the resident copies only) is poisoned and check() raises, a call that does not read it is not, and
  the mark goes when the row is prepared again with finite values."""
  eng = engine(weights, 2, torch.from_numpy(bank_np[0]))
  b = bank_np[:4].copy()
  b[1, 100, 7] = bad
  bank = torch.from_numpy(b).to(eng.device)
  eng.bank_prepare(bank)
  eng.check()                                                      # preparing the row raises nothing by itself
  reads = torch.tensor([1, 0], dtype=torch.int32), torch.tensor([2, 3], dtype=torch.int32)
  other = torch.tensor([0, 2], dtype=torch.int32), torch.tensor([2, 3], dtype=torch.int32)
  ov, yaw, _ = eng.heads(bank, *other)
  eng.check()
  assert torch.isfinite(ov).all() and (yaw != INT32_MIN).all()
  for _ in range(2):                                               # the mark outlives a check()
    ov, yaw, _ = eng.heads(bank, *reads)
    assert torch.isnan(ov).all() and (yaw == INT32_MIN).all(), (ov, yaw)
    with pytest.raises(Exception, match='not finite'):
      eng.check()
  bank[1] = torch.from_numpy(bank_np[1]).to(eng.device)
  eng.bank_prepare(bank, first=1, count=1)
  ov, yaw, _ = eng.heads(bank, *reads)
  eng.check()
  assert torch.isfinite(ov).all() and (yaw != INT32_MIN).all()
  eng.bank_release(bank)
  eng.close()


def test_stage_copy_is_bounded_by_the_stored_pairs(weights, bank_np):
  """The stage copy writes only a range of the pairs the handle holds, whichever entry point ran the heads."""
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=8)
  eng.load_weights(weights)
  assert eng.heads_stage_pairs() == 0
  with pytest.raises(Exception, match='no stored stages'):
    eng.heads_stage('o1', 0, 1)
  bank = torch.from_numpy(bank_np[:8]).to(eng.device)
  idx = torch.arange(5, dtype=torch.int32)
  eng.heads(bank, idx, idx.flip(0))
  assert eng.heads_stage_pairs() == 5
  assert eng.heads_stage('x3').shape == (5, 24, 24, 128)
  with pytest.raises(Exception, match='outside the 5 stored'):
    eng.heads_stage('o1', 4, 2)
  eng.heads_1vsN(bank, bank[0], cand_idx=torch.arange(19, dtype=torch.int32) % 8)   # chunks of 8, 8 and 3 pairs
  assert eng.heads_stage_pairs() == 3
  eng.query_cloud_vs_bank_host(synth.kitti_like_cloud(5), bank, n_cand=7)
  assert eng.heads_stage_pairs() == 7
  assert torch.equal(eng.heads_stage('dense', 6, 1)[0], eng.heads_stage('dense')[6])
  eng.calibrate(bank[2])                                            # overwrites o1 and x3
  assert eng.heads_stage_pairs() == 0
  eng.check()
  eng.close()
  eng = Engine(model=MODEL, precision='fp32', max_batch_scans=1, max_batch_pairs=2)
  eng.load_weights(weights)
  with pytest.raises(Exception, match='OVN_ERR_BAD_CONFIG'):
    eng.heads_stage('centres')
  eng.close()
