"""GPU parity of the leg and the two heads through the C ABI against the float64 oracle
(parity unpinned by the reference, see oracle/network.py): overlap within 1e-3 (the tolerance
BASELINE.json's north_star states), yaw equal except on near-ties of the oracle's own scores."""
import numpy as np
import pytest
import torch

from oracle import network as N
from oracle import tc_heads as T
from overlapnet_b200 import synth
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
OVERLAP_TOL = 1e-3          # BASELINE.json north_star: "overlap/yaw floats within 1e-3"
YAW_TIE_REL = 2e-4          # a yaw flip is accepted only if the oracle's two scores differ by less
# Glorot heads give logits that are a near-cancelling sum (|logit| ~ 0.05, std over pairs ~ 0.01,
# sum of |terms| ~ 8): the natural overlaps hug 0.5 and any path passes 1e-3 trivially.  The tests
# therefore rescale the Dense layer so the logits of the test pairs have this standard deviation
# (overlaps spread over ~0.1..0.9), which multiplies every upstream rounding error by the same
# factor (~170x here).  Both precisions are gated at the SAME spread (VERDICT r1): the tensor-core
# path gets there with the feature-centre offset and the hi/lo split of W2 (DESIGN.md section 2); the
# measured maxima are printed (pytest -s).
SPREAD_STD = {'fp32': 1.5, 'f16_tc': 1.5}


def check_yaw(yaw_gpu, yaw_ref, corr_ref, bound=None):
  """A yaw flip is accepted on a near-tie of the oracle's scores: within YAW_TIE_REL of the score range, or, given
  the per-bin bound of the path (oracle/tc_heads.py), within the two bins' bounds."""
  bad = []
  for p in range(len(yaw_ref)):
    if int(yaw_gpu[p]) != int(yaw_ref[p]):
      kg, kr = 180 - int(yaw_gpu[p]), 180 - int(yaw_ref[p])
      gap = corr_ref[p, kr] - corr_ref[p, kg]
      tie = YAW_TIE_REL * np.abs(corr_ref[p]).max() if bound is None else bound[p, kr] + bound[p, kg]
      if gap > tie:
        bad.append((p, int(yaw_gpu[p]), int(yaw_ref[p]), float(gap)))
  assert not bad, bad


@pytest.fixture(scope='module')
def setup():
  w = N.glorot_weights(4, MODEL, seed=0)
  x = synth.range_like_images(1234, 6, 4)
  fv_ref = N.leg_forward(x, w, MODEL)                     # float64 oracle -> float32 (6,1,360,128)
  return w, x, fv_ref


# End-to-end gates of the tensor-core leg, as max |error| / max |volume| against the float64 oracle.  The hi / lo split
# alone costs 1.6e-6 (tests/test_oracle_tc_leg.py); the rest is the tensor cores' truncating fp32 accumulation, which
# errs in one direction and so grows with the length of an accumulation chain: a call of 1-2 scans cuts every layer's
# K walk into 6-36 slices that are added with round-to-nearest (3.2e-6 .. 4.0e-6 measured on an H100 at 700 W), a
# batch walks it in one chain (3.4e-5 .. 3.6e-5 measured; every layer sits at half its per-element bound in
# tests/test_gpu_leg_stages.py, against 0.2-0.4 for the sliced layers).
LEG_TC_TOL_SLICED = 2e-5
LEG_TC_TOL_BATCH = 1e-4


@pytest.mark.parametrize('prec,leg_tol', [('fp32', 2e-5), ('f16_tc', LEG_TC_TOL_BATCH)])
def test_leg_matches_oracle(setup, prec, leg_tol):
  w, x, fv_ref = setup
  eng = Engine(model=MODEL, precision=prec, max_batch_scans=4, max_batch_pairs=16)
  eng.load_weights(w)
  fv = eng.leg(torch.from_numpy(x).to(eng.device)).cpu().numpy()      # 6 scans > max_batch_scans=4
  ref = fv_ref[:, 0]
  err = np.abs(fv - ref).max() / np.abs(ref).max()
  print('\n[parity] leg %s, chunks of 4 and 2 scans: max rel err vs float64 oracle = %.3e' % (prec, err))
  assert err <= leg_tol, err
  assert (fv >= 0).all()
  eng.close()


@pytest.mark.parametrize('prec', ['fp32', 'f16_tc'])
def test_heads_match_oracle(setup, prec):
  w, x, fv_ref = setup
  eng = Engine(model=MODEL, precision=prec, max_batch_scans=4, max_batch_pairs=4)
  eng.load_weights(w)
  bank_np = fv_ref[:, 0].copy()
  # strongly related pairs: LEFT = roll(RIGHT, 37) (+ noise) => yaw = -37 (R = roll(L, s) => yaw = s)
  rng = np.random.default_rng(5)
  bank_np[1] = np.roll(bank_np[5], 37, axis=0) + np.abs(rng.normal(0, 0.01, bank_np[5].shape)).astype(np.float32)
  bank_np[2] = np.roll(bank_np[5], -120, axis=0)
  bank = torch.from_numpy(bank_np).to(eng.device)
  left = np.array([0, 1, 2, 3, 4, 5, 5, 2], np.int32)          # 8 pairs > max_batch_pairs=4
  right = np.array([5, 5, 5, 5, 5, 5, 0, 1], np.int32)
  # rescale the Dense layer so the overlaps of these 8 pairs spread over (0,1): strict 1e-3 check
  _, _, _, z0 = N.heads_forward(bank_np[left][:, None], bank_np[right][:, None], w, MODEL, batch=2, return_logit=True)
  w = N.spread_dense(w, z0, target_std=SPREAD_STD[prec])
  eng.load_weights(w)
  ov_ref, yaw_ref, corr_ref = N.heads_forward(bank_np[left][:, None], bank_np[right][:, None], w, MODEL, batch=2)
  ov, yaw, corr = eng.heads(bank, torch.from_numpy(left), torch.from_numpy(right), want_corr=True)
  ov, yaw, corr = ov.cpu().numpy(), yaw.cpu().numpy(), corr.cpu().numpy()
  print('\n[parity] heads %s @ logit spread %.1f: max |overlap - oracle| = %.3e over %d pairs (overlaps %.2f..%.2f)'
        % (prec, SPREAD_STD[prec], np.abs(ov - ov_ref).max(), len(left), ov_ref.min(), ov_ref.max()))
  assert np.abs(ov - ov_ref).max() <= OVERLAP_TOL, (ov, ov_ref)
  assert ov_ref.max() - ov_ref.min() > 0.25                      # the test is not degenerate
  # f16_tc: the per-bin gate of its hi/lo split correlation (oracle/tc_heads.py, 2.9e-6 of the bin's magnitude: the
  # split's bound plus an empirical allowance for the fp32 accumulation); plain fp16 operands are 1e-5 off and fail it
  bound = np.stack([T.corr_stage(bank_np[a], bank_np[b])[1] for a, b in zip(left, right)]) if prec == 'f16_tc' else None
  check_yaw(yaw, yaw_ref, corr_ref, bound)
  assert yaw_ref[1] == -37 and yaw[1] == -37 and yaw[2] == 120 and yaw[5] == 0 and yaw[7] == 157
  rel = np.abs(corr - corr_ref).max() / np.abs(corr_ref).max()
  if prec == 'fp32':
    assert rel <= 1e-5, rel
  else:
    r = (np.abs(corr - corr_ref) / bound).max()
    print('[parity] heads f16_tc: corr max rel err %.3e, %.3f of the per-bin bound' % (rel, r))
    assert r <= 1.0, (rel, r)
  # 1-vs-N entry point == pair list with RIGHT fixed
  ov1, yaw1, _ = eng.heads_1vsN(bank, bank[5], cand_idx=torch.tensor([0, 1, 2, 3, 4, 5], dtype=torch.int32))
  assert np.array_equal(ov1.cpu().numpy(), ov[:6]) and np.array_equal(yaw1.cpu().numpy(), yaw[:6])
  ov2, yaw2, _ = eng.heads_1vsN(bank, bank[5], n_cand=6)
  assert np.array_equal(ov2.cpu().numpy(), ov[:6]) and np.array_equal(yaw2.cpu().numpy(), yaw[:6])
  # resident bank (ovn_bank_prepare): identical results without the per-call operand conversion
  eng.bank_prepare(bank)
  ov3, yaw3, corr3 = eng.heads(bank, torch.from_numpy(left), torch.from_numpy(right), want_corr=True)
  assert np.array_equal(ov3.cpu().numpy(), ov) and np.array_equal(yaw3.cpu().numpy(), yaw)
  assert np.array_equal(corr3.cpu().numpy(), corr)
  ov4, yaw4, _ = eng.heads_1vsN(bank, bank[5], n_cand=6)
  assert np.array_equal(ov4.cpu().numpy(), ov[:6]) and np.array_equal(yaw4.cpu().numpy(), yaw[:6])
  eng.bank_release(bank)
  eng.close()


@pytest.mark.parametrize('prec', ['fp32', 'f16_tc'])
def test_yaw_shift_known_answer(prec):
  """KAT of the correlation head (NormalizedCorrelation2D.py:112-144, SURVEY 8a row 11):
  R = roll(L, s) along the width  =>  yaw = s  for every s in [-179, 180]."""
  w = N.glorot_weights(4, MODEL, seed=1)
  eng = Engine(model=MODEL, precision=prec, max_batch_scans=1, max_batch_pairs=512)
  eng.load_weights(w)
  base = synth.feature_volumes(3, 1)[0, 0]                       # (360,128), non-negative
  shifts = np.arange(-179, 181)
  bank_np = np.stack([base] + [np.roll(base, s, axis=0) for s in shifts])
  bank = torch.from_numpy(bank_np).to(eng.device)
  n = len(shifts)
  left = torch.zeros(n, dtype=torch.int32)                       # LEFT = base
  right = torch.arange(1, n + 1, dtype=torch.int32)              # RIGHT = rolled
  _, yaw, _ = eng.heads(bank, left, right)
  assert np.array_equal(yaw.cpu().numpy(), shifts)
  eng.close()


@pytest.mark.parametrize('channels,use', [(5, {'use_intensity': True}),
                                          (25, {'use_intensity': True, 'use_class_probabilities': True})])
def test_leg_other_channel_counts(channels, use):
  w = N.glorot_weights(channels, MODEL, seed=2)
  x = synth.range_like_images(7, 2, channels)
  ref = N.leg_forward(x, w, MODEL)[:, 0]
  for prec, tol in (('fp32', 2e-5), ('f16_tc', LEG_TC_TOL_SLICED)):
    eng = Engine(use=use, model=MODEL, precision=prec, max_batch_scans=2, max_batch_pairs=1)
    assert eng.C == channels
    eng.load_weights(w)
    fv = eng.leg(torch.from_numpy(x).to(eng.device)).cpu().numpy()
    err = np.abs(fv - ref).max() / np.abs(ref).max()
    print('\n[parity] leg %s C=%d, 2 scans: max rel err vs float64 oracle = %.3e' % (prec, channels, err))
    assert err <= tol, err
    eng.close()


@pytest.mark.parametrize('channels,use', [(5, {'use_intensity': True}),
                                          (25, {'use_intensity': True, 'use_class_probabilities': True})])
def test_batched_leg_other_channel_counts(channels, use):
  """Batches of more than two scans take the batched layer-1 kernel: fp32-grade against the float64
  oracle, and the same volumes as the one-scan-at-a-time path."""
  w = N.glorot_weights(channels, MODEL, seed=3)
  x = synth.range_like_images(9, 5, channels)
  ref = N.leg_forward(x, w, MODEL)[:, 0]
  scale = np.abs(ref).max()
  eng = Engine(use=use, model=MODEL, precision='f16_tc', max_batch_scans=5, max_batch_pairs=1)
  eng1 = Engine(use=use, model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=1)
  eng.load_weights(w); eng1.load_weights(w)
  xt = torch.from_numpy(x).to(eng.device)
  a = eng.leg(xt)
  assert torch.equal(eng.leg(xt), a)
  err = np.abs(a.cpu().numpy() - ref).max() / scale
  print('\n[parity] batched leg C=%d: max rel err vs float64 oracle = %.3e' % (channels, err))
  assert err <= 1e-4
  assert (a - eng1.leg(xt)).abs().max().item() / scale <= 1e-4
  eng.check()
  eng.close(); eng1.close()


def test_full_size_1xN_properties():
  """BASELINE config 2 size (1 query x 1101 candidates) through the product path: results are
  independent of candidate order / chunking, equal to the pairwise entry point, the query
  against itself gives yaw 0, and 68 of the 1101 pairs (64 random + 4 fixed) agree with the
  float64 oracle within 1e-3 at the same logit spread as the fp32 path (1.5)."""
  w = N.glorot_weights(4, MODEL, seed=0)
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=1101)
  n = 1101
  bank_np = synth.feature_volumes(11, n)[:, 0] * np.float32(0.2)
  sel = np.unique(np.concatenate([np.array([0, 17, 500, 1100]),
                                  np.random.default_rng(2).choice(n, 64, replace=False)]))
  right_np = np.repeat(bank_np[17][None, None], len(sel), 0)
  _, _, _, z0 = N.heads_forward(bank_np[sel][:, None], right_np, w, MODEL, return_logit=True)
  w = N.spread_dense(w, z0, target_std=SPREAD_STD['f16_tc'])
  eng.load_weights(w)
  bank = torch.from_numpy(bank_np).to(eng.device)
  q = bank[17].clone()
  ov, yaw, _ = eng.heads_1vsN(bank, q, n_cand=n)
  perm = torch.randperm(n, generator=torch.Generator().manual_seed(0)).to(torch.int32)
  ovp, yawp, _ = eng.heads_1vsN(bank, q, cand_idx=perm)
  assert torch.equal(ov[perm.long().to(eng.device)], ovp) and torch.equal(yaw[perm.long().to(eng.device)], yawp)
  eng.check()
  assert int(yaw[17]) == 0
  assert torch.isfinite(ov).all() and (ov >= 0).all() and (ov <= 1).all()
  ov_ref, yaw_ref, corr_ref = N.heads_forward(bank_np[sel][:, None], right_np, w, MODEL)
  err = np.abs(ov.cpu().numpy()[sel] - ov_ref)
  print('\n[parity] 1 x 1101 f16_tc @ logit spread %.1f: max |overlap - oracle| = %.3e, rms %.3e over %d pairs '
        '(overlaps %.2f..%.2f)' % (SPREAD_STD['f16_tc'], err.max(), np.sqrt((err ** 2).mean()), len(sel),
                                  ov_ref.min(), ov_ref.max()))
  assert err.max() <= OVERLAP_TOL
  assert ov_ref.max() - ov_ref.min() > 0.5
  check_yaw(yaw.cpu().numpy()[sel], yaw_ref, corr_ref)
  eng.close()


def test_feature_center_is_calibrated_once_and_settable():
  """The per-channel centre of the fp16 operand copies: calibrated on the first volumes seen, frozen,
  readable, settable; any centre gives the same answer within the gate (|l - r| is offset-invariant)."""
  w = N.glorot_weights(4, MODEL, seed=0)
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=8)
  eng.load_weights(w)
  mu, is_set = eng.get_feature_center()
  assert not is_set and not mu.any()
  bank_np = synth.feature_volumes(5, 6)[:, 0] + np.float32(0.5)
  bank = torch.from_numpy(bank_np).to(eng.device)
  ov1, yaw1, _ = eng.heads_1vsN(bank, bank[2], n_cand=6)
  mu, is_set = eng.get_feature_center()
  assert is_set
  want = bank_np[2].astype(np.float64).mean(0)                    # calibrated on the RIGHT volume of the first call
  assert np.abs(mu - want).max() <= 1e-3 * np.abs(want).max() + 1e-6
  assert np.array_equal(mu, mu.astype(np.float16).astype(np.float32))
  ov2, _, _ = eng.heads_1vsN(bank, bank[3], n_cand=6)             # frozen: a second query does not move it
  assert np.array_equal(eng.get_feature_center()[0], mu)
  eng.set_feature_center(np.zeros(128, np.float32))               # explicit centre 0 = the round-1 operands
  ov0, yaw0, _ = eng.heads_1vsN(bank, bank[2], n_cand=6)
  assert np.abs(ov0.cpu().numpy() - ov1.cpu().numpy()).max() <= 1e-3
  assert torch.equal(yaw0, yaw1)
  eng.bank_prepare(bank)
  with pytest.raises(Exception, match='release the resident bank'):
    eng.set_feature_center(np.ones(128, np.float32))
  eng.bank_release(bank)
  eng.set_feature_center(None)
  assert not eng.get_feature_center()[1]
  eng.close()


def test_tc_precision_rejects_other_head_geometry():
  """precision f16_tc is specialised to leg_output_width 360 / conv1size 15 (config/network.yml); any
  other geometry must fail loudly at load time (and works with precision fp32)."""
  model = dict(MODEL, conv1NetworkHead_conv1size=12)
  w = N.glorot_weights(4, model, seed=0)
  eng = Engine(model=model, precision='f16_tc', max_batch_scans=1, max_batch_pairs=2)
  with pytest.raises(Exception, match='supports leg_output_width=360, conv1size=15 only'):
    eng.load_weights(w)
  eng.close()
  eng = Engine(model=model, precision='fp32', max_batch_scans=1, max_batch_pairs=2)
  eng.load_weights(w)
  eng.close()


def test_single_scan_leg_is_bit_reproducible_and_matches_batched():
  """The tensor-core leg uses no floating-point atomics: repeated runs are bit-identical, and one scan
  per launch agrees with six scans per launch within the leg tolerance."""
  w = N.glorot_weights(4, MODEL, seed=4)
  x = synth.range_like_images(21, 6, 4)
  eng1 = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=1)     # one scan per launch
  eng6 = Engine(model=MODEL, precision='f16_tc', max_batch_scans=6, max_batch_pairs=1)     # all six in one launch
  eng1.load_weights(w); eng6.load_weights(w)
  xt = torch.from_numpy(x).to(eng1.device)
  a = eng1.leg(xt)
  for _ in range(3):
    assert torch.equal(eng1.leg(xt), a)
  b = eng6.leg(xt)
  ref = N.leg_forward(x, w, MODEL)[:, 0]
  scale = np.abs(ref).max()
  err1, err6 = (np.abs(t.cpu().numpy() - ref).max() / scale for t in (a, b))
  print('\n[parity] leg f16_tc: max rel err vs float64 oracle, one scan per call %.3e, six %.3e' % (err1, err6))
  assert err1 <= LEG_TC_TOL_SLICED and err6 <= LEG_TC_TOL_BATCH, (err1, err6)
  assert (a - b).abs().max().item() / scale <= 1e-4
  eng1.close(); eng6.close()


def test_batched_leg_matches_oracle_and_single_scan_path():
  """A batch of 20 scans through the tensor-core leg against the float64 oracle and against the same
  scans encoded one at a time."""
  w = N.glorot_weights(4, MODEL, seed=6)
  x = synth.range_like_images(31, 20, 4)
  ref = N.leg_forward(x, w, MODEL)[:, 0]
  scale = np.abs(ref).max()
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=20, max_batch_pairs=1)
  eng1 = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=1)
  eng.load_weights(w); eng1.load_weights(w)
  xt = torch.from_numpy(x).to(eng.device)
  a = eng.leg(xt)
  b = eng1.leg(xt)
  assert torch.equal(eng.leg(xt), a)                                   # bit-reproducible
  err = np.abs(a.cpu().numpy() - ref).max() / scale
  print('\n[parity] batched leg f16_tc (hi/lo split operands): max rel err vs float64 oracle = %.3e' % err)
  assert err <= 1e-4
  assert (a - b).abs().max().item() / scale <= 1e-4
  eng.close(); eng1.close()


def test_pair_chunk_larger_than_grid_y_limit():
  """A chunk of 3000 pairs (more than 65535 / 24 work units of the delta kernel on a grid's y axis) gives
  exactly the results of the same pairs in chunks of 1000."""
  w = N.glorot_weights(4, MODEL, seed=0)
  src = torch.from_numpy(synth.feature_volumes(13, 8)[:, 0])
  n = 3000
  out = []
  for maxp in (n, 1000):
    eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=maxp)
    eng.load_weights(w)
    s = src.to(eng.device)
    bank = torch.stack([torch.roll(s[i % 8], i // 8, 0) for i in range(n)])
    ov, yaw, _ = eng.heads_1vsN(bank, bank[1], n_cand=n)
    eng.check()
    out.append((ov, yaw))
    eng.close()
  assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
  assert int(out[0][1][1]) == 0 and torch.isfinite(out[0][0]).all()
