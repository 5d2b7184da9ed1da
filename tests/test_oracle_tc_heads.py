"""The float64 stage model of the tensor-core heads (oracle/tc_heads.py) against the float64 oracle, and the
sensitivity of its bounds: with the fp16 roundings off the stages chain to oracle.network exactly; with them on
the o1 stage agrees with delta_conv1_naive within the fp16 input roundings; and errors that a wrong row, lane or
operand term would make in the kernels exceed the bounds by far."""
import numpy as np
import pytest

from oracle import network as N
from oracle import tc_heads as T
from overlapnet_b200 import synth

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}


@pytest.fixture(scope='module')
def pair():
  w = N.glorot_weights(4, MODEL, seed=0)
  v = synth.feature_volumes(11, 3)[:, 0] * np.float32(0.2)
  return w, v


def rel(a, b):
  return np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-300)


def test_stages_without_rounding_chain_to_the_oracle(pair):
  w, v = pair
  l, r = v[1], v[0]
  rng = np.random.default_rng(3)
  mu = v[0].astype(np.float64).mean(0)
  mu_o1 = rng.normal(0, 0.1, 64)
  mu_x3 = np.abs(rng.normal(0, 0.1, 128))
  acts, z, out = N.delta_head(l[None, None], r[None, None], w, MODEL, return_all=True)
  o1, _ = T.o1_stage(l, r, mu, w['c_conv1'][0], mu_o1, rounding=False)
  assert rel(o1 + w['c_conv1'][1] + mu_o1, acts[0][0]) <= 1e-12
  b2eff, _ = T.b2eff_model(w, mu_o1)
  x3, _, _ = T.x3_stage(o1, w['c_conv2'][0], b2eff, mu_x3, rounding=False)
  assert rel(x3 + mu_x3, acts[1][0]) <= 1e-12
  b3eff, _ = T.b3eff_model(w, mu_x3)
  part, _ = T.dense_stage(x3, w['c_conv3'][0], b3eff, w['overlap_output'][0], rounding=False)
  wd = w['overlap_output'][0].astype(np.float64).reshape(22, 22, 2, 128)
  want = (acts[2][0].reshape(22, 22, 2, 128) * wd).sum(-1)
  assert rel(part[:22, :22], want) <= 1e-12 and not part[22:].any() and not part[:, 22:].any()
  ov, _ = T.overlap_stage(part, w['overlap_output'][1])
  assert abs(part.sum() + w['overlap_output'][1][0] - z[0, 0]) <= 1e-12 * np.abs(part).sum()
  assert abs(ov - out[0, 0]) <= 1e-12
  corr, _ = T.corr_stage(l, r)
  assert rel(corr, N.correlation_naive(l, r)) <= 1e-12


def test_rounded_o1_agrees_with_delta_conv1_naive_on_small_slices(pair):
  """Volumes of 45 columns (3 column blocks): the modelled fp16 operands, differences and weights stay within their
  roundings of the exact c_conv1 (without its bias, minus the o1 centre)."""
  w, v = pair
  k1, b1 = w['c_conv1']
  mu = T.h(v[0].astype(np.float64).mean(0))
  mu_o1 = T.h(np.random.default_rng(4).normal(0, 0.1, 64))
  for rows in (slice(0, 45), slice(300, 345)):
    l, r = v[1][rows], np.roll(v[2], 7, axis=0)[rows]
    model, tol = T.o1_stage(l, r, mu, k1, mu_o1)
    exact = N.delta_conv1_naive(l, r, k1, b1, 15) - b1 - mu_o1
    a = np.abs(l.astype(np.float64) - mu)
    b = np.abs(r.astype(np.float64) - mu)
    W = np.abs(k1[0].astype(np.float64))
    # sum_{dj, c} (|l - mu| + |r - mu|) |W1|: what the roundings of the operands, of |l - r| and of W1 act on
    mag = np.stack([np.einsum('ic,dco->io', a, W) + np.einsum('dc,dco->o', b[15 * jb:15 * jb + 15], W)[None]
                    for jb in range(3)], 1)
    bound = 2.0 ** -9 * mag + tol + T.ulp16(np.abs(mu_o1))
    assert (np.abs(model - exact) <= bound).all()
    assert np.abs(model - exact).max() > 0                        # the roundings are modelled, not skipped


def o1_setup(pair):
  w, v = pair
  mu, mu_o1, _ = T.calibrate(v[0], w)
  l, r = v[1], v[0]
  model, tol = T.o1_stage(l, r, mu, w['c_conv1'][0], mu_o1)
  W = T.h(w['c_conv1'][0][0])                                       # (15, 128, 64)
  L, R = T.operand(l, mu), T.operand(r, mu)
  return w, v, mu, model, tol, W, L, R


def test_o1_bound_catches_one_missing_slice_of_a_fragment_half(pair):
  """Rows 352-359 of column block 23 (one 8-row half of an MMA fragment) lose one 32-channel W1 slice."""
  _, _, _, model, tol, W, L, R = o1_setup(pair)
  d = T.h(np.abs(L[352:360, None, :32] - R[None, 15 * 23, :32]))    # (8, 1, 32): dj 0, channels 0..31
  lost = np.einsum('ic,co->io', d[:, 0], W[0, :32])
  ratio = (np.abs(lost) / tol[352:360, 23]).max()
  print('\n[tc_heads] missing slice: o1 off by %.1f %% of max|o1|, %.0fx its bound'
        % (100 * np.abs(lost).max() / np.abs(model).max(), ratio))
  assert ratio >= 100


def test_o1_bound_catches_a_stale_right_row(pair):
  """Row 0 of column block 0 reads, for dj 0, the RIGHT row the previous work unit left (another volume's row 345)."""
  _, v, mu, model, tol, W, L, R = o1_setup(pair)
  stale = T.operand(v[2], mu)[345]
  good = T.h(np.abs(L[0] - R[0]))
  bad = T.h(np.abs(L[0] - stale))
  delta = (bad - good) @ W[0]
  ratio = (np.abs(delta) / tol[0, 0]).max()
  print('\n[tc_heads] stale RIGHT row: o1 off by %.1f %% of max|o1|, %.0fx its bound'
        % (100 * np.abs(delta).max() / np.abs(model).max(), ratio))
  assert ratio >= 100


@pytest.mark.parametrize('terms', [('hh',), ('hh', 'hl')])
def test_corr_bound_catches_missing_lo_terms(pair, terms):
  _, v = pair
  for p in (1, 2):
    exact, bound = T.corr_stage(v[p], v[0])
    full = T.corr_split(v[p], v[0])
    assert (np.abs(full - exact) <= 0.1 * bound).all()
    cut = T.corr_split(v[p], v[0], terms)
    ratio = (np.abs(cut - exact) / bound).max()
    print('\n[tc_heads] corr with %s only: %.1fx the bound' % ('+'.join(terms), ratio))
    assert ratio > 1.5


def test_corr_bound_has_an_absolute_term_for_subnormal_lo():
  """Scaled by 2^-12 the lo halves are subnormal: the split is worse than 2^-22 relative, the bound still holds."""
  v = synth.feature_volumes(11, 2)[:, 0] * np.float32(0.2 * 2.0 ** -12)
  exact, bound = T.corr_stage(v[1], v[0])
  err = np.abs(T.corr_split(v[1], v[0]) - exact)
  assert (err <= bound).all()
  A = T.correlation(np.abs(v[1]), np.abs(v[0]))
  assert (err / A).max() > 2.0 ** -22


def test_fp16_helpers():
  assert T.h(np.array([2.0 ** -25, 3 * 2.0 ** -26, 65519.0, 1 + 2.0 ** -11]))[:3].tolist() == [0.0, 2.0 ** -24, 65504.0]
  assert T.h(np.array([1 + 2.0 ** -11]))[0] == 1.0                    # ties to even
  assert T.ulp16(np.array([0.0, 1.0, 1.5, -2.0])).tolist() == [2.0 ** -24, 2.0 ** -10, 2.0 ** -10, 2.0 ** -9]
