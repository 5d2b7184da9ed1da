"""The float64 layer model of the tensor-core leg (oracle/tc_leg.py) against the float64 oracle, and the sensitivity
of its bounds: with the fp16 roundings off the layers chain to oracle.network.leg_forward exactly; five wrong
products a kernel defect would make differ from the true model by more than the bound, on a stated fraction of
elements, in every k_leg_mma layer; and the model fed with its own outputs gives the end-to-end error the design
expects of the hi / lo split, which the end-to-end tolerances of the GPU tests rest on."""
import numpy as np
import pytest

from oracle import network as N
from oracle import tc_leg as T
from overlapnet_b200 import synth

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
SMS = 132                                          # H100 SXM: the slice counts of a single scan follow the SM count

# The wrong products: what a kernel defect would compute in place of xh wh + xl wh + xh wl
MUTANTS = {'xl wh dropped': dict(terms=('hh', 'hl')),
           'xh wl dropped': dict(terms=('hh', 'lh')),
           'plain h(x) h(w)': dict(terms=('hh',)),
           'tap dw off by one': dict(dw_shift=1),
           'last K slice omitted': dict(drop_last_slice=True)}
# Least fraction of a layer's elements that must differ from the true model by more than its bound.  About half of
# the elements of a layer are clamped by the ReLU in the model and in the mutant alike; nearly every other one tells.
MIN_FRACTION = 0.35


def rel(a, b):
  return np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize('use3a', [True, False])
@pytest.mark.parametrize('C', [4, 25])
def test_layers_without_rounding_chain_to_the_oracle(C, use3a):
  model = dict(MODEL, additional_unsymmetric_layer3a=use3a)
  w = N.glorot_weights(C, model, seed=1)
  x = synth.range_like_images(3, 1, C)
  specs = T.layer_specs(C, model)
  assert [s['name'] for s in specs] == [r[0] for r in N.leg_layers(model)] and len(specs) == (11 if use3a else 10)
  ref = N.leg_forward(x, w, model, return_all=True)
  got = T.forward(x[0], w, specs, rounding=False)
  for spec, a, b in zip(specs, got, ref):
    assert a.shape == b[0].shape == (spec['h_out'], spec['w_out'], spec['cout'])
    assert rel(a, b[0]) <= 1e-12, spec['name']
  # K slices change the order of an exact sum only
  sl = T.forward(x[0], w, specs, [1] + [T.leg_split(s, 1, SMS) for s in specs[1:]], rounding=False)
  assert rel(sl[-1], ref[-1][0]) <= 1e-12


def test_leg_split_restates_the_kernel_choice():
  """Single scans and pairs of scans are K-sliced (at least 4 iterations per slice), batches are not."""
  specs = T.layer_specs(4, MODEL)
  assert [T.leg_split(s, 1, SMS) for s in specs[1:]] == [6, 13, 36, 18, 18, 18, 18, 14, 10, 6]
  assert [T.leg_split(s, 2, SMS) for s in specs[1:]] == [3, 7, 19, 18, 18, 18, 18, 14, 10, 6]
  assert all(T.leg_split(s, 3, SMS) == 1 for s in specs[1:])
  for s in specs[1:]:
    assert s['kh'] * s['kw'] * (s['cin'] // 16) // T.leg_split(s, 1, SMS) >= 4


def test_split_and_plane_relations():
  rng = np.random.default_rng(0)
  v = np.abs(rng.standard_normal(20000) * np.exp(rng.uniform(-20, 10, 20000))).astype(np.float32).astype(np.float64)
  hi, lo = T.split(v)
  assert T.check_planes(hi, lo) == []
  assert (np.abs(hi + lo - v) <= T.split_quantum(v)).all()
  assert T.check_planes(hi, lo + T.ulp16(hi)) != []            # lo beyond half a step of hi
  assert T.check_planes(hi * (1 + 2.0 ** -12), lo) != []       # not an fp16 value
  assert T.check_planes(-hi - 1, lo) != []
  assert T.check_planes(np.array([np.inf]), np.array([-np.inf])) == ['not finite']


@pytest.fixture(scope='module')
def chain():
  """The scan tests/test_gpu_leg_stages.py checks first, with every layer's input taken from the model itself."""
  w = N.glorot_weights(4, MODEL, seed=0)
  x = synth.range_like_images(1234, 1, 4)
  specs = T.layer_specs(4, MODEL)
  splits = [1] + [T.leg_split(s, 1, SMS) for s in specs[1:]]
  return w, x, specs, splits, T.forward(x[0], w, specs, splits)


def test_bounds_tell_wrong_products_apart_in_every_mma_layer(chain):
  w, x, specs, splits, vs = chain
  print()
  for l in range(1, len(specs)):
    spec = specs[l]
    k, b = w[spec['name']]
    hi, lo = T.split(vs[l - 1])
    last = l == len(specs) - 1
    assert splits[l] > 1
    v, tol, _ = T.mma_layer(hi, lo, k, b, spec, splits[l], last)
    assert np.array_equal(v, vs[l])
    frac = {}
    for name, kw in MUTANTS.items():
      m, _, _ = T.mma_layer(hi, lo, k, b, spec, splits[l], last, **kw)
      frac[name] = float((np.abs(m - v) > tol).mean())
    print('[tc_leg] %-9s bound / max %.1e; fraction beyond the bound: %s'
          % (spec['name'], tol.max() / v.max(), ', '.join('%s %.2f' % kv for kv in frac.items())))
    for name, f in frac.items():
      assert f >= MIN_FRACTION, (spec['name'], name, f)


def test_layer1_bound_tells_a_wrong_tap_or_channel(chain):
  w, x, specs, splits, vs = chain
  k, b = w['s_conv1']
  v, tol, _ = T.layer1(x[0], k, b, specs[0])
  assert tol.max() <= 3e-5 * v.max()
  for wrong in (np.roll(k, 1, axis=1), np.roll(k, 1, axis=2), k * np.float32(1 + 2.0 ** -13)):
    m, _, _ = T.layer1(x[0], wrong, b, specs[0])
    assert (np.abs(m - v) > tol).mean() >= MIN_FRACTION


@pytest.mark.parametrize('log2_scale', [-8, 0, 6])
def test_end_to_end_error_of_the_split_design(log2_scale):
  """The model fed with its own outputs against the float64 oracle: what the hi / lo split of activations and
  weights costs end to end (the fp32 accumulation excluded), as max |error| / max |volume|, with the depth channel
  and then s_conv1's kernel scaled by a power of two.  A few 1e-6 at every scale: the end-to-end tolerances of
  tests/test_gpu_network.py and tests/test_gpu_geometry.py allow for the fp32 accumulation on top of this."""
  f = np.float32(2.0 ** log2_scale)
  w = N.glorot_weights(4, MODEL, seed=0)
  x = synth.range_like_images(1234, 1, 4)
  specs = T.layer_specs(4, MODEL)
  splits = [1] + [T.leg_split(s, 1, SMS) for s in specs[1:]]
  xs = x.copy()
  xs[..., 0] *= f
  ws = dict(w, s_conv1=(w['s_conv1'][0] * f, w['s_conv1'][1]))
  for what, xi, wi in (('depth', xs, w), ('s_conv1 kernel', x, ws)):
    ref = N.leg_forward(xi, wi, MODEL, return_all=True)[-1][0]
    got = T.forward(xi[0], wi, specs, splits)[-1]
    print('\n[tc_leg] %s x 2^%d: end-to-end split error %.2e of the largest feature %.3g'
          % (what, log2_scale, rel(got, ref), ref.max()))
    assert rel(got, ref) <= 5e-6
