"""Float64 model of the tensor-core leg (precision ``f16_tc``), layer by layer (TEST INFRASTRUCTURE).

Each function models one layer from the GPU's own input to that layer (the hi / lo planes of the layer before,
read back with ``Engine.leg_stage``), so an error is caught in the layer that makes it and is not smeared by the
convolutions and ReLUs after it.  Each returns ``(model, tol, near_kink)``: the fp32 value ``v`` the kernel forms
before it splits it into planes (after bias and ReLU), computed in float64 with every fp16 rounding the kernel
makes, a per-element bound on ``|gpu - model|`` where ``gpu = hi + lo`` of the stored planes (the fp32 volume for
the last layer), and the number of elements whose pre-activation lies within the bound of 0 (ReLU is 1-Lipschitz,
so they need no exemption).  ``rounding=False`` switches the fp16 roundings off; the layers then chain to
``oracle.network.leg_forward(..., return_all=True)`` exactly.  ``split(v)`` gives the planes of a model value.

Rounding points (``csrc/network_tc.cu``); ``h`` = fp16 round-to-nearest-even with subnormals kept:
* planes (every layer but the last): ``hi = h(v)``, ``lo = h(v - hi)`` of the fp32 ``v``.  ``hi + lo`` is within
  half an fp16 ulp of ``lo`` of ``v``: ``2^-25`` once ``lo`` is subnormal.  hi itself is NOT compared with the model's:
  a ``v`` next to a rounding boundary of fp16 may fall on either side; the sum is compared, and the planes must
  satisfy the exact relations of ``check_planes``.
* s_conv1 (``k_leg_layer1_small`` / ``k_leg_layer1_direct``): an fp32 ``fmaf`` chain over (dh, dw, c) that starts
  at the bias.  Bound: half an fp32 ulp of the running partial sum per step (its magnitude taken from the float64
  partial sums in that order), not ``steps * 2^-24 * sum |x| |w|``.
* s_conv2.. (``k_leg_mma``): the input is ``xh + xl``, the weights ``wh = h(w)``, ``wl = h(fp32(w - wh))``
  (``tc_pack_weights``), the product ``xh wh + xl wh + xh wl`` (``xl wl`` is dropped: at most ``2^-22`` relative,
  and part of the model, not of the bound).  K is walked as iterations (tap = dh kw + dw, 16 channels), three
  m16n8k16 MMAs each, into an fp32 accumulator that starts at 0; with ``n_split`` K slices, slice s takes the
  iterations ``[n_it s / n_split, n_it (s + 1) / n_split)`` and ``k_leg_splitk_reduce`` adds the slices in slice
  order in fp32, then the bias.  The tensor core aligns the 16 products and the accumulator of an MMA to the
  largest exponent and truncates, so each MMA loses a few units of the last place of the largest of them.  Bound:
  ``MMA_ULPS`` fp32 ulps per MMA of ``max(|acc before|, |acc after|, sum |xh| |wh| of the iteration)``, from the
  float64 partial sums in the kernel's order, plus half an fp32 ulp per slice add and for the bias add.
  ``MMA_ULPS = 1`` is an allowance, not a worst case (17 truncated addends could lose 4-5 ulps, and always in the
  same direction): the worst case over s_conv3's 270 MMAs would not tell a dropped ``xl wh`` term from the true
  product.  The GPU tests print the measured ratio of error to bound per layer
  (``tests/test_gpu_leg_stages.py``); ``tests/test_oracle_tc_leg.py`` shows that the bound separates the kernel's
  product from each of five wrong ones in every layer.
"""
import numpy as np

from .tc_heads import h, ulp16

MMA_ULPS = 1.0
F16_MAX = 65504.0


def ulp32(x):
  """Spacing of the fp32 numbers at |x| (that of the smallest normal number below it)."""
  a = np.maximum(np.abs(np.asarray(x, np.float64)), 2.0 ** -126).astype(np.float32)
  return np.spacing(a).astype(np.float64)


def layer_specs(in_channels, model_cfg=None, H=64, W=900):
  """The leg's layers as dicts (name, kh, kw, sh, sw, cin, cout, h_in, w_in, h_out, w_out), input to output."""
  from . import network as N
  out = []
  cin, hh, ww = in_channels, H, W
  for name, (kh, kw), (sh, sw), cout in N.leg_layers(model_cfg):
    ho, wo = (hh - kh) // sh + 1, (ww - kw) // sw + 1
    out.append(dict(name=name, kh=kh, kw=kw, sh=sh, sw=sw, cin=cin, cout=cout, h_in=hh, w_in=ww, h_out=ho, w_out=wo))
    cin, hh, ww = cout, ho, wo
  return out


def leg_split(spec, n, sm_count):
  """K slices of a layer (s_conv2..) for a call of n scans: ``leg_split`` of csrc/network_tc.cu restated."""
  if n > 2:
    return 1
  tiles = n * spec['h_out'] * ((spec['w_out'] + 63) // 64) * ((spec['cout'] + 63) // 64)
  n_it = spec['kh'] * spec['kw'] * (spec['cin'] // 16)
  return max(1, min((4 * sm_count + tiles - 1) // tiles, n_it // 4))


def split(v, rounding=True):
  """The hi / lo planes of a value: hi = h(v), lo = h(v - hi); (v, 0) without rounding."""
  v = np.asarray(v, np.float64)
  if not rounding:
    return v, np.zeros_like(v)
  hi = h(v)
  return hi, h(v - hi)


def split_quantum(v):
  """Bound on |hi + lo - v|: half an fp16 ulp of lo, |lo| <= ulp16(v) / 2."""
  return 0.5 * ulp16(0.5 * ulp16(v))


def check_planes(hi, lo):
  """The relations the stored planes satisfy whatever the value: finite, hi >= 0, |lo| <= ulp16(hi) / 2, and
  hi == h(fp32(hi + lo)) bit for bit, except where lo is exactly half an ulp of hi: lo is itself rounded, so it can
  reach the tie, which h() resolves to the even neighbour.  Returns the list of violated relations."""
  hi, lo = np.asarray(hi, np.float64), np.asarray(lo, np.float64)
  bad = []
  if not (np.isfinite(hi).all() and np.isfinite(lo).all()):
    return ['not finite']
  if not (hi == h(hi)).all() or not (lo == h(lo)).all():
    bad.append('not fp16 values')
  if (hi < 0).any():
    bad.append('hi < 0')
  half = 0.5 * ulp16(hi)
  if (np.abs(lo) > half).any():
    bad.append('|lo| > ulp16(hi) / 2')
  again = h((hi + lo).astype(np.float32))
  if ((again != hi) & (np.abs(lo) < half)).any():
    bad.append('hi != h(hi + lo)')
  return bad


def _windows(x, spec):
  """x[(H, W, C)] -> a function (dh, dw) -> the (h_out * w_out, C) rows the tap reads."""
  ho, wo, sh, sw = spec['h_out'], spec['w_out'], spec['sh'], spec['sw']

  def tap(dh, dw):
    return x[dh:dh + (ho - 1) * sh + 1:sh, dw:dw + (wo - 1) * sw + 1:sw].reshape(ho * wo, -1)
  return tap


def layer1(x, w, b, spec, rounding=True):
  """s_conv1 of one scan x (H, W, C) float32."""
  del rounding                                    # no fp16 rounding before the split
  tap = _windows(np.asarray(x, np.float64), spec)
  W = np.asarray(w, np.float64)
  acc = np.broadcast_to(np.asarray(b, np.float64), (spec['h_out'] * spec['w_out'], spec['cout'])).copy()
  tol = np.zeros_like(acc)
  for dh in range(spec['kh']):
    for dw in range(spec['kw']):
      xs = tap(dh, dw)
      for c in range(spec['cin']):
        acc += xs[:, c:c + 1] * W[dh, dw, c][None, :]
        tol += 0.5 * ulp32(acc)
  shape = (spec['h_out'], spec['w_out'], spec['cout'])
  tol = (tol * (1 + 2.0 ** -20)).reshape(shape)
  pre = acc.reshape(shape)
  v = np.maximum(pre, 0)
  return v, tol + split_quantum(v + tol), int((np.abs(pre) <= tol).sum())


def weight_split(w):
  """(wh, wl) as tc_pack_weights stores them: wh = h(w), wl = h(fp32(w - wh))."""
  w = np.asarray(w, np.float32)
  wh = w.astype(np.float16)
  wl = (w - wh.astype(np.float32)).astype(np.float16)
  return wh.astype(np.float64), wl.astype(np.float64)


def mma_layer(xh, xl, w, b, spec, n_split=1, last=False, rounding=True, terms=('hh', 'lh', 'hl'), dw_shift=0,
              drop_last_slice=False):
  """One k_leg_mma layer of one scan from the planes xh, xl (H, W, C_in) of the layer before.  ``last``: the fp32
  volume (no split).  ``terms``, ``dw_shift`` and ``drop_last_slice`` build deliberately wrong models for the
  mutation tests: a subset of the three products, the window of tap (dh, dw + dw_shift) under the weights of
  (dh, dw), and the reduction without the last K slice."""
  xh, xl = np.asarray(xh, np.float64), np.asarray(xl, np.float64)
  if rounding:
    wh, wl = weight_split(w)
  else:
    wh, wl = np.asarray(w, np.float64), np.zeros(np.shape(w))
    xh, xl = xh + xl, np.zeros_like(xh)
  if dw_shift:                                   # the tap's window moved by whole pixels (circularly: test only)
    xh, xl = np.roll(xh, -dw_shift, axis=1), np.roll(xl, -dw_shift, axis=1)
  th, tl, ta = _windows(xh, spec), _windows(xl, spec), _windows(np.abs(xh), spec)
  wa = np.abs(wh)
  P, cout = spec['h_out'] * spec['w_out'], spec['cout']
  per_tap = spec['cin'] // 16
  n_it = spec['kh'] * spec['kw'] * per_tap
  total = np.zeros((P, cout))
  tol = np.zeros((P, cout))
  n_used = n_split - 1 if drop_last_slice else n_split
  for s in range(n_used):
    acc = np.zeros((P, cout))
    for it in range(n_it * s // n_split, n_it * (s + 1) // n_split):
      t, c0 = it // per_tap, 16 * (it % per_tap)
      dh, dw = t // spec['kw'], t % spec['kw']
      c = slice(c0, c0 + 16)
      ah = th(dh, dw)[:, c]
      before = np.abs(acc)
      if 'hh' in terms:
        acc += ah @ wh[dh, dw, c]
      if 'lh' in terms:
        acc += tl(dh, dw)[:, c] @ wh[dh, dw, c]
      if 'hl' in terms:
        acc += ah @ wl[dh, dw, c]
      if rounding:
        mag = np.maximum(np.maximum(before, np.abs(acc)), ta(dh, dw)[:, c] @ wa[dh, dw, c])
        tol += 3 * MMA_ULPS * ulp32(mag * (1 + 2.0 ** -9))
    if n_split > 1:                               # the reduce kernel's fp32 adds, slice order, from 0
      total += acc
      tol += 0.5 * ulp32(np.abs(total) + tol)
    else:
      total = acc
  pre = total + np.asarray(b, np.float64)
  shape = (spec['h_out'], spec['w_out'], cout)
  if not rounding:
    return np.maximum(pre, 0).reshape(shape), np.zeros(shape), 0
  tol += 0.5 * ulp32(np.abs(pre) + tol)
  tol = tol.reshape(shape)
  pre = pre.reshape(shape)
  v = np.maximum(pre, 0)
  if not last:
    tol = tol + split_quantum(v + tol)
  return v, tol, int((np.abs(pre) <= tol).sum())


def forward(x, weights, specs, splits=None, rounding=True):
  """The model fed with its own outputs: every layer's value v of one scan x (H, W, C), s_conv1 .. the last layer.
  ``splits``: K slices per layer (default 1 each)."""
  out = []
  hi = lo = None
  for l, spec in enumerate(specs):
    k, b = weights[spec['name']]
    if l == 0:
      v, _, _ = layer1(x, k, b, spec, rounding)
    else:
      v, _, _ = mma_layer(hi, lo, k, b, spec, splits[l] if splits else 1, l == len(specs) - 1, rounding)
    out.append(v)
    hi, lo = split(v, rounding)
  return out
