"""The three-term hi/lo product the tensor-core path uses for the leg layers and the correlation head
(overlapnet_b200/csrc/network_tc.cu: k_leg_mma, k_corr_mma), restated in NumPy: x * w ~= x_hi w_hi + x_hi w_lo
+ x_lo w_hi with fp16 halves and fp32-grade accumulation."""
import numpy as np


def test_hi_lo_stacked_product_is_fp32_grade():
  """x*w ~= x_hi*w_hi + x_hi*w_lo + x_lo*w_hi with fp16 halves and fp32 accumulation: the term left out
  (x_lo*w_lo) is below 2^-22 relative."""
  rng = np.random.default_rng(0)
  x = rng.normal(size=(512, 240)).astype(np.float32)
  w = rng.normal(size=(240, 16)).astype(np.float32)
  xh = x.astype(np.float16); xl = (x - xh.astype(np.float32)).astype(np.float16)
  wh = w.astype(np.float16); wl = (w - wh.astype(np.float32)).astype(np.float16)
  f = lambda a: a.astype(np.float64)
  got = f(xh) @ f(wh) + f(xh) @ f(wl) + f(xl) @ f(wh)
  ref = x.astype(np.float64) @ w.astype(np.float64)
  assert np.abs(got - ref).max() / np.abs(ref).max() < 2e-6
