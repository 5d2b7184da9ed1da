"""The work split of the tensor-core heads does not reach the results.  k_delta_conv1_wgmma gives each persistent
CTA a contiguous range of the n_pairs * 24 (pair, jb) units, and c_conv2, c_conv3 and the correlation head split
their rows the same way, so where a CTA's share starts and ends depends on the number of pairs.  Every row takes
the same K steps in any share, so a call over the first n candidates must give those candidates' results of the
1101-candidate call bit for bit: n = 1, 2, 3 (at most one delta unit per CTA on an H100), and n = 8 and 37 (more
units than SMs, shares that start and end inside a pair)."""
import numpy as np
import pytest
import torch

from oracle import network as N
from overlapnet_b200 import synth
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}


def test_first_n_candidates_match_the_full_call_bit_for_bit():
  w = N.glorot_weights(4, MODEL, seed=0)
  n = 1101
  eng = Engine(model=MODEL, precision='f16_tc', max_batch_scans=1, max_batch_pairs=n)
  bank_np = synth.feature_volumes(11, n)[:, 0] * np.float32(0.2)
  sel = np.arange(16)
  right_np = np.repeat(bank_np[17][None, None], len(sel), 0)
  _, _, _, z0 = N.heads_forward(bank_np[sel][:, None], right_np, w, MODEL, return_logit=True)
  eng.load_weights(N.spread_dense(w, z0, target_std=1.5))
  bank = torch.from_numpy(bank_np).to(eng.device)
  q = bank[17].clone()
  ov, yaw, corr = eng.heads_1vsN(bank, q, n_cand=n, want_corr=True)
  ov, yaw, corr = ov.clone(), yaw.clone(), corr.clone()
  assert float(ov.max() - ov.min()) > 0.1          # spread overlaps: the comparison sees the logits' low bits
  for k in (1, 2, 3, 8, 37):
    ovk, yawk, corrk = eng.heads_1vsN(bank, q, n_cand=k, want_corr=True)
    assert torch.equal(ovk, ov[:k]), k
    assert torch.equal(yawk, yaw[:k]), k
    assert torch.equal(corrk, corr[:k]), k
  eng.check()
  eng.close()
