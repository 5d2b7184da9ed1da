"""The per-point class probabilities the raw-scan entry points take are checked before anything reaches the device;
the library and its bindings list the new entry points together."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT
from overlapnet_b200.engine import check_probs

NEW_SYMBOLS = ('ovn_preprocess_cues_batch', 'ovn_encode_clouds_probs_host', 'ovn_query_cloud_probs_vs_bank_host')


def test_probabilities_that_fit_pass_through():
  p = np.zeros((7, 20), np.float32)
  assert check_probs(p, 7, 20, 'f') is p
  t = torch.zeros((5, 3))
  assert check_probs(t, 5, 3, 'f') is t
  assert check_probs(None, 7, 20, 'f') is None               # the library refuses a missing array itself
  assert check_probs(np.zeros((0, 20), np.float32), 0, 20, 'f').shape == (0, 20)


@pytest.mark.parametrize('shape', [(6, 20), (8, 20), (7, 19), (7, 3), (7,), (7, 20, 1), (140,)])
def test_wrong_shapes_are_refused(shape):
  with pytest.raises(ValueError, match=r'f: class probabilities of shape .*expected \(7, 20\)'):
    check_probs(np.zeros(shape, np.float32), 7, 20, 'f')


def test_probabilities_on_a_geometric_handle_are_refused():
  with pytest.raises(ValueError, match='no probability channels'):
    check_probs(np.zeros((7, 20), np.float32), 7, 0, 'f')


def test_new_entry_points_are_declared_bound_and_documented():
  from overlapnet_b200 import _cabi
  header = open(os.path.join(ROOT, 'include', 'ovn_b200.h')).read()
  integration = open(os.path.join(ROOT, 'INTEGRATION.md')).read()
  for name in NEW_SYMBOLS:
    assert re.search(r'\bint %s\(' % name, header), name
    assert name in _cabi.SYMBOLS and name in integration, name
