"""Yaw augmentation of training pairs: the RIGHT scan is rotated about z and its orientation label moved by the
amount the geometry implies (DESIGN.md section 7).

The projection puts a point at column 0.5 (-atan2(y, x) / pi + 1) W (utils.py:86-90), so rolling a range image
by s columns is the image of the cloud rotated by theta = -2 pi s / W; the normal vectors rotate with it
(``ovn_gather_images``).  The label is the yaw bin floor(-(yaw / pi) Wf / 2) + Wf / 2 of cur_inv . pose_ref
(com_overlap_yaw.py:54) with RIGHT the reference frame, and rotating RIGHT by theta replaces pose_ref with
pose_ref . Rz(-theta), so the label becomes (label - s Wf / W) mod Wf.  That is a whole bin only when s is a
multiple of the column pitch p = W / gcd(W, Wf); the shifts drawn here are such multiples.
"""
import math

import numpy as np


def column_pitch(W, Wf):
  """The smallest column shift p of a W-column image that moves the Wf-bin label by a whole number of bins."""
  return W // math.gcd(int(W), int(Wf))


def sample_shifts(n, W, Wf):
  """n column shifts, uniform over the multiples of the column pitch in [0, W), from NumPy's global RNG."""
  p = column_pitch(W, Wf)
  return (np.random.randint(0, W // p, n) * p).astype(np.int32)


def rotation(shifts, W):
  """(cos theta, sin theta) of theta = -2 pi s / W per shift, computed in float64, as float32 [n, 2]."""
  theta = -2.0 * np.pi * np.asarray(shifts, np.float64) / W
  return np.stack([np.cos(theta), np.sin(theta)], axis=-1).astype(np.float32)


def move_labels(orientation, shifts, W, Wf):
  """Orientation labels of the RIGHT scans rolled by ``shifts`` columns: (label - s Wf / W) mod Wf.  Works on
  NumPy arrays and on integer torch tensors (on their device); every shift must be a multiple of the pitch."""
  p = column_pitch(W, Wf)
  rem = shifts % p
  if bool(rem.any() if hasattr(rem, 'any') else rem):
    raise ValueError('shifts must be multiples of the column pitch %d (W = %d, Wf = %d)' % (p, W, Wf))
  return (orientation - shifts * Wf // W) % Wf
