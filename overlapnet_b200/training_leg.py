"""The body of the reference's ``src/two_heads/training.py`` on the GPU path for its default configuration,
``legsType: 360OutputkLegs`` (config/network.yml:70, generateNet.py:119-219): every layer is trained, the leg
included, so a model can be trained from scratch and the orientation loss reaches the weights through the leg.

Every distinct scan's packed input is loaded once, through Infer's cue loader, into an image bank on the GPU.
A training step gathers its 2B images from that bank, runs the leg and both heads forward and the whole
network backward (``ovn_net_gradients``), then an Adagrad update of every layer (``ovn_net_adagrad_step``).
Each epoch re-encodes the image bank with the current leg for the validation pairs.  The loop, the logging, the history and the
weight file are those of ``overlapnet_b200.training``.

  python -m overlapnet_b200.training config.yml        (dispatches here on legsType 360OutputkLegs)

Not supported (an Exception says so): ``rotate_training_data`` -- the reference rolls the RIGHT image without
moving its yaw label (ImagePairOverlapOrientationSequence.py:112,209-212) -- and TensorBoard output.
``yaw_augmentation: True`` is the geometric version (overlapnet_b200.training, overlapnet_b200.augment).
"""
import torch

from . import training
from .training import logger


def check_config(config):
  """Refuse the configurations this driver cannot train."""
  legs = config['model'].get('legsType')
  if legs == '360OutputkLegsFixed':
    raise Exception('legsType 360OutputkLegsFixed freezes the leg: that is overlapnet_b200.training; this flow '
                    'trains 360OutputkLegs')
  if legs != '360OutputkLegs':
    raise Exception('legsType %r is not supported for training; use 360OutputkLegs' % (legs,))
  training.check_unsupported_options(config)
  training.check_yaw_augmentation(config)
  training.check_training_precision(config)


def load_image_bank(infer, keys, chunk=256):
  """Packed network inputs of the distinct (dir, scan) keys, through Infer's cue loader (one sequence
  directory at a time), in one device tensor [n, H, W, C].  Returns it and {key: row}."""
  eng = infer._engine
  rows = {}
  for d in sorted({k[0] for k in keys}):
    for name in sorted(k[1] for k in keys if k[0] == d):
      rows[(d, name)] = len(rows)
  bank = torch.empty((len(rows), eng.H, eng.W, eng.C), dtype=torch.float32, device=eng.device)
  for d in sorted({k[0] for k in keys}):
    names = sorted(k[1] for k in keys if k[0] == d)
    infer.seq = d
    for s in range(0, len(names), chunk):
      x = infer._prepare_inputs(names[s:s + chunk])
      r0 = rows[(d, names[s])]
      bank[r0:r0 + len(x)] = torch.from_numpy(x).to(eng.device)
  return bank, rows


class WholeNetwork:
  """The training step of 360OutputkLegs on an image bank."""

  def __init__(self, infer, keys, rotate_keys=None):
    self.eng = infer._engine
    self.images, self.rows = load_image_bank(infer, keys)
    self.image_rows = self.rows
    logger.info('Loaded %d scans into the image bank (%.1f MB on the GPU)', len(self.rows),
                self.images.numel() * 4 / 1e6)

  whole_network = True           # the layers the gradients cover (Engine.copy_gradients, adagrad_step_sum)

  def step(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, lr, rotate=None):
    """``rotate`` = (image rows, column shifts, (cos, sin)) of the batch's RIGHT scans, or None: the step then
    trains on a 2n-image batch of the LEFT images and the rotated RIGHT images."""
    loss = self.gradients(left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate)
    self.eng.net_adagrad_step(lr)
    return loss

  def gradients(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate=None):
    """``step`` without its update: the losses; the gradients stay in the handle (the data-parallel step)."""
    images = self.images
    if rotate is not None:
      rows, shifts, rot = rotate
      n = left.numel()
      images = self.images.new_empty((2 * n,) + tuple(self.images.shape[1:]))
      # LEFT is copied without a rotation: even a rotation by (1, 0) could flip the sign of a zero normal component
      self.eng.gather_images(self.images, left, out=images[:n])
      self.eng.gather_images(self.images, rows, shifts, rot, out=images[n:])
      pairs = torch.arange(2 * n, dtype=torch.int32, device=self.eng.device)
      left, right = pairs[:n], pairs[n:]
    return self.eng.net_gradients(images, left, right, gt_overlap, gt_orientation, min_overlap_for_angle)

  def evaluate(self, left, right):
    """(overlap, yaw) device tensors of the validation pairs: the scans re-encoded by the current leg."""
    bank = self.eng.leg(self.images)
    ov, yaw, _ = self.eng.heads(bank, left, right)
    return ov, yaw


def train(config, device=None):
  """Run the training of training.py with a trainable leg for a loaded YAML dict.  Returns the history dict
  of ``training.train``."""
  check_config(config)
  return training.run(config, device, WholeNetwork)
