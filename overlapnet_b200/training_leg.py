"""The body of the reference's ``src/two_heads/training.py`` on the GPU path for its default configuration,
``legsType: 360OutputkLegs`` (config/network.yml:70, generateNet.py:119-219): every layer is trained, the leg
included, so a model can be trained from scratch and the orientation loss reaches the weights through the leg.

Every distinct scan's packed input is loaded once, through Infer's cue loader, into an image bank: on the GPU
when it fits beside the largest step's working set, else sharded over the GPUs of a node's data-parallel ranks or
in pinned host memory, from which each step's images are staged through a two-slot device ring while the previous
step computes (overlapnet_b200.image_bank).
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

from . import data_parallel
from . import image_bank as _image_bank
from . import training
from .engine import FEAT_C
from .image_bank import bank_rows  # noqa: F401 -- the row order of this flow's image bank, public here as well
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


class WholeNetwork:
  """The training step of 360OutputkLegs on an image bank.  ``image_bank`` None places the bank on the GPU when it
  fits beside the largest step's working set, sharded over the GPUs of a node's data-parallel ranks or in pinned host
  memory otherwise (overlapnet_b200.image_bank); 'device', 'host' or 'sharded' forces a placement.  All train the
  same bits."""

  def __init__(self, infer, keys, rotate_keys=None, image_bank=None, gradient_chunks=None):
    self.eng = infer._engine
    dp = data_parallel.default_group()
    world = 1 if dp is None else dp.world
    b_share = _image_bank.share_pairs(self.eng.max_batch_pairs, world, gradient_chunks)
    self.image_bank, self.images, self.rows = _image_bank.open_bank(
        infer, keys, image_bank, b_share, True, 2 * b_share if rotate_keys else 0, len(set(keys)), 'Image bank',
        _image_bank.parts_bytes(self.eng, True, world, gradient_chunks))
    self.image_rows = self.rows
    if self.image_bank == 'device':
      logger.info('Loaded %d scans into the image bank (%.1f MB on the GPU)', len(self.rows),
                  self.images.numel() * 4 / 1e6)
    else:
      self.ring = _image_bank.StagingRing(self.eng, self.images, 2 * b_share)

  whole_network = True           # the layers the gradients cover (Engine.copy_gradients, adagrad_step_sum)
  ring = None                    # the image_bank.StagingRing of a host or sharded image bank

  def begin_epoch(self, spans, left, right, rotate_rows=None):
    """With a host bank: the steps this rank runs in the coming epoch, in order -- pairs [a, b) of the training
    pairs' image rows ``left``, ``right`` and (yaw augmentation) ``rotate_rows``, host arrays -- whose images the
    ring then stages ahead of each step."""
    second = right if rotate_rows is None else rotate_rows
    self.ring.plan([(left[a:b], second[a:b]) for a, b in spans])

  def step(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, lr, rotate=None):
    """``rotate`` = (image rows, column shifts, (cos, sin)) of the batch's RIGHT scans, or None: the step then
    trains on a 2n-image batch of the LEFT images and the rotated RIGHT images."""
    loss = self.gradients(left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate)
    self.eng.net_adagrad_step(lr)
    return loss

  def gradients(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate=None, chunks=None):
    """``step`` without its update: the losses; the gradients stay in the handle (the data-parallel step).  With
    a host bank, ``left``, ``right`` and the rows of ``rotate`` are the next span begin_epoch planned: the step
    reads their images from the ring's slot, at the local indices of that plan.  ``chunks`` = (offsets, parts):
    the gradients of each chunk [offsets[c], offsets[c + 1]) of the pairs go to parts[c] in one call
    (Engine.net_gradients_chunks), and the losses of each chunk are returned."""
    images = self.images
    if self.ring is not None:
      images, (left, second) = self.ring.take()
      if rotate is not None:
        rotate = (second,) + tuple(rotate[1:])
      else:
        right = second
    try:
      if rotate is not None:
        rows, shifts, rot = rotate
        n = left.numel()
        src = images
        images = src.new_empty((2 * n,) + tuple(src.shape[1:]))
        # LEFT is copied without a rotation: even a rotation by (1, 0) could flip the sign of a zero normal
        # component
        self.eng.gather_images(src, left, out=images[:n])
        self.eng.gather_images(src, rows, shifts, rot, out=images[n:])
        pairs = torch.arange(2 * n, dtype=torch.int32, device=self.eng.device)
        left, right = pairs[:n], pairs[n:]
      if chunks is not None:
        return self.eng.net_gradients_chunks(images, left, right, chunks[0], gt_overlap, gt_orientation,
                                             min_overlap_for_angle, out=chunks[1])[0]
      return self.eng.net_gradients(images, left, right, gt_overlap, gt_orientation, min_overlap_for_angle)
    finally:
      if self.ring is not None:
        self.ring.release()

  def evaluate(self, left, right):
    """(overlap, yaw) device tensors of the validation pairs: the scans re-encoded by the current leg.  With a
    host bank only the scans these pairs use, streamed through the ring in slot-sized chunks into a feature bank
    (the fp32 leg computes every image on its own, so the chunking changes no bit)."""
    if self.ring is None:
      bank = self.eng.leg(self.images)
      ov, yaw, _ = self.eng.heads(bank, left, right)
      return ov, yaw
    rows, (l, r) = _image_bank.plan_rows(left.cpu().numpy(), right.cpu().numpy())
    k = self.ring.slot_rows
    chunks = [rows[i:i + k] for i in range(0, rows.size, k)]
    bank = torch.empty((rows.size, self.eng.Wf, FEAT_C), dtype=torch.float32, device=self.eng.device)
    self.ring.plan([(c,) for c in chunks])
    for i, c in enumerate(chunks):
      x, _ = self.ring.take()
      self.eng.leg(x[:c.size], out=bank[i * k:i * k + c.size])
      self.ring.release()
    dev = self.eng.device
    ov, yaw, _ = self.eng.heads(bank, torch.from_numpy(l).to(dev), torch.from_numpy(r).to(dev))
    return ov, yaw


def train(config, device=None):
  """Run the training of training.py with a trainable leg for a loaded YAML dict.  Returns the history dict
  of ``training.train``."""
  check_config(config)
  return training.run(config, device, WholeNetwork)
