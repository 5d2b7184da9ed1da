"""The body of the reference's ``src/two_heads/training.py`` on the GPU path, for the
``360OutputkLegsFixed`` configuration (generateNet.py:222-324): the leg is frozen and the four layers of
the overlap head (c_conv1..3, overlap_output) are trained with Adagrad on the losses of training.py:71-92.

Every distinct scan is encoded once by the frozen leg into a feature bank that stays on the GPU; a training
step is then the heads' forward plus the overlap head's backward (``ovn_head_gradients``) and an Adagrad
update (``ovn_head_adagrad_step``).  The orientation loss has no gradient with a frozen leg, but it is
computed and logged as part of the total loss like training.py does.

  python -m overlapnet_b200.training config.yml

The same command trains the whole network when the config's legsType is 360OutputkLegs: ``main`` hands such
a config to ``overlapnet_b200.training_leg``, which runs this loop with the leg's backward added.

Not supported (an Exception says so): ``rotate_training_data`` (it would re-encode the rolled RIGHT image for
every pair of every epoch) and TensorBoard output.

``yaw_augmentation: True`` (both legsTypes, default False) is the geometric version of that rotation
(overlapnet_b200.augment): every epoch each training pair's RIGHT scan is rotated about z by a random multiple of
the column pitch, its normals with it, and its orientation label moved to match.  Here the frozen leg encodes
each step's rotated RIGHT images.  Validation is never augmented.

An image bank (the whole network's; the frozen leg's RIGHT scans under yaw augmentation) that does not fit on the
GPU beside the largest step's working set is kept in pinned host memory, and each step's images are staged to the
GPU while the previous step computes (overlapnet_b200.image_bank, DESIGN.md section 6); the weights are the same.
Under data-parallel training on one node, a bank whose 1/world share fits every GPU is instead sharded over the
ranks' GPUs, and each step gathers its images from the owners' memory.

``training_precision: tf32x3`` (both legsTypes, default fp32) runs every product of the gradient steps on tensor
cores in 3xTF32 with fp32 accumulation (Engine.set_train_precision); validation stays fp32.

Both flows train data-parallel over the GPUs of a node (overlapnet_b200.data_parallel, DESIGN.md section 6):

  python -m torch.distributed.run --nproc_per_node G -m overlapnet_b200.training config.yml

``batch_size`` stays the global batch; each rank trains on a contiguous share of every batch, and the ranks'
gradients are all-gathered and summed in rank order on the device, so every rank keeps the same weights.

``gradient_chunks: K`` (both legsTypes, 1 <= K <= min(64, batch_size), K >= the world size; default off) makes the
bits independent of the world size: every batch of n pairs is cut into K contiguous chunks, each rank computes the
gradients of its contiguous range of chunks in one call (Engine.head_gradients_chunks / net_gradients_chunks), and
g = sum_k (n_k / n) g_k is summed in chunk order.  A run with the key gives the same weights, accumulators, history
and checkpoints on any number of GPUs up to K, and may be resumed on another; K = 1 on one GPU is the run without
the key.

``checkpoint: True`` (both legsTypes, default False) writes ``<experiments_path>/<testname>/checkpoint.npz`` after
every epoch, atomically: the weights, the Adagrad accumulators (Engine.train_state), NumPy's random state, the
training pairs in the run's order, the history so far and a fingerprint of the config keys that fix the
trajectory.  ``resume: True`` (implies ``checkpoint``) continues such a run from its last completed epoch up to
``no_epochs``, with the same learning-rate schedule, batch orders and yaw shifts, so that its weights and history
are those of the uninterrupted run bit for bit (DESIGN.md section 6).  It refuses a checkpoint whose fingerprint,
layers or state do not fit the config; ``no_epochs``, ``no_test_pairs``, the validation files,
``training_precision`` and the world size may change, and ``pretrained_weightsfilename`` is ignored.
"""
import json
import logging
import os
import sys
import time

import numpy as np
import torch

from . import augment
from . import data_parallel
from . import evaluate
from . import image_bank as _image_bank
from . import weights as _weights
from .config import load_config

logger = logging.getLogger('overlapnet_b200.training')

OVERLAP_THRESHOLDS = (0.3, 0.4, 0.5, 0.6, 0.7, 0.8, 0.9)          # training.py:398
CUE_DEFAULTS = (('use_depth', True), ('use_normals', True), ('use_class_probabilities', False),
                ('use_class_probabilities_pca', False), ('use_intensity', False))              # training.py:137-160
CHECKPOINT = 'checkpoint.npz'
CHECKPOINT_VERSION = 1


def learning_rate(epoch, initial_lr=1e-3, alpha=0.99):
  """learning_rate_schedule (training.py:47-57): epoch 0 uses 0.1 lr, then lr alpha^(epoch-1)."""
  if epoch < 1:
    return initial_lr * 0.1
  return initial_lr * np.power(alpha, epoch - 1.0)


def check_config(config):
  """Refuse the configurations this driver cannot train."""
  model = config['model']
  legs = model.get('legsType')
  if legs == '360OutputkLegs':
    raise Exception('legsType 360OutputkLegs trains the leg: that is overlapnet_b200.training_leg (python -m '
                    'overlapnet_b200.training dispatches it); this flow trains 360OutputkLegsFixed (frozen leg)')
  if legs != '360OutputkLegsFixed':
    raise Exception('legsType %r is not supported for training; use 360OutputkLegsFixed' % (legs,))
  check_unsupported_options(config)
  check_yaw_augmentation(config)
  check_training_precision(config)


TRAINING_PRECISIONS = ('fp32', 'tf32x3')
MAX_GRADIENT_CHUNKS = 64             # the most parts of one ovn_adagrad_step_sum


def check_gradient_chunks(config, world=1):
  """``gradient_chunks: K`` (both legsTypes, default off): each batch's gradient is the weighted sum of the
  gradients of K fixed chunks, so that the run's bits do not depend on the world size.  Returns K, or None without
  the key; raises an Exception that names the problem for a K the loop cannot train on ``world`` ranks."""
  if 'gradient_chunks' not in config:
    return None
  k = config['gradient_chunks']
  if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or k < 1:
    raise Exception('gradient_chunks %r is not an integer >= 1' % (k,))
  k = int(k)
  if k > MAX_GRADIENT_CHUNKS:
    raise Exception('gradient_chunks %d exceeds %d, the most parts one Adagrad step sums' % (k, MAX_GRADIENT_CHUNKS))
  batch_size = int(config['batch_size'])
  if k > batch_size:
    raise Exception('gradient_chunks %d exceeds batch_size %d: a full batch would have empty chunks' % (k, batch_size))
  if k < world:
    raise Exception('gradient_chunks %d is below the world size %d: every rank trains at least one chunk' % (k, world))
  return k


def check_training_precision(config):
  """``training_precision`` (both legsTypes, default fp32) is the arithmetic of the gradient steps:
  ``tf32x3`` runs their products on tensor cores in 3xTF32 (Engine.set_train_precision)."""
  p = config.get('training_precision', 'fp32')
  if p not in TRAINING_PRECISIONS:
    raise Exception('training_precision %r is not supported; use one of %s' % (p, ', '.join(TRAINING_PRECISIONS)))


def check_yaw_augmentation(config):
  """``yaw_augmentation: True`` needs a rotation that moves the label by whole bins: some multiple of the column
  pitch below W (overlapnet_b200.augment)."""
  if not config.get('yaw_augmentation', False):
    return
  model = config['model']
  W, Wf = int(model['inputShape'][1]), int(model.get('leg_output_width', 360))
  if augment.column_pitch(W, Wf) == W:
    raise Exception('yaw_augmentation: no rotation of a W = %d image moves the Wf = %d orientation label by whole '
                    'bins (gcd(W, Wf) = 1)' % (W, Wf))


def check_unsupported_options(config):
  """Options neither training flow implements."""
  if config.get('rotate_training_data', 0) != 0:
    raise Exception('rotate_training_data != 0 is not supported: with a frozen leg it would re-encode the '
                    'rolled RIGHT image of every pair in every epoch')
  if config.get('tensorboard', False):
    raise Exception('TensorBoard output is not supported')


def npz_files(config):
  """training.py:124-134: per-sequence train / validation sets, or two single files."""
  root = config.get('data_root_folder', '')
  if 'training_seqs' in config:
    seqs = str(config['training_seqs']).split()
    return ([os.path.join(root, s, 'ground_truth/train_set.npz') for s in seqs],
            [os.path.join(root, s, 'ground_truth/validation_set.npz') for s in seqs])
  return [config['traindata_npzfile']], [config['validationdata_npzfile']]


def orientation_rms(overlap, argmax, gt_orientation, width):
  """training.py:398-415: yaw RMS over the pairs whose predicted overlap exceeds each threshold
  (NaN when no pair does)."""
  out = {}
  for thr in OVERLAP_THRESHOLDS:
    sel = overlap > thr
    a = np.abs(argmax[sel] - gt_orientation[sel])
    d = np.minimum(a, width - a)
    out[thr] = float(np.sqrt(np.mean(d * d))) if d.size else float('nan')
  return out


def _encode_bank(infer, keys):
  """Feature volumes of the distinct (dir, scan) keys with the frozen leg, through Infer's cue loader
  (one sequence directory at a time).  Returns the bank [n, Wf, 128] and {key: row} (image_bank.bank_rows)."""
  rows, parts = _image_bank.bank_rows(keys), []
  for d in sorted({k[0] for k in rows}):
    infer.seq = d
    parts.append(infer._create_feature_volumes_device([name for dd, name in rows if dd == d]))
  return torch.cat(parts).contiguous(), rows


def save_weights(path, weights):
  """The full model (leg + head) in the .npz container, written through a file object so that the
  name stays exactly ``path`` (np.savez appends .npz to a path)."""
  with open(path, 'wb') as f:
    _weights.save_npz(f, weights)


def _plain(value):
  """``value`` as JSON reads it back (tuples become lists), so that a config and a stored fingerprint compare."""
  return json.loads(json.dumps(value, sort_keys=True))


def trajectory_fingerprint(config):
  """The config values that fix a run's trajectory -- its draws, batches, steps and learning rates -- as the loop
  reads them.  A checkpoint is resumed only under the same values."""
  fp = {'model': config['model']}
  fp.update((key, config.get(key, default)) for key, default in CUE_DEFAULTS)
  fp.update(batch_size=int(config['batch_size']), no_batches_in_epoch=int(config['no_batches_in_epoch']),
            learning_rate=float(config['learning_rate']), lr_alpha=float(config.get('lr_alpha', 0.99)),
            min_overlap_for_angle=float(config.get('min_overlap_for_angle', 0.7)),
            yaw_augmentation=bool(config.get('yaw_augmentation', False)),
            data_root_folder=config.get('data_root_folder', ''))
  if 'training_seqs' in config:                                    # npz_files: the training files
    fp.update(training_seqs=str(config['training_seqs']), traindata_npzfile=None)
  else:
    fp.update(training_seqs=None, traindata_npzfile=config['traindata_npzfile'])
  if 'gradient_chunks' in config:          # only with the key, so that the fingerprints of other runs stay
    fp.update(gradient_chunks=config['gradient_chunks'])
  return _plain(fp)


def write_checkpoint(path, epochs, weights, accum, pairs, history, fingerprint):
  """The state after ``epochs`` completed epochs, in an .npz that loads without pickle: a temp file in the same
  directory, flushed to disk, then renamed over ``path``, so that ``path`` is always a whole checkpoint."""
  _, keys, pos, has_gauss, cached_gaussian = np.random.get_state()
  arrays = {'format_version': np.int64(CHECKPOINT_VERSION), 'epochs': np.int64(epochs),
            'accum': np.asarray(accum, np.float32),
            'rng_keys': np.asarray(keys, np.uint32), 'rng_pos': np.int64(pos), 'rng_has_gauss': np.int64(has_gauss),
            'rng_cached_gaussian': np.float64(cached_gaussian),
            'history': np.str_(json.dumps({k: history[k] for k in ('epoch_loss', 'batch_losses', 'validation')})),
            'fingerprint': np.str_(json.dumps(fingerprint, sort_keys=True))}
  for key, values in zip(('f1', 'f2', 'd1', 'd2'), pairs[:4]):
    arrays[key] = np.asarray(values, np.str_)
  arrays['overlap'], arrays['orientation'] = np.asarray(pairs[4]), np.asarray(pairs[5])
  for name, (k, b) in weights.items():                             # the keys of weights.save_npz
    arrays[name + '/kernel'] = np.asarray(k, np.float32)
    arrays[name + '/bias'] = np.asarray(b, np.float32)
  tmp = path + '.tmp'
  with open(tmp, 'wb') as f:
    np.savez(f, **arrays)
    f.flush()
    os.fsync(f.fileno())
  os.replace(tmp, path)


def read_checkpoint(path, fingerprint, no_epochs):
  """The state write_checkpoint stored at ``path``, checked against this run: its format version, the
  ``fingerprint`` of this config, its epoch count below ``no_epochs`` and its accumulators (finite, >= 0).  Returns
  a dict (epochs, weights, accum, rng, pairs, history); raises an Exception that names the problem."""
  try:
    with np.load(path, allow_pickle=False) as z:
      ck = {k: z[k] for k in z.files}
  except Exception as e:
    raise Exception('resume: cannot read the checkpoint %s: %s' % (path, e)) from e
  if 'format_version' not in ck or int(ck['format_version']) != CHECKPOINT_VERSION:
    raise Exception('resume: the checkpoint %s has format version %s; this code reads version %d'
                    % (path, ck['format_version'] if 'format_version' in ck else 'none', CHECKPOINT_VERSION))
  required = ('epochs', 'accum', 'rng_keys', 'rng_pos', 'rng_has_gauss', 'rng_cached_gaussian', 'history',
              'fingerprint', 'f1', 'f2', 'd1', 'd2', 'overlap', 'orientation')
  missing = [k for k in required if k not in ck]
  if missing:
    raise Exception('resume: the checkpoint %s lacks %s' % (path, ', '.join(missing)))
  saved = json.loads(str(ck['fingerprint']))
  for key in sorted(set(saved) | set(fingerprint)):
    a, b = saved.get(key), fingerprint.get(key)
    if a != b:
      if key == 'model' and isinstance(a, dict) and isinstance(b, dict):
        key = 'model.' + next(k for k in sorted(set(a) | set(b)) if a.get(k) != b.get(k))
      raise Exception('resume: config key %s differs from the run that wrote %s; a resumed run must keep the '
                      'keys that fix its trajectory' % (key, path))
  epochs = int(ck['epochs'])
  if epochs >= no_epochs:
    raise Exception('resume: the checkpoint %s holds %d completed epochs, no_epochs is %d: nothing to train'
                    % (path, epochs, no_epochs))
  accum = ck['accum']
  if accum.dtype != np.float32 or accum.ndim != 1:
    raise Exception('resume: the accumulators in %s are %s %s, not a float32 vector' % (path, accum.dtype,
                                                                                       accum.shape))
  bad = ~np.isfinite(accum) | (accum < 0)
  if bad.any():
    raise Exception('resume: %d Adagrad accumulators in %s are negative or not finite (first at %d)'
                    % (int(bad.sum()), path, int(np.argmax(bad))))
  history = json.loads(str(ck['history']))
  for stats in history['validation']:                              # JSON object keys are strings
    stats['orientation_rms'] = {float(k): v for k, v in stats['orientation_rms'].items()}
  names = sorted({k.split('/')[0] for k in ck if '/' in k})
  return {'epochs': epochs, 'accum': accum, 'history': history,
          'weights': {n: (ck[n + '/kernel'], ck[n + '/bias']) for n in names},
          'rng': ('MT19937', ck['rng_keys'], int(ck['rng_pos']), int(ck['rng_has_gauss']),
                  float(ck['rng_cached_gaussian'])),
          'pairs': tuple(ck[k].tolist() for k in ('f1', 'f2', 'd1', 'd2')) + (ck['overlap'], ck['orientation'])}


def _read_checkpoint_on_rank0(path, fingerprint, no_epochs, dp):
  """read_checkpoint on rank 0; every rank gets its contents, or raises its refusal."""
  if dp is None:
    return read_checkpoint(path, fingerprint, no_epochs)
  got = None
  if dp.rank == 0:
    try:
      got = read_checkpoint(path, fingerprint, no_epochs)
    except Exception as e:
      got = str(e)
  got = dp.broadcast(got)
  if isinstance(got, str):
    raise Exception(got)
  return got


def check_checkpoint_fits(ck, eng, whole_network, path):
  """Refuse a checkpoint whose layers, shapes or accumulator length differ from the handle's."""
  have = {n: (np.shape(k), np.shape(b)) for n, (k, b) in eng.get_weights().items()}
  saved = {n: (np.shape(k), np.shape(b)) for n, (k, b) in ck['weights'].items()}
  if sorted(have) != sorted(saved):
    raise Exception('resume: the checkpoint %s has the layers %s; the model has %s' % (path, sorted(saved),
                                                                                     sorted(have)))
  for name in sorted(have):
    if have[name] != saved[name]:
      raise Exception('resume: layer %s of the checkpoint %s has kernel / bias shapes %s; the model has %s'
                      % (name, path, saved[name], have[name]))
  n = eng.gradient_size(whole_network)
  if ck['accum'].size != n:
    raise Exception('resume: the checkpoint %s holds %d Adagrad accumulators; this flow trains %d'
                    % (path, ck['accum'].size, n))


class FrozenLeg:
  """The training step of 360OutputkLegsFixed: every distinct scan is encoded once by the frozen leg into a
  feature bank on the GPU; a step trains the overlap head on it."""

  def __init__(self, infer, keys, rotate_keys=None, image_bank=None, gradient_chunks=None):
    """``image_bank`` (yaw augmentation only: without it there is no image bank) None places the RIGHT scans'
    images on the GPU when they fit beside the largest step's working set, sharded over the GPUs of a node's
    data-parallel ranks or in pinned host memory otherwise (overlapnet_b200.image_bank); 'device', 'host' or
    'sharded' forces a placement.  All train the same bits.
    ``gradient_chunks`` (the config key) sizes that working set for a rank's largest chunk range."""
    logger.info('Encoding %d scans with the frozen leg ...', len(keys))
    self.eng = infer._engine
    self.bank, self.rows = _encode_bank(infer, keys)
    self.image_bank = None
    if rotate_keys:
      # Yaw augmentation: the images of the scans a step may rotate, and max_batch_scans scratch rows after the
      # bank that receive a step's rotated RIGHT volumes.
      dp = data_parallel.default_group()
      world = 1 if dp is None else dp.world
      b_share = _image_bank.share_pairs(self.eng.max_batch_pairs, world, gradient_chunks)
      n, B = len(self.rows), self.eng.max_batch_scans
      self.image_bank, self.images, self.image_rows = _image_bank.open_bank(
          infer, rotate_keys, image_bank, b_share, False, b_share, n + B, 'Image bank of the rotated RIGHT scans',
          _image_bank.parts_bytes(self.eng, False, world, gradient_chunks))
      if self.image_bank in _image_bank.STAGED:
        self.ring = _image_bank.StagingRing(self.eng, self.images, 2 * b_share)
      self.bank = torch.cat([self.bank, self.bank.new_empty((B,) + tuple(self.bank.shape[1:]))])
      self.scratch = torch.arange(n, n + B, dtype=torch.int32, device=self.eng.device)

  whole_network = False          # the layers the gradients cover (Engine.copy_gradients, adagrad_step_sum)
  ring = None                    # the image_bank.StagingRing of a host or sharded image bank

  def begin_epoch(self, spans, left, right, rotate_rows=None):
    """With a host or sharded bank: the steps this rank runs in the coming epoch, in order -- pairs [a, b) of the
    training pairs' RIGHT image rows ``rotate_rows`` (host array) -- whose images the ring then stages ahead of each
    step."""
    self.ring.plan([(rotate_rows[a:b],) for a, b in spans])

  def step(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, lr, rotate=None):
    """``rotate`` = (image rows, column shifts, (cos, sin)) of the batch's RIGHT scans, or None: the rotated
    images are encoded by the frozen leg into the scratch rows, which then stand in for ``right``."""
    loss = self.gradients(left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate)
    self.eng.adagrad_step(lr)
    return loss

  def gradients(self, left, right, gt_overlap, gt_orientation, min_overlap_for_angle, rotate=None, chunks=None):
    """``step`` without its update: the losses; the gradients stay in the handle (the data-parallel step).
    ``chunks`` = (offsets, parts): the gradients of each chunk [offsets[c], offsets[c + 1]) of the pairs go to
    parts[c] in one call (Engine.head_gradients_chunks), and the losses of each chunk are returned."""
    if rotate is not None:
      rows, shifts, rot = rotate
      images = self.images
      if self.ring is not None:                  # the next span begin_epoch planned, staged in the ring's slot
        images, (rows,) = self.ring.take()
      n, n0 = rows.numel(), len(self.rows)
      x = self.eng.gather_images(images, rows, shifts, rot)
      if self.ring is not None:
        self.ring.release()
      self.eng.leg(x, out=self.bank[n0:n0 + n])
      right = self.scratch[:n]
    if chunks is not None:
      return self.eng.head_gradients_chunks(self.bank, left, right, chunks[0], gt_overlap, gt_orientation,
                                            min_overlap_for_angle, out=chunks[1])[0]
    return self.eng.head_gradients(self.bank, left, right, gt_overlap, gt_orientation, min_overlap_for_angle)

  def evaluate(self, left, right):
    """(overlap, yaw) device tensors of the validation pairs with the current weights."""
    ov, yaw, _ = self.eng.heads(self.bank, left, right)
    return ov, yaw


def close_image_bank(flow):
  """Release a flow's sharded image bank (ShardedImageBank.close, collective); a host bank is released with its
  handle."""
  if getattr(flow, 'image_bank', None) == 'sharded':
    flow.images.close()


def train(config, device=None):
  """Run the training of training.py for a loaded YAML dict.  Returns a dict with the per-epoch
  losses, the batch losses, the validation statistics and the weight file name."""
  check_config(config)
  return run(config, device, FrozenLeg)


def run(config, device, flow):
  """The loop of training.py with ``flow`` (FrozenLeg or training_leg.WholeNetwork) making the steps.  Trains
  data-parallel over the ranks of the default process group when one with more than one rank is initialised
  (overlapnet_b200.data_parallel); only rank 0 then writes the log and the weight file."""
  from .infer import Infer
  dp = data_parallel.default_group()
  model = config['model']
  root = config.get('data_root_folder', '')
  imgpath = config.get('imgpath', root)
  out_dir = os.path.join(config['experiments_path'], config['testname'])
  handler = None
  if dp is None or dp.rank == 0:
    os.makedirs(out_dir, exist_ok=True)
    handler = logging.FileHandler(os.path.join(out_dir, 'training.log'),             # training.py:204-208
                                  mode='a' if config.get('resume', False) else 'w')
    handler.setFormatter(logging.Formatter(fmt='%(asctime)s %(message)s', datefmt='%H:%M:%S'))
    logger.addHandler(handler)
  if logger.level == logging.NOTSET or logger.level > logging.INFO:
    logger.setLevel(logging.INFO)
  made = []                 # the flow _train builds: its sharded image bank is closed here, also after an exception
  try:
    return _train(config, model, imgpath, out_dir, device, Infer, flow, dp=dp, made=made)
  finally:
    for steps in made:
      close_image_bank(steps)
    if handler is not None:
      logger.removeHandler(handler)
      handler.close()


def _train(config, model, imgpath, out_dir, device, Infer, flow, dp=None, made=None):
  """The loop; ``dp`` (a data_parallel.DataParallel) makes it data-parallel: the config's batch_size is the
  global batch, rank 0 makes every random draw a one-process run makes and hands the results to the other
  ranks, and each step is data_parallel's gradient sum.  The flow it builds is appended to ``made``."""
  weights_filename = os.path.join(out_dir, model['modelType'] + '_' + config['testname'] + '.weight')
  initial_lr = float(config['learning_rate'])
  lr_alpha = float(config.get('lr_alpha', 0.99))
  batch_size = int(config['batch_size'])
  no_batches_in_epoch = int(config['no_batches_in_epoch'])
  no_epochs = int(config['no_epochs'])
  no_test_pairs = int(config['no_test_pairs'])
  min_overlap_for_angle = float(config.get('min_overlap_for_angle', 0.7))
  yaw_augmentation = bool(config.get('yaw_augmentation', False))
  world, rank = (1, 0) if dp is None else (dp.world, dp.rank)
  gradient_chunks = check_gradient_chunks(config, world)
  resume = bool(config.get('resume', False))
  checkpoint = resume or bool(config.get('checkpoint', False))
  checkpoint_path = os.path.join(out_dir, CHECKPOINT)
  fingerprint = trajectory_fingerprint(config) if checkpoint else None
  resumed = _read_checkpoint_on_rank0(checkpoint_path, fingerprint, no_epochs, dp) if resume else None

  train_files, val_files = npz_files(config)
  logger.info('load training data ...')
  if resumed is not None:                                          # the saved run's pairs, in its order
    t_f1, t_f2, t_d1, t_d2, t_ov, t_or = resumed['pairs']
  elif dp is None:
    t_f1, t_f2, t_d1, t_d2, t_ov, t_or = evaluate.load_overlap_npz(train_files)
  else:                                                            # rank 0's shuffle
    t_f1, t_f2, t_d1, t_d2, t_ov, t_or = dp.broadcast(evaluate.load_overlap_npz(train_files) if dp.rank == 0
                                                      else None)
  n = min(len(t_ov), batch_size * no_batches_in_epoch)                                # training.py:275-286
  t_f1, t_f2, t_d1, t_d2, t_ov, t_or = t_f1[:n], t_f2[:n], t_d1[:n], t_d2[:n], t_ov[:n], t_or[:n]
  logger.info('load validation data ...')
  v_f1, v_f2, v_d1, v_d2, v_ov, v_or = evaluate.load_overlap_npz(val_files, shuffle=False)
  n_val = min(len(v_ov), no_test_pairs)                                                 # training.py:291-300
  v_f1, v_f2, v_d1, v_d2, v_ov, v_or = v_f1[:n_val], v_f2[:n_val], v_d1[:n_val], v_d2[:n_val], v_ov[:n_val], v_or[:n_val]

  cfg = dict(config)
  for key, default in CUE_DEFAULTS:
    cfg.setdefault(key, default)
  cfg['data_root_folder'] = imgpath
  cfg['infer_seqs'] = ''
  cfg['model'] = dict(model)
  cfg['model']['inputShape'] = list(model['inputShape'])
  if resumed is not None:                                          # the checkpoint's weights replace them
    cfg['pretrained_weightsfilename'] = ''
  infer = Infer(cfg, precision='fp32', device=device, max_batch_pairs=batch_size)
  eng = infer._engine
  width = infer.network_output_size
  if 'training_precision' in config:        # every rank, so that data-parallel ranks compute alike
    eng.set_train_precision(config['training_precision'])
    logger.info('Training precision: %s', config['training_precision'])
  if len(cfg['pretrained_weightsfilename']) > 0:
    logger.info('Load old weights from %s', cfg['pretrained_weightsfilename'])
  if resumed is not None:          # every rank; the weights first: ovn_finalize_weights resets the accumulators
    check_checkpoint_fits(resumed, eng, flow.whole_network, checkpoint_path)
    eng.load_weights(resumed['weights'])
    eng.set_train_state(resumed['accum'], flow.whole_network)
  elif dp is not None:             # one start for every rank (glorot_init draws from its own generator)
    start = dp.broadcast(eng.get_weights() if dp.rank == 0 else None)
    if dp.rank != 0:
      eng.load_weights(start)

  keys = set(zip(t_d1, t_f1)) | set(zip(t_d2, t_f2)) | set(zip(v_d1, v_f1)) | set(zip(v_d2, v_f2))
  chunk_kw = {} if gradient_chunks is None else {'gradient_chunks': gradient_chunks}
  steps = flow(infer, keys, set(zip(t_d2, t_f2)), **chunk_kw) if yaw_augmentation else flow(infer, keys, **chunk_kw)
  if made is not None:
    made.append(steps)
  rows = steps.rows
  dev = eng.device
  t_left = torch.tensor([rows[k] for k in zip(t_d1, t_f1)], dtype=torch.int32, device=dev)
  t_right = torch.tensor([rows[k] for k in zip(t_d2, t_f2)], dtype=torch.int32, device=dev)
  t_ov_d = torch.as_tensor(np.asarray(t_ov, np.float32), device=dev)
  t_or_d = torch.as_tensor(np.asarray(t_or).astype(np.int32), device=dev)
  v_left = torch.tensor([rows[k] for k in zip(v_d1, v_f1)], dtype=torch.int32, device=dev)
  v_right = torch.tensor([rows[k] for k in zip(v_d2, v_f2)], dtype=torch.int32, device=dev)

  n_batches = int(np.ceil(n / float(batch_size)))                  # len() of the Keras Sequence
  logger.info('Training loop, saving weights to %s', weights_filename)
  logger.info('  batch size is           : %d', batch_size)
  logger.info('  number of training pairs: %d', n)
  logger.info('  number of test pairs    : %d', n_val)
  if yaw_augmentation:
    W = eng.W
    pitch = augment.column_pitch(W, width)
    t_right_img = torch.tensor([steps.image_rows[k] for k in zip(t_d2, t_f2)], dtype=torch.int32, device=dev)
    logger.info('  rotation of training data: RIGHT images by a random multiple of %d columns (%d bins), labels '
                'moved', pitch, pitch * width // W)
  else:
    logger.info('  NO rotation of training data')
  staged = getattr(steps, 'image_bank', None) in _image_bank.STAGED
  if staged:                      # the image rows of the pairs (LEFT, RIGHT, rotated RIGHT) for begin_epoch's plans
    right_h = np.asarray([steps.image_rows[k] for k in zip(t_d2, t_f2)], np.int64)
    left_h = np.asarray([steps.image_rows[k] for k in zip(t_d1, t_f1)], np.int64) if steps.whole_network else None
    t_rows_h = (left_h, right_h, right_h if yaw_augmentation else None)
  local, parts = _step_buffers(dp, steps, eng, gradient_chunks)
  history = {'epoch_loss': [], 'batch_losses': [], 'validation': [], 'weights_filename': weights_filename}
  first_epoch = 0
  if resumed is not None:
    history.update(resumed['history'])
    first_epoch = resumed['epochs']
    if dp is None or dp.rank == 0:                                 # the draws continue where the saved run stopped
      np.random.set_state(resumed['rng'])
    logger.info('Resuming from %s after epoch %d of %d', checkpoint_path, first_epoch, no_epochs)
  for epoch in range(first_epoch, no_epochs):
    lr = learning_rate(epoch, initial_lr, lr_alpha)
    losses, sizes = [], []
    t_or_epoch, rotate = t_or_d, None
    shifts = perm = None
    if dp is None or dp.rank == 0:
      if yaw_augmentation:                                         # one rotation per training pair and epoch
        shifts = augment.sample_shifts(n, W, width)
      perm = np.random.permutation(n_batches)                      # Keras reshuffles a Sequence's batches
    if dp is not None:
      shifts, perm = dp.broadcast((shifts, perm))
    if yaw_augmentation:
      shifts_d = torch.from_numpy(shifts).to(dev)
      rot_d = torch.from_numpy(augment.rotation(shifts, W)).to(dev)
      t_or_epoch = augment.move_labels(t_or_d, shifts_d, W, width)
      rotate = (t_right_img, shifts_d, rot_d)
    batches = []                                                   # (first pair, pairs, this rank's plan) per step
    for b in perm:
      s0, s1 = b * batch_size, min(n, (b + 1) * batch_size)
      batches.append((s0, s1 - s0, data_parallel.step_plan(s1 - s0, world, rank, gradient_chunks)))
    if staged:                                                     # this rank's pairs of each step, in order
      steps.begin_epoch([(s0 + p.lo, s0 + p.hi) for s0, _, p in batches if p.hi > p.lo], *t_rows_h)
    for s0, size, plan in batches:
      loss = _step(dp, steps, eng, plan, local, parts, s0, t_left, t_right, t_ov_d, t_or_epoch, min_overlap_for_angle,
                   lr, rotate)
      losses.append(loss)
      sizes.append(size)
      logger.info('  epoch %d batch %d: loss %.6f (overlap %.6f, orientation %.6f)', epoch + 1, len(losses),
                  loss[0], loss[1], loss[2])
    epoch_loss = float(np.average([l[0] for l in losses], weights=sizes))
    history['epoch_loss'].append(epoch_loss)
    history['batch_losses'].append([l[0] for l in losses])

    logger.info('                  saving model weights ...')                          # training.py:346-349
    if dp is None or dp.rank == 0:
      save_weights(weights_filename, eng.get_weights())

    logger.info('  Evaluation on test data ...')                                       # training.py:352-415
    if dp is None:
      ov, yaw = steps.evaluate(v_left, v_right)
      eng.check()
      overlap = ov.cpu().numpy().astype(np.float64)
      argmax = 180 - yaw.cpu().numpy().astype(np.int64)           # yaw = 180 - argmax (infer.py:158)
    else:                                                          # a share per rank, gathered in rank order
      bounds, _ = data_parallel.shares(n_val, dp.world)
      lo, hi = bounds[dp.rank]
      ov, yaw = steps.evaluate(v_left[lo:hi], v_right[lo:hi])
      eng.check()
      mine = np.stack([ov.cpu().numpy().astype(np.float64), yaw.cpu().numpy().astype(np.float64)], axis=1)
      both = dp.gather_rows(mine, [b - a for a, b in bounds])
      overlap = both[:, 0]
      argmax = 180 - both[:, 1].astype(np.int64)
    diffs = np.abs(overlap - v_ov)
    stats = {'mean': float(np.mean(diffs)), 'max': float(np.max(diffs)),
             'rms': float(np.sqrt(np.mean(diffs * diffs))), 'learning_rate': float(lr),
             'orientation_rms': orientation_rms(overlap, argmax, np.asarray(v_or, np.float64), width)}
    history['validation'].append(stats)
    logger.info('  Evaluation on test data results: ')
    logger.info('           Evaluation: mean overlap difference:   %f', stats['mean'])
    logger.info('           Evaluation: max  overlap difference:   %f', stats['max'])
    logger.info('           Evaluation: RMS  overlap error        : %f', stats['rms'])
    for thr, rms in stats['orientation_rms'].items():
      logger.info('           Evaluation: orientation RMS (overlap > %.1f): %f', thr, rms)
    logger.info('iteration %d, batch/epoch loss: %.9f  /  %.9f', epoch + 1, losses[-1][0], epoch_loss)
    if checkpoint and (dp is None or dp.rank == 0):
      t0 = time.perf_counter()
      accum = eng.train_state(steps.whole_network).cpu().numpy()
      write_checkpoint(checkpoint_path, epoch + 1, eng.get_weights(), accum, (t_f1, t_f2, t_d1, t_d2, t_ov, t_or),
                       history, fingerprint)
      logger.info('  checkpoint after epoch %d written to %s in %.3f s', epoch + 1, checkpoint_path,
                  time.perf_counter() - t0)
  return history


def _step_buffers(dp, steps, eng, gradient_chunks):
  """The gradient parts of the flow ``steps`` for the steps that sum them (_step): (local, parts), this rank's parts
  [m, n] and every rank's all-gathered [world m, n] (one tensor on one process), with m = ceil(K / world) for
  gradient_chunks K and m = 1 without; (None, None) on one process without chunks, whose step is the flow's own."""
  if dp is None and gradient_chunks is None:
    return None, None
  world = 1 if dp is None else dp.world
  m = 1 if gradient_chunks is None else data_parallel.chunk_rows(gradient_chunks, world)
  size = eng.gradient_size(steps.whole_network)
  if gradient_chunks is not None:
    ranges = data_parallel.shares(gradient_chunks, world)[0]
    logger.info('  gradient chunks: %d per batch, summed in chunk order; chunk ranges by rank: %s', gradient_chunks,
                ', '.join('%d: [%d, %d)' % (r, c0, c1) for r, (c0, c1) in enumerate(ranges)))
  if dp is not None:
    logger.info('  data-parallel over %d ranks: each step all-gathers %s gradients per rank', world,
                '%d' % size if gradient_chunks is None else '%d x %d' % (m, size))
  parts = torch.empty((world * m, size), dtype=torch.float32, device=eng.device)
  return (parts if dp is None else torch.empty((m, size), dtype=torch.float32, device=eng.device)), parts


def _step(dp, steps, eng, plan, local, parts, s0, t_left, t_right, t_ov, t_or, min_overlap_for_angle, lr, rotate):
  """One step of the batch whose first training pair is s0, under this rank's ``plan`` (data_parallel.step_plan):
  the pairs [s0 + lo, s0 + hi) of ``t_*`` and of ``rotate`` (the RIGHT image rows, shifts and rotations of every
  training pair, or None).  On one process without chunks that is the flow's own step.  Otherwise this rank's parts
  -- its share's gradients, or its chunks' in one gradient call -- go to ``local`` (_step_buffers); with several ranks
  they are all-gathered into ``parts`` and moved into chunk order; then every rank applies the Adagrad step of
  g = sum_k w_k g_k over the plan's weights.  Each part is what a call on its pairs alone computes, so a chunked step
  does not depend on how the chunks are spread over ranks.  Returns the flow's loss on one process without chunks,
  else the batch loss sum_k w_k loss_k (float64, in the parts' order)."""
  a, b = s0 + plan.lo, s0 + plan.hi
  pairs = [t[a:b] for t in (t_left, t_right, t_ov, t_or)]
  rotate = None if rotate is None else tuple(t[a:b] for t in rotate)
  if local is None:
    return steps.step(*pairs, min_overlap_for_angle, lr, rotate)
  k = 1 if plan.offsets is None else len(plan.offsets) - 1        # the parts this rank computes
  losses = [(0.0, 0.0, 0.0)] * k
  if b == a:                                                       # no pairs: weight 0, skipped by the sum
    local[:k].zero_()
  elif plan.offsets is None:
    losses = [steps.gradients(*pairs, min_overlap_for_angle, rotate)]
    eng.copy_gradients(steps.whole_network, out=local[0])
  else:
    losses = steps.gradients(*pairs, min_overlap_for_angle, rotate, chunks=(plan.offsets, local[:k]))
  losses = np.asarray(losses, np.float64).reshape(k, 3)
  if dp is not None:
    m = local.shape[0]
    dp.gather_flat(local.reshape(-1), parts.view(dp.world, -1))
    d0 = 0
    for r, c in enumerate(plan.counts):            # rank r's rows [r m, r m + c) to parts [d0, d0 + c)
      for j in range(c):                           # d0 <= r m: a row never lands on one still to be read
        if d0 + j != r * m + j:
          parts[d0 + j].copy_(parts[r * m + j])
      d0 += c
    losses = dp.gather_rows(losses, plan.counts)
  eng.adagrad_step_sum(parts[:len(plan.weights)], plan.weights, lr, steps.whole_network)
  return tuple(float(sum(w * l[i] for w, l in zip(plan.weights, losses))) for i in range(3))


def main(argv=None):
  """``python -m overlapnet_b200.training config.yml``; under ``torch.distributed.run`` with WORLD_SIZE > 1
  every rank joins the NCCL group and trains on GPU LOCAL_RANK, data-parallel."""
  argv = sys.argv[1:] if argv is None else argv
  logging.basicConfig(format='%(message)s', level=logging.INFO)
  configfilename = argv[0] if argv else 'network.yml'                                  # training.py:102-104
  logger.info('Using configuration file %s.', configfilename)
  config = load_config(configfilename)
  if config['model'].get('legsType') == '360OutputkLegs':      # the reference's default (network.yml:70)
    from . import training_leg
    train_fn = training_leg.train
  else:
    train_fn = train
  if int(os.environ.get('WORLD_SIZE', '1')) <= 1:
    train_fn(config)
    return
  import torch.distributed as dist
  device = int(os.environ.get('LOCAL_RANK', '0'))
  torch.cuda.set_device(device)
  dist.init_process_group('nccl')
  try:
    train_fn(config, device)
  finally:
    dist.destroy_process_group()


if __name__ == '__main__':
  main()
