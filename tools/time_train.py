"""Step times of the training flows, one subcommand per measurement.  The card (name, power limit, maximum SM clock)
is read in the same run and printed with every timing, because it is part of the number.

Every subcommand but the two image-bank ones times 16-pair steps on one synthetic set-up (Synthetic): an fp32 handle
at C = 4 with s_conv3a and Glorot weights, a 64-row bank and WARMUP + STEPS batches drawn from default_rng(0).  Each
step is timed alone (CUDA events, then a synchronise), and a timing is the median of the STEPS steps after WARMUP
warm-up steps.  Where a subcommand compares configurations, its rounds alternate them in one command.

  python tools/time_train.py step [--flow frozen_leg|whole_network] [--yaw-augmentation] [--training-precision P]
  python tools/time_train.py precision [--rounds R]
  python tools/time_train.py chunks [--rounds R]
  python tools/time_train.py dp
  python tools/time_train.py image-bank [--out results.json]
  python tools/time_train.py sharded-bank [--out results.json]

`python tools/time_train.py <subcommand> --help` says what each one measures."""
import argparse
import functools
import inspect
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import gpu_timing
from overlapnet_b200 import augment, data_parallel, image_bank, synth, training, training_leg
from overlapnet_b200 import weights as W
from overlapnet_b200.engine import Engine

MODEL = {'additional_unsymmetric_layer3a': True, 'strides_layer1': [2, 2]}
PAIRS, BANK, WARMUP, STEPS, ROUNDS = 16, 64, 3, 20, 3
FLOWS = ('frozen_leg', 'whole_network')
PRECISIONS = ('fp32', 'tf32x3')
# per training pair (DESIGN.md section 4): the frozen leg's heads 1.275 G MAC forward + 1.489 G MAC backward, the
# whole network 8.94 G MAC
GFLOP_PER_PAIR = {'frozen_leg': 5.53, 'whole_network': 17.9}
CHUNKS = (1, 2, 4, 8, 16)
USE = {4: {}, 25: {'use_class_probabilities': True, 'use_intensity': True}}
SCANS = 256                    # the image-bank subcommands' synthetic bank
RANKS = 2                      # the sharded bank's data-parallel ranks
SHARE = PAIRS // RANKS         # the pairs of a 16-pair step each of those ranks trains


def images(dev):
  return torch.from_numpy(synth.range_like_images(0, BANK, 4)).to(dev)


class Synthetic:
  """An fp32 handle with Glorot weights (seed 0), a bank and WARMUP + STEPS 16-pair batches of one flow.

  ``bank``: 'volumes', BANK + ``extra_rows`` random leg volumes (torch.rand, generator seed 0); 'images',
  synth.range_like_images(0, BANK, 4); 'leg', the leg's volumes of those images.  A batch is (left, right, overlap,
  orientation), drawn from ``rng`` = default_rng(0) in that order.  The indices are on the device; the labels are
  host arrays, which the gradient call uploads, or with ``labels_on_device`` device tensors."""

  def __init__(self, flow, bank, precision='fp32', extra_rows=0, labels_on_device=False):
    self.whole = flow == 'whole_network'
    self.eng = eng = Engine(model=MODEL, precision='fp32', max_batch_scans=16, max_batch_pairs=PAIRS)
    eng.load_weights(W.glorot_init(4, MODEL, seed=0))
    eng.set_train_precision(precision)
    dev = eng.device
    if bank == 'volumes':
      g = torch.Generator(device=dev).manual_seed(0)
      self.bank = torch.rand((BANK + extra_rows, 360, 128), device=dev, generator=g)
    else:
      self.bank = images(dev) if bank == 'images' else eng.leg(images(dev))
    self.gradients = eng.net_gradients if self.whole else eng.head_gradients
    self.adagrad_step = eng.net_adagrad_step if self.whole else eng.adagrad_step
    self.rng = np.random.default_rng(0)
    self.batches = []
    for _ in range(WARMUP + STEPS):
      li = torch.from_numpy(self.rng.integers(0, BANK, PAIRS).astype(np.int32)).to(dev)
      ri = torch.from_numpy(self.rng.integers(0, BANK, PAIRS).astype(np.int32)).to(dev)
      ov, yaw = self.rng.uniform(0, 1, PAIRS).astype(np.float32), self.rng.integers(0, 360, PAIRS).astype(np.int32)
      if labels_on_device:
        ov, yaw = torch.from_numpy(ov).to(dev), torch.from_numpy(yaw).to(dev)
      self.batches.append((li, ri, ov, yaw))

  def plain(self, batch, lr=1e-6):
    """The flow's own step: the gradients of the batch and the Adagrad step."""
    self.gradients(self.bank, *batch, 0.7)
    self.adagrad_step(lr)

  def share(self, batch, lo, hi, out):
    """The gradients of pairs [lo, hi) of the batch, copied into ``out`` (ovn_copy_gradients)."""
    self.gradients(self.bank, *(t[lo:hi] for t in batch), 0.7)
    self.eng.copy_gradients(self.whole, out=out)


# ---- step, precision ----------------------------------------------------------------------------------------------
def yaw_step(s, lr):
  """The step of ``yaw_augmentation: True``, with the shifts of np.random.seed(0)."""
  eng, dev = s.eng, s.eng.device
  np.random.seed(0)
  shifts = augment.sample_shifts(PAIRS, 900, 360)
  sh, rot = torch.from_numpy(shifts).to(dev), torch.from_numpy(augment.rotation(shifts, 900)).to(dev)
  if s.whole:
    batch = torch.empty((2 * PAIRS,) + tuple(s.bank.shape[1:]), dtype=torch.float32, device=dev)
    pairs = torch.arange(2 * PAIRS, dtype=torch.int32, device=dev)

    def step(b):
      li, ri, ov, yaw = b
      eng.gather_images(s.bank, li, out=batch[:PAIRS])
      eng.gather_images(s.bank, ri, sh, rot, out=batch[PAIRS:])
      eng.net_gradients(batch, pairs[:PAIRS], pairs[PAIRS:], ov, yaw, 0.7)
      eng.net_adagrad_step(lr)
  else:
    imgs = images(dev)
    scratch = torch.arange(BANK, BANK + PAIRS, dtype=torch.int32, device=dev)

    def step(b):
      li, ri, ov, yaw = b
      eng.leg(eng.gather_images(imgs, ri, sh, rot), out=s.bank[BANK:])
      eng.head_gradients(s.bank, li, scratch, ov, yaw, 0.7)
      eng.adagrad_step(lr)
  return step


def time_step(flow, yaw_aug=False, precision='fp32'):
  """The timing of one flow's step, as the step subcommand prints it."""
  whole = flow == 'whole_network'
  s = Synthetic(flow, 'images' if whole else 'volumes', precision, extra_rows=PAIRS if yaw_aug and not whole else 0)
  lr = 1e-6 if whole else 1e-3
  ms = gpu_timing.step_ms(yaw_step(s, lr) if yaw_aug else functools.partial(s.plain, lr=lr), s.batches, WARMUP)
  s.eng.close()
  res = dict({'card': gpu_timing.card(), 'training_precision': precision, 'yaw_augmentation': yaw_aug,
              'pairs_per_step': PAIRS, 'steps': STEPS}, **gpu_timing.summary(ms))
  med = float(np.median(ms))
  res['pairs_per_s'] = round(PAIRS / med * 1e3, 1)
  res['tflops'] = round(PAIRS * GFLOP_PER_PAIR[flow] / med, 3)
  if precision == 'tf32x3':             # three MMAs per product
    res['tflops_issued'] = round(3 * res['tflops'], 3)
  return res


def deviation(flow):
  """Losses and per-layer gradient deviation of tf32x3 from fp32 on the first timed batch of ``flow``'s step."""
  s = Synthetic(flow, 'images' if flow == 'whole_network' else 'volumes')
  names = s.eng.layers if s.whole else ('c_conv1', 'c_conv2', 'c_conv3', 'overlap_output')
  out = {}
  for p in PRECISIONS:
    s.eng.set_train_precision(p)
    out[p] = s.gradients(s.bank, *s.batches[WARMUP], 0.7), s.eng.get_gradients(names)
  s.eng.close()
  (l32, g32), (l3, g3) = out['fp32'], out['tf32x3']
  res = {'flow': flow, 'loss_fp32': l32, 'loss_tf32x3': l3,
         'loss_rel_dev': [abs(a - b) / abs(a) if a else abs(b) for a, b in zip(l32, l3)], 'grad_rel_dev': {}}
  for name in names:
    res['grad_rel_dev'][name] = [float(np.abs(g3[name][i] - g32[name][i]).max() / np.abs(g32[name][i]).max())
                                 for i in range(2)]
  return res


def cmd_step(a):
  """One flow's 16-pair step, reported as ms per step, pairs/s and achieved TFLOP/s against the GFLOP per training
  pair (5.53 for the frozen leg's heads, 17.9 for the whole network, DESIGN.md section 4).

    frozen_leg     ovn_head_gradients + ovn_head_adagrad_step on random leg volumes
    whole_network  ovn_net_gradients + ovn_net_adagrad_step on synthetic images

  --yaw-augmentation times the step of ``yaw_augmentation: True``.  The frozen leg gathers the 16 RIGHT images,
  rolled and rotated (ovn_gather_images), encodes them with the fp32 leg into scratch rows after the bank, and trains
  the heads on those rows; its TFLOP/s count the heads only.  The whole network gathers the 16 LEFT and the 16 rolled
  and rotated RIGHT images into a 32-image batch that ovn_net_gradients trains on.

  --training-precision tf32x3 times the 3xTF32 tensor-core step (Engine.set_train_precision); tflops_issued counts
  its three MMAs per product."""
  print(json.dumps(time_step(a.flow, a.yaw_augmentation, a.training_precision)))


def cmd_precision(a):
  """Both flows' steps at training precision fp32 and tf32x3, each on a fresh handle, alternated over --rounds
  rounds.  Then the deviation between the two precisions on the batch each flow's step timing draws first after its
  warm-up: the three losses, and per layer max |g_tf32x3 - g_fp32| / max |g_fp32|, both computed on one handle at
  the initial weights (the timed runs reach that batch after their warm-up Adagrad steps, at other weights).  One
  JSON line per timing and per flow's deviation."""
  for r in range(a.rounds):
    for flow in FLOWS:
      for p in PRECISIONS:
        print(json.dumps(dict(time_step(flow, False, p), flow=flow, round=r)), flush=True)
  for flow in FLOWS:
    print(json.dumps(deviation(flow)), flush=True)


# ---- chunks -------------------------------------------------------------------------------------------------------
def chunk_timings(flow, precision, card, rnd):
  s = Synthetic(flow, 'images' if flow == 'whole_network' else 'volumes', precision, labels_on_device=True)
  eng = s.eng
  chunked = eng.net_gradients_chunks if s.whole else eng.head_gradients_chunks
  parts = torch.empty((max(CHUNKS), eng.gradient_size(s.whole)), dtype=torch.float32, device=eng.device)

  def chunks(k):
    bounds, weights = data_parallel.shares(PAIRS, k)
    offsets = [a for a, _ in bounds] + [PAIRS]

    def run(batch):
      li, ri, ov, yaw = batch
      chunked(s.bank, li, ri, offsets, ov, yaw, 0.7, out=parts[:k])
      eng.adagrad_step_sum(parts[:k], weights, 1e-6, s.whole)
    return run

  def separate(k):
    bounds, weights = data_parallel.shares(PAIRS, k)

    def run(batch):
      for c, (a, b) in enumerate(bounds):
        s.share(batch, a, b, parts[c])
      eng.adagrad_step_sum(parts[:k], weights, 1e-6, s.whole)
    return run

  modes = [('plain', 1, s.plain)] + [('chunks', k, chunks(k)) for k in CHUNKS] + \
          [('separate', k, separate(k)) for k in CHUNKS if k > 1]
  out = []
  for mode, k, fn in modes:
    ms = gpu_timing.step_ms(fn, s.batches, WARMUP)
    out.append(dict({'card': card, 'round': rnd, 'flow': flow, 'training_precision': precision, 'mode': mode,
                     'chunks': k, 'pairs_per_step': PAIRS, 'steps': STEPS}, **gpu_timing.summary(ms)))
  eng.check()
  eng.close()
  return out


def cmd_chunks(a):
  """Step time of ``gradient_chunks`` (overlapnet_b200.training, DESIGN.md section 6) for both flows at training
  precision fp32 and tf32x3, every configuration alternated over --rounds rounds:

    plain       the flow's step: ovn_head_gradients / ovn_net_gradients + ovn_head_adagrad_step /
                ovn_net_adagrad_step
    chunks K    ovn_*_gradients_chunks over the 16 pairs in K chunks + ovn_adagrad_step_sum of the K parts
    separate K  K one-chunk calls, each followed by ovn_copy_gradients, + ovn_adagrad_step_sum: what the chunked
                call replaces"""
  card = gpu_timing.card()
  for r in range(a.rounds):
    for flow in FLOWS:
      for p in PRECISIONS:
        for line in chunk_timings(flow, p, card, r):
          print(json.dumps(line), flush=True)


# ---- dp -----------------------------------------------------------------------------------------------------------
def dp_setup(kind, world=1):
  """The dp subcommand's set-up of one flow ('frozen': head gradients on the leg's volumes of the images; 'whole': the
  whole network on the images), and max(world, 2) rows of random gradient parts drawn after the batches."""
  whole = kind == 'whole'
  s = Synthetic('whole_network' if whole else 'frozen_leg', 'images' if whole else 'leg', labels_on_device=True)
  n = s.eng.gradient_size(whole)
  parts = torch.from_numpy((s.rng.standard_normal((max(world, 2), n)) * 1e-6).astype(np.float32)).to(s.eng.device)
  return s, parts


def dp_median(s, fn):
  return round(float(np.median(gpu_timing.step_ms(fn, s.batches, WARMUP))), 3)


def dp_steps(s, parts):
  def sum1(batch):
    s.share(batch, 0, PAIRS, parts[0])
    s.eng.adagrad_step_sum(parts[:1], [1.0], 1e-6, s.whole)

  def share8(batch):
    s.share(batch, 0, PAIRS // 2, parts[0])
    s.eng.adagrad_step_sum(parts[:2], [0.5, 0.5], 1e-6, s.whole)
  return {'plain': s.plain, 'sum1': sum1, 'share8': share8}


def dp_rank(kind, rank, world):
  """Rank ``rank``'s median time of the whole data-parallel step of a 16-pair global batch (spawned ranks)."""
  s, parts = dp_setup(kind, world)
  parts = parts[:world]
  dp = data_parallel.DataParallel()
  bounds, weights = data_parallel.shares(PAIRS, world)
  lo, hi = bounds[rank]
  grad = torch.empty((parts.shape[1],), dtype=torch.float32, device=s.eng.device)

  def step(batch):
    s.share(batch, lo, hi, grad)
    dp.gather_flat(grad, parts)
    s.eng.adagrad_step_sum(parts, weights, 1e-6, s.whole)
  return dp_median(s, step)


def cmd_dp(a):
  """Step times of data-parallel training (overlapnet_b200.data_parallel) for both flows, the frozen leg's heads on
  the leg's volumes of the images, three rounds alternated:

    plain   the one-GPU step of 16 pairs: ovn_head_gradients / ovn_net_gradients + the Adagrad step
    sum1    the same 16 pairs through the data-parallel path at world size 1: the gradients, ovn_copy_gradients and
            ovn_adagrad_step_sum with one part (the world-1 overhead of the step)
    share8  one rank's compute of a 16-pair global batch at world size 2: the gradients of 8 pairs, the copy and a
            two-part ovn_adagrad_step_sum (the all-gather is not in it)

  With two or more visible GPUs it also times the whole data-parallel step of a 16-pair global batch at world sizes
  2 .. G (spawned ranks, NCCL all_gather_into_tensor), on rank 0."""
  res = {'card': gpu_timing.card(), 'global_batch_pairs': PAIRS, 'steps': STEPS, 'rounds': ROUNDS,
         'ms_per_step_median': {}}
  benches = {kind: dp_setup(kind) for kind in ('frozen', 'whole')}
  for _ in range(ROUNDS):
    for kind, (s, parts) in benches.items():
      for mode, fn in dp_steps(s, parts).items():
        res['ms_per_step_median'].setdefault('%s/%s' % (kind, mode), []).append(dp_median(s, fn))
  for s, _ in benches.values():
    s.eng.close()
  gpus = torch.cuda.device_count()
  if gpus >= 2:
    res['nccl_ms_per_step_median'] = {}
    for kind in ('frozen', 'whole'):
      for world in range(2, gpus + 1):
        res['nccl_ms_per_step_median']['%s/world%d' % (kind, world)] = \
            gpu_timing.spawn_ranks(functools.partial(dp_rank, kind), world, 'nccl')
  else:
    res['nccl_ms_per_step_median'] = 'not measured: %d visible GPU' % gpus
  print(json.dumps(res))


# ---- image-bank, sharded-bank -------------------------------------------------------------------------------------
class SyntheticInfer:
  """What the flows read of overlapnet_b200.infer.Infer, over an in-memory bank: the handle, the cue loader
  (``_prepare_inputs``) and the frozen leg's encoder."""

  def __init__(self, eng, images):
    self._engine, self.images, self.seq = eng, images, None

  def _prepare_inputs(self, names):
    return self.images[[int(n) for n in names]]

  def _create_feature_volumes_device(self, names):
    dev = self._engine.device
    return torch.cat([self._engine.leg(torch.from_numpy(self._prepare_inputs(names[s:s + 16])).to(dev))
                      for s in range(0, len(names), 16)])


def bank_engine(C):
  """The image-bank subcommands' fp32 handle at C = 4 or 25 and its SCANS random images (default_rng(C))."""
  eng = Engine(use=USE[C], model=MODEL, precision='fp32', max_batch_scans=16, max_batch_pairs=PAIRS)
  assert eng.C == C, eng.C
  eng.load_weights(W.glorot_init(C, MODEL, seed=0))
  return eng, np.random.default_rng(C).random((SCANS, eng.H, eng.W, C), dtype=np.float32)


def staged_steps(eng, imgs, legs, placement, pairs, seed):
  """WARMUP + STEPS steps of ``pairs`` pairs of the training flow itself ('whole', or 'frozen' with yaw
  augmentation) with its image bank on ``placement``, pairs drawn from default_rng(seed), timed back to back
  (gpu_timing.back_to_back_ms).  Returns the flow, the step times and, with a staged bank, the distinct images
  staged per step, both after the warm-up."""
  infer = SyntheticInfer(eng, imgs)
  keys = {('00', '%06d' % i) for i in range(SCANS)}
  yaw = legs == 'frozen'
  if yaw:
    flow = training.FrozenLeg(infer, keys, keys, image_bank=placement)
  else:
    flow = training_leg.WholeNetwork(infer, keys, image_bank=placement)
  rng = np.random.default_rng(seed)
  n = (WARMUP + STEPS) * pairs
  left_h, right_h = rng.integers(0, SCANS, n), rng.integers(0, SCANS, n)
  dev = eng.device
  left, right = torch.from_numpy(left_h.astype(np.int32)).to(dev), torch.from_numpy(right_h.astype(np.int32)).to(dev)
  ov = torch.from_numpy(rng.uniform(0, 1, n).astype(np.float32)).to(dev)
  orient = torch.from_numpy(rng.integers(0, 360, n).astype(np.int32)).to(dev)
  rotate = None
  if yaw:
    shifts = augment.sample_shifts(n, eng.W, eng.Wf)
    rotate = (right, torch.from_numpy(shifts).to(dev), torch.from_numpy(augment.rotation(shifts, eng.W)).to(dev))
  if flow.ring is not None:
    flow.ring.timing = True
    flow.begin_epoch([(s, s + pairs) for s in range(0, n, pairs)], left_h, right_h, right_h if yaw else None)
  rows = []

  def step(s):
    flow.step(left[s:s + pairs], right[s:s + pairs], ov[s:s + pairs], orient[s:s + pairs], 0.7, 1e-3,
              None if rotate is None else tuple(t[s:s + pairs] for t in rotate))
    if flow.ring is not None:
      rows.append(flow.ring.step_rows)
  ms = gpu_timing.back_to_back_ms(step, range(0, n, pairs), WARMUP)
  eng.check()
  return flow, ms, rows[WARMUP:]


def ring_fields(flow, rows, rows_key):
  """The staging ring's copy waits (StagingRing.wait_ms) and the mean of ``rows`` as ``rows_key``."""
  if flow.ring is None:
    return {}
  waits = flow.ring.wait_ms()[WARMUP:]
  return {'copy_wait_ms_per_step_median': round(float(np.median(waits)), 3),
          'copy_wait_ms_per_step_max': round(float(np.max(waits)), 3), rows_key: round(float(np.mean(rows)), 2)}


def h2d_rate(eng, imgs):
  """GB/s of one step's row copies (2 x PAIRS distinct random rows) from a pinned bank into a device slot."""
  host = image_bank.HostBank(eng, imgs.shape[0])
  host.images[:] = imgs
  slot = torch.empty((2 * PAIRS,) + imgs.shape[1:], dtype=torch.float32, device=eng.device)
  rng = np.random.default_rng(1)
  rows = [rng.choice(imgs.shape[0], 2 * PAIRS, replace=False) for _ in range(WARMUP + STEPS)]
  with torch.cuda.stream(torch.cuda.Stream(device=eng.device)):
    ms = gpu_timing.step_ms(lambda r: eng.stage_rows(host.images, r, slot), rows, WARMUP)
  host.close()
  med = float(np.median(ms))
  nbytes = 2 * PAIRS * imgs[0].nbytes
  return {'bytes_per_step': int(nbytes), 'ms_median': round(med, 3), 'gb_per_s': round(nbytes / med / 1e6, 2)}


def cmd_image_bank(a):
  """Step time of training with the image bank on the GPU against the image bank in pinned host memory
  (overlapnet_b200.image_bank): 16-pair steps of both flows -- the whole network, and the frozen leg with yaw
  augmentation -- at C = 4 and C = 25, the two placements alternated over three rounds.  The flows are the training
  flows themselves, built on a synthetic bank of 256 scans (random cues, Glorot weights, fp32), and their steps run
  back to back (gpu_timing.back_to_back_ms), so the ring's copies overlap the following steps as they do in
  training.

  Reported per run: ms per step (between events on the compute stream at the step boundaries); with the host bank
  also the milliseconds per step the compute stream waited on copy-done events and the distinct images staged per
  step; per C the realised host-to-device rate of one step's row copies (ovn_stage_rows from the pinned bank into a
  slot, CUDA events on the copy stream)."""
  results = {'card': gpu_timing.card(), 'pairs_per_step': PAIRS, 'scans': SCANS, 'steps': STEPS, 'warmup': WARMUP,
             'runs': []}
  for C in (4, 25):
    eng, imgs = bank_engine(C)
    results['h2d_C%d' % C] = h2d_rate(eng, imgs)
    print(json.dumps({'C': C, 'h2d': results['h2d_C%d' % C]}), flush=True)
    for legs in ('whole', 'frozen'):
      for r in range(ROUNDS):
        for placement in ('device', 'host'):
          flow, ms, rows = staged_steps(eng, imgs, legs, placement, PAIRS, 0)
          res = dict({'flow': legs, 'image_bank': flow.image_bank}, **gpu_timing.summary(ms))
          res['ms_per_step_mean'] = round(float(np.mean(ms)), 3)
          res.update(ring_fields(flow, rows, 'images_copied_per_step_mean'), C=C, round=r)
          if flow.image_bank != 'device':
            flow.images.close()
          results['runs'].append(res)
          print(json.dumps(res), flush=True)
    eng.close()
  print(json.dumps(results))
  if a.out:
    with open(a.out, 'w') as f:
      json.dump(results, f, indent=1)


def gather_rate(eng, bank):
  """k_gather_rows' bytes/s over one step's rows (2 x SHARE distinct random rows) into a device slot."""
  slot = torch.empty((2 * SHARE, eng.H, eng.W, eng.C), dtype=torch.float32, device=eng.device)
  rng = np.random.default_rng(1)
  eng.profile_enable(True)
  eng.profile_read('gather_rows')
  ms = []
  for i in range(WARMUP + STEPS):
    bank.stage(rng.choice(SCANS, 2 * SHARE, replace=False), slot)
    t, launches = eng.profile_read('gather_rows')                  # synchronises
    assert launches == 1, launches
    if i >= WARMUP:
      ms.append(t)
  eng.profile_enable(False)
  med = float(np.median(ms))
  nbytes = 2 * SHARE * eng.H * eng.W * eng.C * 4
  return {'bytes_per_step': int(nbytes), 'ms_median': round(med, 4), 'gb_per_s': round(nbytes / med / 1e6, 2)}


def sharded_rank(backend, rank, world):
  """One rank of the sharded-bank subcommand; rank 0 prints each run and returns every result."""
  results = {'card': gpu_timing.card(), 'backend': backend, 'ranks': world, 'pairs_per_step': PAIRS,
             'pairs_per_rank': SHARE, 'scans': SCANS, 'steps': STEPS, 'warmup': WARMUP, 'runs': []}
  for C in (4, 25):
    eng, imgs = bank_engine(C)
    for r in range(ROUNDS):
      for placement in ('device', 'sharded', 'host'):
        flow, ms, rows = staged_steps(eng, imgs, 'whole', placement, SHARE, rank)
        res = dict({'image_bank': flow.image_bank}, **gpu_timing.summary(ms))
        res.update(ring_fields(flow, rows, 'images_staged_per_step_mean'))
        if flow.image_bank == 'sharded':
          res['gather'] = gather_rate(eng, flow.images)
        res.update(C=C, round=r)
        if flow.image_bank != 'device':
          flow.images.close()                              # collective for the sharded bank
        results['runs'].append(res)
        if rank == 0:
          print(json.dumps(res), flush=True)
    eng.close()
  return results


def cmd_sharded_bank(a):
  """Step time of training the whole network with the image bank on the GPU, sharded over the GPUs of two
  data-parallel ranks, and in pinned host memory (overlapnet_b200.image_bank): 16-pair steps, 8 pairs per rank, at
  C = 4 and C = 25, the three placements alternated over three rounds.  The two ranks use NCCL on two GPUs when the
  machine has them, otherwise gloo with both ranks on one GPU.  The flow is training_leg.WholeNetwork itself, built
  on a synthetic bank of 256 scans (random cues, Glorot weights, fp32), with its steps run back to back as in
  training; each rank runs its own steps (the flow's step, without the gradient all-gather), so the numbers are
  those of the staging.

  Reported per run and rank 0: ms per step (events on the compute stream at the step boundaries), and with a staged
  bank the milliseconds per step the compute stream waited on copy-done events (StagingRing.wait_ms) and the
  distinct images staged per step; per C the realised rate of k_gather_rows over one step's rows (2 x 8 distinct
  random rows of the sharded bank, half of them in the peer's shard on average), from its CUDA events
  (ovn_profile_read) and the bytes it moved."""
  backend = 'nccl' if torch.cuda.device_count() >= 2 else 'gloo'
  results = gpu_timing.spawn_ranks(functools.partial(sharded_rank, backend), RANKS, backend)
  print(json.dumps(results))
  if a.out:
    with open(a.out, 'w') as f:
      json.dump(results, f, indent=1)


def main():
  p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  sub = p.add_subparsers(dest='command', required=True)

  def command(name, fn):
    c = sub.add_parser(name, description=inspect.cleandoc(fn.__doc__),
                       formatter_class=argparse.RawDescriptionHelpFormatter)
    c.set_defaults(run=fn)
    return c

  c = command('step', cmd_step)
  c.add_argument('--flow', choices=FLOWS, default='frozen_leg')
  c.add_argument('--yaw-augmentation', action='store_true')
  c.add_argument('--training-precision', choices=PRECISIONS, default='fp32')
  command('precision', cmd_precision).add_argument('--rounds', type=int, default=3)
  command('chunks', cmd_chunks).add_argument('--rounds', type=int, default=3)
  command('dp', cmd_dp)
  command('image-bank', cmd_image_bank).add_argument('--out')
  command('sharded-bank', cmd_sharded_bank).add_argument('--out')
  a = p.parse_args()
  gpu_timing.require_cuda('time_train.py ' + a.command)
  a.run(a)


if __name__ == '__main__':
  main()
