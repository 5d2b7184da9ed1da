"""Time the surfel render of virtual scans on the GPU against the point render (DESIGN.md sections 4 and 5, "Surfel
renders"): virtual frames per second for each render alone and with the leg, at M = 1, 8 and 16 keyframes per frame
and 64 frames per call, the surfel_scatter share of the surfel render, and the time to build the bank of a
KITTI-00-sized lattice from points and from surfels.

  python tools/time_surfels.py [--steps 20] [--warmup 3] [--out result.json]

The scene is tools/time_render.py's: synthetic street scenes (synth.street_scene_cloud, seed 5) every 4 m along
y = 0, virtual frames at 1 m lattice points within 5 m of them.  "points" is ovn_render_preprocess_batch, "surfels"
ovn_render_surfels_preprocess_batch from the keyframes' surfel banks (built once, outside the timed window, at the
default parameters); the kernels are read from the profiler.  The bank builds are virtual_map.encode over
om.scenario()'s 4.4 km drive at M = 8 within 50 m, with 16 synthetic clouds reused along the drive; the surfel build
includes the keyframes' surfel banks.  Times are CUDA events around calls that end in a device synchronise.
Prints one JSON line with the card's name and power limit beside the numbers."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import gpu_timing                                                 # noqa: E402
from oracle import mcl as om                                      # noqa: E402
from overlapnet_b200 import synth, virtual_map                    # noqa: E402
from overlapnet_b200.infer import Infer                           # noqa: E402

MODEL = {'modelType': 'SiameseNetworkTemplate', 'legsType': '360OutputkLegs',
         'overlap_head': 'DeltaLayerConv1NetworkHead', 'orientation_head': 'CorrelationHead',
         'inputShape': [64, 900], 'leg_output_width': 360, 'strides_layer1': [2, 2],
         'additional_unsymmetric_layer3a': True}
FRAMES_PER_CALL = 64


def poses4(p, z=1.73):
  p = np.asarray(p, np.float64).reshape(-1, 3)
  T = np.tile(np.eye(4), (p.shape[0], 1, 1))
  c, s = np.cos(p[:, 2]), np.sin(p[:, 2])
  T[:, 0, 0], T[:, 0, 1], T[:, 1, 0], T[:, 1, 1] = c, -s, s, c
  T[:, 0, 3], T[:, 1, 3], T[:, 2, 3] = p[:, 0], p[:, 1], z
  return T


def main(argv=None):
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=3)
  ap.add_argument('--out', default=None)
  args = ap.parse_args(argv)
  gpu_timing.require_cuda('time_surfels')
  cfg = {'pretrained_weightsfilename': '', 'use_depth': True, 'use_normals': True, 'use_class_probabilities': False,
         'use_class_probabilities_pca': False, 'use_intensity': False, 'data_root_folder': '', 'infer_seqs': '',
         'batch_size': FRAMES_PER_CALL, 'model': MODEL}
  infer = Infer(cfg)
  eng = infer._engine
  out = {'card': gpu_timing.card(), 'frames_per_call': FRAMES_PER_CALL}

  # ---- per-call rates on a 80 m street ----------------------------------------------------------------------
  kp = poses4([(x, 0.0, 0.02 * x) for x in range(0, 81, 4)])
  clouds = [synth.street_scene_cloud(T, seed=5) for T in kp]
  batch = eng.upload_clouds(clouds)
  frames = virtual_map.lattice(kp, 1.0, 5.0)
  sel = np.random.default_rng(0).choice(frames.shape[0], FRAMES_PER_CALL, replace=False)
  vp = frames[np.sort(sel)]
  x = torch.empty((FRAMES_PER_CALL, eng.H, eng.W, eng.C), dtype=torch.float32, device=eng.device)
  fv = torch.empty((FRAMES_PER_CALL, eng.Wf, 128), dtype=torch.float32, device=eng.device)
  banks = eng.surfels(batch)
  rates = {}
  for m in (1, 8, 16):
    eo, ec, ep = virtual_map.entries(vp, kp, m, 50.0)
    row = {'entries': int(ec.size)}
    for name, fn, kernels in (
        ('points', lambda: eng.render_preprocess(batch, eo, ec, ep, out=x), ('render_scatter', 'render_gather')),
        ('surfels', lambda: eng.render_surfels_preprocess(banks, eo, ec, ep, out=x), ('surfel_scatter', 'surfel_gather'))):
      alone = gpu_timing.step_ms(lambda _: fn(), range(args.warmup + args.steps), args.warmup)
      both = gpu_timing.step_ms(lambda _: eng.leg(fn(), out=fv), range(args.warmup + args.steps), args.warmup)
      eng.profile_enable(True)
      for k in kernels:
        eng.profile_read(k)
      for _ in range(args.steps):
        fn()
      ks, kg = (eng.profile_read(k)[0] / args.steps for k in kernels)
      eng.profile_enable(False)
      r, b = float(np.median(alone)), float(np.median(both))
      row[name] = {'ms_per_call': round(r, 3), 'frames_per_s': round(FRAMES_PER_CALL / r * 1e3, 1),
                   'kernels_ms': {'scatter': round(ks, 3), 'gather': round(kg, 3)},
                   'scatter_share': round(ks / r, 3),
                   'with_leg_ms_per_call': round(b, 3),
                   'with_leg_frames_per_s': round(FRAMES_PER_CALL / b * 1e3, 1)}
    rates['M=%d' % m] = row
  leg = gpu_timing.step_ms(lambda _: eng.leg(x, out=fv), range(args.warmup + args.steps), args.warmup)
  out['leg_ms_per_call'] = round(float(np.median(leg)), 3)
  out['rates'] = rates

  # ---- the bank of a KITTI-00-sized lattice, from points and from surfels ---------------------------------------
  drive = om.scenario(spacing=4.0)
  kp_big = poses4(drive)
  src = [synth.street_scene_cloud(T, seed=5) for T in poses4([(4.0 * i, 0.0, 0.0) for i in range(16)])]
  big = [src[i % len(src)] for i in range(kp_big.shape[0])]
  lat = virtual_map.lattice(kp_big, 1.0, 5.0)
  out['bank'] = {'keyframes': int(kp_big.shape[0]), 'lattice_frames': int(lat.shape[0]), 'render_sources': 8,
                 'note': 'wall time of virtual_map.encode: entries on the host, cloud upload, surfel banks, render + '
                         'leg'}
  for name, surf in (('points', None), ('surfels', {})):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    bank = virtual_map.encode(infer, big, kp_big, lat, 8, 50.0, surfels=surf)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    out['bank'][name] = {'seconds': round(t1 - t0, 2), 'frames_per_s': round(lat.shape[0] / (t1 - t0), 1)}
    del bank
  line = json.dumps(out)
  print(line)
  if args.out:
    with open(args.out, 'w') as f:
      f.write(line + '\n')
  return out


if __name__ == '__main__':
  main()
