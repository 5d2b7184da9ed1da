"""Time robust pose-graph optimization on the GPU (ovn_pgo_optimize_host): synthetic drives of n = 1101 (KITTI 07's
length) and 4541 nodes (KITTI 00's) with 0, 50 and 500 loops, at 1, 8 and 132 graphs per launch.  Reports ms per
launch, ms per graph, graphs/s, the LM trials and CG iterations per graph, and the float64 SciPy oracle's time on
the same graph in the same run; and the time `--close-loops` adds to lcd_eval.evaluate_clouds on a 64-scan
street-scene loop (tools/time_icp.py's sequence).

  python tools/time_pgo.py [--repeats 3] [--out result.json]

``call_ms`` is gpu_timing.step_ms around one whole synchronous call (the host checks and CSR build, the copies in and
out, and the kernel); ``kernel_ms`` is the k_pgo_graphs launch alone, from the library's profiling events
("pgo_graphs").  Both are medians of ``--repeats`` calls after one warm-up call of the same shape.  ``--skip``
drops rows given as n:loops (e.g. 4541:500).  Prints one JSON line with the card's name and power limit beside the
numbers."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import gpu_timing                                                 # noqa: E402
import time_icp                                                   # noqa: E402
from oracle import pose_graph as P                                # noqa: E402
from overlapnet_b200 import lcd_eval, synth                       # noqa: E402
from overlapnet_b200.engine import Engine                         # noqa: E402


def time_close_loops(repeats):
  """Seconds of evaluate_clouds with register and with close_loops on the 64-scan loop, alternating, median of each."""
  import copy
  import tempfile
  import torch
  from oracle import network as N
  from overlapnet_b200 import weights as W
  from overlapnet_b200.infer import Infer
  clouds, poses = time_icp.loop_sequence()
  with tempfile.TemporaryDirectory() as tmp:
    wpath = os.path.join(tmp, 'weights.npz')
    W.save_npz(wpath, N.glorot_weights(4, time_icp.MODEL, seed=5))
    cfg = {'pretrained_weightsfilename': wpath, 'use_depth': True, 'use_normals': True,
           'use_class_probabilities': False, 'use_class_probabilities_pca': False, 'use_intensity': False,
           'data_root_folder': tmp, 'infer_seqs': '07', 'batch_size': 16, 'model': copy.deepcopy(time_icp.MODEL)}
    t = {False: [], True: []}
    for rep in range(repeats + 1):
      for close in (False, True):
        infer = Infer(copy.deepcopy(cfg))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s, _ = lcd_eval.evaluate_clouds(infer, clouds, poses, top_k=3, exclude_frames=10, exclude_distance=20.0,
                                        register=True, close_loops=close)
        torch.cuda.synchronize()
        if rep:                                                   # the first round warms up both
          t[close].append(time.perf_counter() - t0)
  reg, close = float(np.median(t[False])), float(np.median(t[True]))
  return {'scans': len(clouds), 'evaluate_register_s_median': round(reg, 3),
          'evaluate_close_loops_s_median': round(close, 3), 'close_loops_overhead_s': round(close - reg, 3),
          'pose_graph': s['pose_graph']}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--repeats', type=int, default=3)
  ap.add_argument('--skip', default='', help='comma-separated n:loops rows to leave out')
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  gpu_timing.require_cuda('time_pgo')
  skip = {tuple(int(v) for v in r.split(':')) for r in args.skip.split(',') if r}
  eng = Engine(precision='fp32', max_batch_scans=1, max_batch_pairs=1)
  rows = []
  for n in (1101, 4541):
    for loops in (0, 50, 500):
      if (n, loops) in skip:
        continue
      g, _ = synth.pose_graph_scene(n, loops, seed=n + loops)
      t0 = time.perf_counter()
      ref = P.optimize(g)
      oracle_s = time.perf_counter() - t0
      for batch in (1, 8, 132):
        graphs = [g] * batch
        box = {}
        eng.profile_enable(True)

        def call(_):
          box['out'] = eng.pose_graph(graphs)

        kernel = []
        ms = []
        for i in range(args.repeats + 1):
          ms += gpu_timing.step_ms(call, [i], 0)
          kernel.append(eng.profile_read('pgo_graphs')[0])
        eng.profile_enable(False)
        call_ms, kernel_ms = float(np.median(ms[1:])), float(np.median(kernel[1:]))
        r = box['out'][0]
        rows.append({'n': n, 'loops': loops, 'graphs': batch, 'call_ms': call_ms, 'kernel_ms': kernel_ms,
                     'kernel_ms_per_graph': kernel_ms / batch, 'graphs_per_s': 1e3 * batch / call_ms,
                     'trials': r['iterations'], 'accepted': r['accepted'], 'cg_iterations': r['cg_iterations'],
                     'status': r['status'], 'oracle_s': oracle_s, 'oracle_trials': ref['iterations'],
                     'oracle_status': ref['status']})
        print(json.dumps(rows[-1]), file=sys.stderr)
  eng.close()
  result = {'tool': 'time_pgo', 'card': gpu_timing.card(), 'rows': rows, 'close_loops': time_close_loops(args.repeats)}
  line = json.dumps(result)
  print(line)
  if args.out:
    with open(args.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
