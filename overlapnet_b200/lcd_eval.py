"""Loop-closure evaluation of a trained model over a whole sequence, on the GPU: the experiment of the OverlapNet
paper, with the candidate rules of the reference's demo 3 (demo/demo3_lcd.py).

  python -m overlapnet_b200.lcd_eval [config/demo.yml] [--top-k K] [--exclude-frames 100] [--exclude-distance 50]
                                     [--gt-overlap 0.3] [--register [--min-inlier-fraction 0.3]] [--close-loops]
  torchrun --nproc_per_node G -m overlapnet_b200.lcd_eval ...            (the rows split over G GPUs)

The protocol (DESIGN.md section 7):
  poses       demo 3's LiDAR-frame poses T_velo_cam . pose0^-1 . pose . T_cam_velo (gt_files.kitti_poses_in_lidar);
              the travelled distance L_i accumulates the xy steps as lcd.LoopClosureDetector.step does.
  candidates  of query i: the scans j < i - exclude_frames with L_i - L_j > exclude_distance (gate_candidates'
              time and distance rules, without the covariance ellipse).  L is non-decreasing, so they are a
              prefix [0, c_i) (``past_prefix``).
  direction   LEFT = candidate j, RIGHT = query i, as demo 3 calls Infer.infer_multiple.
  records     the best k of each row, by overlap descending then index ascending, with the heads' yaw
              (Engine.heads_prefix_topk); empty slots are index -1, overlap -1, yaw 0.
  truth       g[i, j] = the overlap of row j of com_overlap_yaw(frame_idx = i) (gt.overlap_yaw_all_pairs);
              query i is positive when max_{j < c_i} g[i, j] > gt_overlap, and correct when g[i, j*_i] > gt_overlap
              for its top record j*_i.  Queries are the rows with c_i > 0.
  curve       for every distinct top score t, the queries with s_i >= t are declared (``metrics``).
  register    (opt-in) each top record is registered by point-to-plane ICP on the GPU (registration.register),
              LEFT = j*_i, RIGHT = i, once from the heads' yaw seed and once from the identity, against the
              ground-truth pose T_j*^-1 T_i; a success is a translation error < 0.5 m and a rotation error < 2 deg.
  close loops (opt-in, implies register) the odometry steps (i - 1, i) are registered by ICP from the identity, and
              five pose graphs over them (PGO_GRAPHS: no loops, verified, s >= F1max threshold, every top record,
              the correct records) are optimized in one launch (pose_graph.py); ground-truth poses only select the
              correct records and score the trajectories.  Untested on KITTI; scans about 1 m apart fit ICP's 2 m
              start distance.

Scans are encoded from the raw ``.bin`` files (Infer.encode_clouds); configs with class probabilities are
refused, since they would need a ``.label`` file per scan.  Results go to ``<experiments_path>/<testname>`` of
the network config: ``lcd_results.npz`` and ``lcd_summary.json``."""
import argparse
import json
import logging
import os
import sys

import numpy as np
import torch

from ._cabi import TOPK_MAX

logger = logging.getLogger('overlapnet_b200.lcd_eval')

OPERATING_POINT = 0.3          # demo3_lcd.py:119 declares a loop when max overlap > 0.3 (strict)
SUCCESS_TRANSLATION = 0.5      # metres: a registration within this and SUCCESS_ROTATION of the ground truth succeeds
SUCCESS_ROTATION = 2.0         # degrees
SEEDS = ('yaw', 'identity')    # the seed axis of the registration_* arrays


# ---- the candidate prefix ---------------------------------------------------------------------------------
def travelled_distance(traj):
  """L_i: the xy steps of ``traj`` (n, 2) accumulated one by one, as lcd.LoopClosureDetector.step does."""
  traj = np.asarray(traj, dtype=float)
  L = [0]
  for i in range(1, len(traj)):
    L.append(L[-1] + np.linalg.norm(traj[i] - traj[i - 1]))
  return np.asarray(L, dtype=float)


def past_prefix(traj, exclude_frames=100, exclude_distance=50):
  """c (int64 [n]): query i's candidates are the scans [0, c_i), those with j < i - exclude_frames and
  L_i - L_j > exclude_distance (lcd.gate_candidates' time and distance rules)."""
  L = travelled_distance(traj)
  n = L.size
  c = np.zeros(n, np.int64)
  for i in range(n):
    m = max(i - int(exclude_frames), 0)
    # L is non-decreasing, so L_i - L_j > d holds on a prefix of j: count it with the rule's own expression
    c[i] = int(np.count_nonzero(L[i] - L[:m] > exclude_distance))
  return c


def split_rows(c, world):
  """Contiguous row ranges [(lo, hi)] of equal sum of c, up to one row: rank r starts at the first row whose
  preceding sum reaches r * sum(c) / world."""
  c = np.asarray(c, np.int64)
  before = np.concatenate([[0], np.cumsum(c)])[:-1]
  total = int(c.sum())
  cuts = [0] + [int(np.searchsorted(before * world, r * total, side='left')) for r in range(1, world)] + [c.size]
  for r in range(1, world + 1):
    cuts[r] = max(cuts[r], cuts[r - 1])
  return [(cuts[r], cuts[r + 1]) for r in range(world)]


# ---- search and ground truth --------------------------------------------------------------------------------
def search(engine, bank, c, k, row_lo=0, row_hi=None):
  """Rows [row_lo, row_hi) of the causal search: each scan's best k records among its candidates [0, c_i).
  Returns host arrays (overlap f32, index i32, yaw i32), each [rows, k]."""
  row_hi = int(bank.shape[0]) if row_hi is None else int(row_hi)
  ov, idx, yaw = engine.heads_prefix_topk(bank, row_lo, row_hi, np.asarray(c)[row_lo:row_hi], k)
  engine.check()
  return ov.cpu().numpy(), idx.cpu().numpy(), yaw.cpu().numpy()


def ground_truth(clouds, poses, rows, c, top_index, width=360, local=False):
  """The ground truth of ``rows`` (one per query; ``c`` and ``top_index`` [rows, k] are theirs): a dict of
  best (float64: max_{j < c_i} g[i, j], -1 when c_i = 0), top_overlap (float64 [rows, k]: g at each record, -1 in
  an empty slot) and top_yaw_bin (int64 [rows, k]: the ground-truth yaw bin of each record, 0 in an empty slot).
  Only rows with candidates are computed, with gt.overlap_yaw_all_pairs; ``width``: the yaw bins' resolution
  (leg_output_width); ``local``: on this process only, even in a process group."""
  from . import gt
  rows = np.asarray(rows, np.int64)
  c = np.asarray(c, np.int64)
  k = top_index.shape[1]
  best = np.full(rows.size, -1.0)
  top_ov = np.full((rows.size, k), -1.0)
  top_bin = np.zeros((rows.size, k), np.int64)
  live = np.flatnonzero(c > 0)
  if live.size:
    if local:
      # the ranks of a node may share a GPU: each takes half of the free memory over the world size for the clouds
      budget = torch.cuda.mem_get_info()[0] // (2 * torch.distributed.get_world_size())
      res = gt._all_pairs_local(clouds, np.asarray(poses, np.float64), rows[live], width, budget, 0, 0)
    else:
      res = gt.overlap_yaw_all_pairs(clouds, poses, frames=rows[live], leg_output_width=width)
    if np.any(res.valid_num == 0):
      raise ZeroDivisionError('a query scan has no valid pixel (valid_num = 0)')
    g = res.counts.astype(np.int64) / res.valid_num.astype(np.int64)[:, None]    # as gt.all_pairs_rows divides
    for q, r in enumerate(live):
      best[r] = g[q, :c[r]].max()
      ok = top_index[r] >= 0
      top_ov[r, ok] = g[q, top_index[r, ok]]
      top_bin[r, ok] = res.yaw_bin[q, top_index[r, ok]]
  return {'best': best, 'top_overlap': top_ov, 'top_yaw_bin': top_bin}


# ---- metrics ------------------------------------------------------------------------------------------------
def metrics(top_overlap, top_index, gt_top_overlap, gt_best, gt_overlap=0.3, operating_point=OPERATING_POINT):
  """Precision-recall of the detector from the records (``top_overlap`` / ``top_index`` [rows, k]) and their
  ground truth (``gt_top_overlap`` [rows, k], ``gt_best`` [rows]).  Queries are the rows whose top record exists;
  a NaN score raises.  Returns (summary dict, curve dict of arrays over the thresholds, descending)."""
  top_overlap = np.asarray(top_overlap, np.float32)
  top_index = np.asarray(top_index)
  gt_top = np.asarray(gt_top_overlap, np.float64)
  query = top_index[:, 0] >= 0
  s = top_overlap[query, 0].astype(np.float64)
  if np.isnan(s).any():
    raise ValueError('a query has a NaN top overlap: the scores are poisoned')
  correct_k = (top_index[query] >= 0) & (gt_top[query] > gt_overlap)
  correct = correct_k[:, 0]
  positive = np.asarray(gt_best, np.float64)[query] > gt_overlap
  n_pos = int(positive.sum())
  thr = np.unique(s)[::-1]
  order = np.argsort(-s, kind='stable')
  tp_cum = np.cumsum(correct[order])
  # declared at threshold t: every query with s >= t, i.e. the first (number of scores >= t) of the descending order
  n_decl = np.searchsorted(-s[order], -thr, side='right')
  tp = tp_cum[n_decl - 1] if thr.size else np.zeros(0, np.int64)
  fp = n_decl - tp
  precision = np.where(n_decl > 0, tp / np.maximum(n_decl, 1), 1.0)
  recall = tp / n_pos if n_pos else np.full(thr.size, np.nan)
  if n_pos:
    ap = float(np.sum(np.diff(np.concatenate([[0.0], recall])) * precision))
    pr = precision + recall
    f1 = np.where(pr > 0, 2 * precision * recall / np.where(pr > 0, pr, 1), 0.0)
    b = int(np.argmax(f1)) if thr.size else -1
  else:
    ap, f1, b = float('nan'), np.full(thr.size, np.nan), -1
  op = s > operating_point
  op_tp = int((op & correct).sum())
  op_n = int(op.sum())
  summary = {
      'queries': int(query.sum()), 'positives': n_pos, 'average_precision': ap,
      'f1_max': float(f1[b]) if b >= 0 else float('nan'),
      'f1_max_threshold': float(thr[b]) if b >= 0 else float('nan'),
      'precision_at_f1_max': float(precision[b]) if b >= 0 else float('nan'),
      'recall_at_f1_max': float(recall[b]) if b >= 0 else float('nan'),
      'operating_point': operating_point,
      'precision_at_operating_point': op_tp / op_n if op_n else 1.0,
      'recall_at_operating_point': op_tp / n_pos if n_pos else float('nan'),
      'recall_at_1': float((positive & correct).sum()) / n_pos if n_pos else float('nan'),
      'recall_at_k': float((positive & correct_k.any(1)).sum()) / n_pos if n_pos else float('nan'),
      'k': int(top_index.shape[1]),
  }
  curve = {'threshold': thr, 'tp': tp.astype(np.int64), 'fp': fp.astype(np.int64), 'precision': precision,
           'recall': recall, 'f1': f1}
  return summary, curve


def true_positives_at(top_overlap, top_index, gt_top_overlap, threshold, gt_overlap=0.3):
  """The rows whose top record is declared at ``threshold`` (s_i >= t) and correct."""
  s = np.asarray(top_overlap)[:, 0]
  return np.flatnonzero((np.asarray(top_index)[:, 0] >= 0) & (s >= threshold) &
                        (np.asarray(gt_top_overlap)[:, 0] > gt_overlap))


def yaw_errors(engine, bank, rows, cand, gt_bin, width=360):
  """Circular yaw-bin errors of the pairs LEFT = bank[rows], RIGHT = bank[cand] (the direction of testing.py and
  the training labels), scored by one heads call, against the ground-truth bins ``gt_bin``."""
  from .evaluate import yaw_to_argmax
  if len(rows) == 0:
    return np.zeros(0, np.float64)
  _, yaw, _ = engine.heads(bank, torch.as_tensor(np.asarray(rows, np.int32)), torch.as_tensor(np.asarray(cand, np.int32)))
  engine.check()
  a = np.abs(yaw_to_argmax(yaw.cpu().numpy()).astype(float) - np.asarray(gt_bin, float))
  return np.minimum(a, width - a)                                  # evaluate.error_statistics' circular rule


# ---- registration of the top records --------------------------------------------------------------------------
def register_records(engine, clouds, poses, rows, top_index, top_yaw, params=None):
  """Register the top record of each of ``rows`` (LEFT = top_index[r, 0], RIGHT = rows[r]) twice in one call, from
  the yaw seed of top_yaw[r, 0] and from the identity.  Returns a dict of arrays over the rows, the seed axis in
  SEEDS order: pose [rows, 2, 4, 4], gt_pose [rows, 4, 4] (T_j*^-1 T_i), error [rows, 2, 2] (metres, degrees),
  inlier_fraction [rows, 2] (inliers over valid source pixels), rms [rows, 2], status / iterations [rows, 2] int32.
  A row without a record holds NaN, status -1 and 0 iterations."""
  from .evaluate import yaw_to_argmax
  from .registration import pose_error, register, seed_pose
  rows = np.asarray(rows, np.int64)
  n = rows.size
  out = {'pose': np.full((n, 2, 4, 4), np.nan), 'gt_pose': np.full((n, 4, 4), np.nan),
         'error': np.full((n, 2, 2), np.nan), 'inlier_fraction': np.full((n, 2), np.nan),
         'rms': np.full((n, 2), np.nan), 'status': np.full((n, 2), -1, np.int32),
         'iterations': np.zeros((n, 2), np.int32)}
  live = np.flatnonzero(np.asarray(top_index)[:, 0] >= 0) if n else np.zeros(0, np.int64)
  if live.size:
    left = np.asarray(top_index)[live, 0].astype(np.int64)
    right = rows[live]
    init = np.concatenate([seed_pose(yaw_to_argmax(np.asarray(top_yaw)[live, 0]), engine.Wf),
                           np.broadcast_to(np.eye(4), (live.size, 4, 4))])
    res = register(engine, clouds, np.concatenate([left, left]), np.concatenate([right, right]), init, params)
    gt = np.linalg.solve(poses[left], poses[right])
    m = live.size
    pose = np.stack([res['pose'][:m], res['pose'][m:]], 1)
    t_err, r_err = pose_error(pose, gt[:, None])
    out['pose'][live] = pose
    out['gt_pose'][live] = gt
    out['error'][live] = np.stack([t_err, np.rad2deg(r_err)], -1)
    for key in ('rms', 'status', 'iterations'):
      out[key][live] = np.stack([res[key][:m], res[key][m:]], 1)
    frac = res['inliers'] / np.maximum(res['valid'], 1).astype(np.float64)
    out['inlier_fraction'][live] = np.stack([frac[:m], frac[m:]], 1)
  return out


def registration_summary(top_overlap, top_index, gt_top_overlap, gt_best, tp_rows, error, inlier_fraction,
                         gt_overlap=0.3, min_inlier_fraction=0.3, operating_point=OPERATING_POINT):
  """The ``registration`` section of the summary: over the true positives ``tp_rows`` at F1max, the success rate
  from each seed and the yaw seed's median / max errors; and precision / recall at the operating point when a
  declared loop must also reach ``min_inlier_fraction`` from the yaw seed (``error`` [rows, 2, 2] and
  ``inlier_fraction`` [rows, 2] as register_records gives them)."""
  error = np.asarray(error, np.float64)
  tp_rows = np.asarray(tp_rows, np.int64)
  e = error[tp_rows]
  ok = (e[..., 0] < SUCCESS_TRANSLATION) & (e[..., 1] < SUCCESS_ROTATION)
  out = {'success_translation_m': SUCCESS_TRANSLATION, 'success_rotation_deg': SUCCESS_ROTATION,
         'min_inlier_fraction': min_inlier_fraction, 'true_positives': int(tp_rows.size)}
  for k, seed in enumerate(SEEDS):
    out['success_rate_' + seed] = float(ok[:, k].mean()) if tp_rows.size else float('nan')
  for k, what in enumerate(('translation_m', 'rotation_deg')):
    v = e[:, 0, k]
    out['median_error_%s_yaw' % what] = float(np.median(v)) if v.size else float('nan')
    out['max_error_%s_yaw' % what] = float(np.max(v)) if v.size else float('nan')
  top_index = np.asarray(top_index)
  query = top_index[:, 0] >= 0
  s = np.asarray(top_overlap, np.float64)[:, 0]
  correct = query & (np.asarray(gt_top_overlap, np.float64)[:, 0] > gt_overlap)
  n_pos = int((query & (np.asarray(gt_best, np.float64) > gt_overlap)).sum())
  declared = query & (s > operating_point) & (np.asarray(inlier_fraction, np.float64)[:, 0] >= min_inlier_fraction)
  tp = int((declared & correct).sum())
  out['precision_at_operating_point_verified'] = tp / int(declared.sum()) if declared.any() else 1.0
  out['recall_at_operating_point_verified'] = tp / n_pos if n_pos else float('nan')
  return out


# ---- closing the loops: ICP odometry and pose graphs ------------------------------------------------------------
PGO_GRAPHS = ('odometry', 'verified', 'f1_max', 'all_records', 'true_loops')   # the graph axis of the pgo_* arrays
VERIFIED_SCORE = 0.3           # a verified loop: s_i > VERIFIED_SCORE and the yaw seed's inlier fraction is high enough


def register_odometry(engine, clouds, poses, rows, params=None):
  """The odometry steps of ``rows``: each row i >= 1 registers (LEFT = i - 1, RIGHT = i) from the identity, in one
  registration.register call.  Returns pose [rows, 4, 4] (T_{i-1}^-1 T_i estimated), status [rows] int32 and error
  [rows, 2] (metres, degrees against the ground-truth step); row 0 holds NaN and status -1."""
  from .registration import pose_error, register
  rows = np.asarray(rows, np.int64)
  out = {'pose': np.full((rows.size, 4, 4), np.nan), 'status': np.full(rows.size, -1, np.int32),
         'error': np.full((rows.size, 2), np.nan)}
  live = np.flatnonzero(rows >= 1)
  if live.size:
    i = rows[live]
    res = register(engine, clouds, i - 1, i, np.broadcast_to(np.eye(4), (live.size, 4, 4)), params)
    t, r = pose_error(res['pose'], np.linalg.solve(poses[i - 1], poses[i]))
    out['pose'][live] = res['pose']
    out['status'][live] = res['status']
    out['error'][live] = np.stack([t, np.degrees(r)], -1)
  return out


def loop_sets(top_overlap, top_index, gt_top_overlap, inlier_fraction, f1_threshold, gt_overlap=0.3,
              min_inlier_fraction=0.3):
  """The loop edges of each graph of PGO_GRAPHS, as bool masks over the rows (a row's loop is its top record):
  none; verified (s_i > 0.3 and the yaw seed's inlier fraction >= min_inlier_fraction); s_i >= the F1max threshold;
  every top record; the correct records by ground truth (the upper bound)."""
  top_index = np.asarray(top_index)
  has = top_index[:, 0] >= 0
  s = np.asarray(top_overlap, np.float64)[:, 0]
  f1 = has & (s >= f1_threshold) if np.isfinite(f1_threshold) else np.zeros_like(has)
  return {'odometry': np.zeros_like(has),
          'verified': has & (s > VERIFIED_SCORE) & (np.asarray(inlier_fraction, np.float64)[:, 0] >= min_inlier_fraction),
          'f1_max': f1, 'all_records': has,
          'true_loops': has & (np.asarray(gt_top_overlap, np.float64)[:, 0] > gt_overlap)}


def loop_graphs(odometry_pose, top_index, loop_pose, masks):
  """One pose graph per mask (PGO_GRAPHS order) over every scan: the chain measures odometry_pose[1:], the loops
  (j*_i, i) of the masked rows measure loop_pose[i] (the yaw-seeded registration), with the default weights.  The
  initial poses compose the odometry from the identity; no ground-truth pose enters a graph."""
  from .pose_graph import chain_graph
  rows_all = np.arange(len(top_index))
  graphs = []
  for name in PGO_GRAPHS:
    rows = rows_all[masks[name]]
    edges = np.stack([np.asarray(top_index)[rows, 0], rows], 1)
    graphs.append(chain_graph(odometry_pose[1:], (edges, loop_pose[rows])))
  return graphs


def close_loops_graphs(engine, odometry_pose, top_index, loop_pose, masks):
  """Optimize the loop_graphs of ``masks`` in one Engine.pose_graph call.  Returns the pgo_* arrays: poses [G, n, 4, 4],
  loop_mask / loop_scale / loop_chi2 [G, rows] (NaN off-graph), status / iterations [G], cost [G, 2] (F before
  and after)."""
  from .pose_graph import optimize
  graphs = loop_graphs(odometry_pose, top_index, loop_pose, masks)
  res = optimize(engine, graphs)
  n = odometry_pose.shape[0]
  G = len(graphs)
  out = {'poses': np.stack([r['poses'] for r in res]), 'loop_mask': np.stack([masks[k] for k in PGO_GRAPHS]),
         'loop_scale': np.full((G, n), np.nan), 'loop_chi2': np.full((G, n), np.nan),
         'status': np.array([r['status'] for r in res], np.int32),
         'iterations': np.array([r['iterations'] for r in res], np.int32),
         'cost': np.array([[r['initial_cost'], r['final_cost']] for r in res])}
  for g, r in enumerate(res):
    rows = np.flatnonzero(out['loop_mask'][g])
    out['loop_scale'][g, rows] = r['scale'][n - 1:]
    out['loop_chi2'][g, rows] = r['chi2'][n - 1:]
  return out


def pose_graph_summary(pgo, odometry, poses, gt_top_overlap, gt_overlap=0.3):
  """The ``pose_graph`` section of the summary: the odometry steps' errors and end states, and per graph the loops
  (correct ones), the kept loops (s >= 1/2) split into correct and incorrect, the trajectory error before (the
  composed odometry) and after, its status and iterations."""
  from ._cabi import ICP_STATUS, PGO_STATUS
  from .pose_graph import KEEP_SCALE, trajectory_error
  steps = odometry['status'] >= 0
  e = odometry['error'][steps]
  st = odometry['status'][steps]
  n = poses.shape[0]
  before = np.empty((n, 4, 4))
  before[0] = np.eye(4)
  for k in range(1, n):
    before[k] = before[k - 1] @ odometry['pose'][k]
  correct = np.asarray(gt_top_overlap, np.float64)[:, 0] > gt_overlap
  names = {v: k for k, v in PGO_STATUS.items()}
  out = {'odometry': {'steps': int(steps.sum()),
                      'median_error_translation_m': float(np.median(e[:, 0])) if e.size else float('nan'),
                      'max_error_translation_m': float(np.max(e[:, 0])) if e.size else float('nan'),
                      'median_error_rotation_deg': float(np.median(e[:, 1])) if e.size else float('nan'),
                      'max_error_rotation_deg': float(np.max(e[:, 1])) if e.size else float('nan'),
                      'degenerate': int((st == ICP_STATUS['degenerate']).sum()),
                      'too_few_inliers': int((st == ICP_STATUS['too_few_inliers']).sum())},
         'error_before': trajectory_error(before, poses), 'keep_scale': KEEP_SCALE, 'graphs': {}}
  for g, name in enumerate(PGO_GRAPHS):
    m = pgo['loop_mask'][g]
    kept = m & (pgo['loop_scale'][g] >= KEEP_SCALE)
    out['graphs'][name] = {'loops': int(m.sum()), 'correct_loops': int((m & correct).sum()),
                           'kept_correct': int((kept & correct).sum()), 'kept_incorrect': int((kept & ~correct).sum()),
                           'error_after': trajectory_error(pgo['poses'][g], poses),
                           'status': names[int(pgo['status'][g])], 'iterations': int(pgo['iterations'][g])}
  return out


# ---- the driver ---------------------------------------------------------------------------------------------
def _dist():
  dist = torch.distributed
  if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
    return dist, dist.get_rank(), dist.get_world_size()
  return None, 0, 1


def encode_share(infer, clouds, rank=0, world=1):
  """This rank's share of the scans' volumes on the device, and every rank's share [(lo, hi)].  The scans are
  encoded in batches of the Infer's batch_size at fixed positions of the sequence, and each rank takes a
  contiguous run of whole batches: every volume comes out of the same batch, so the same bits, at any world size."""
  from .search import shard_range
  n = len(clouds)
  bs = max(1, int(infer.batch_size))
  n_batches = (n + bs - 1) // bs
  shares = [tuple(min(n, bs * b) for b in shard_range(n_batches, r, world)) for r in range(world)]
  lo, hi = shares[rank]
  eng = infer._engine
  out = torch.empty((hi - lo, eng.Wf, 128), dtype=torch.float32, device=eng.device)
  for s0 in range(lo, hi, bs):
    s1 = min(hi, s0 + bs)
    batch = [np.ascontiguousarray(clouds[i]() if callable(clouds[i]) else clouds[i], np.float32) for i in range(s0, s1)]
    out[s0 - lo:s1 - lo] = infer.encode_clouds(batch)
  return out, shares


def gather_bank(local, shares):
  """The whole bank on every rank: one all_gather of the padded shares (as ShardedSearch.gather_bank), on the
  device with NCCL and through host memory with other backends."""
  dist = torch.distributed
  on_device = dist.get_backend() == 'nccl'
  pad = torch.zeros((max(hi - lo for lo, hi in shares),) + tuple(local.shape[1:]), dtype=local.dtype,
                    device=local.device if on_device else 'cpu')
  pad[:local.shape[0]] = local
  parts = [torch.empty_like(pad) for _ in shares]
  dist.all_gather(parts, pad)
  return torch.cat([parts[r][:hi - lo] for r, (lo, hi) in enumerate(shares)]).to(local.device)


def save_npz(path, arrays):
  """np.savez with a fixed time stamp on every member: the same arrays give the same bytes."""
  import zipfile
  with zipfile.ZipFile(path, 'w', zipfile.ZIP_STORED, allowZip64=True) as z:
    for key in sorted(arrays):
      info = zipfile.ZipInfo(key + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
      with z.open(info, 'w', force_zip64=True) as f:
        np.lib.format.write_array(f, np.asanyarray(arrays[key]), allow_pickle=False)


def evaluate_clouds(infer, clouds, poses, top_k=5, exclude_frames=100, exclude_distance=50, gt_overlap=0.3,
                    out_dir=None, register=False, min_inlier_fraction=0.3, close_loops=False):
  """Evaluate loop closure over a sequence: ``clouds`` (N, 4) float32 arrays or zero-argument callables returning
  one, ``poses`` (n, 4, 4) LiDAR-frame poses, ``infer`` an overlapnet_b200.Infer.  In a process group every rank
  encodes a contiguous share of the scans, the bank is all-gathered, every rank scores and labels the rows of an
  equal share of the pairs, and rank 0 gathers them; the results do not depend on the world size.  Returns on
  rank 0 (summary dict, results dict of arrays), None elsewhere; rank 0 writes lcd_results.npz and
  lcd_summary.json to ``out_dir`` when given.  With ``register`` each rank also registers its rows' top records
  (register_records) and the results gain the registration_* arrays and a ``registration`` summary section
  (registration_summary, with ``min_inlier_fraction``); without it nothing differs from an evaluation without
  registration.  ``close_loops`` implies ``register``: each rank also registers the odometry steps (i - 1, i) of its
  rows (register_odometry), and rank 0 optimizes the five loop_graphs in one pose-graph call (close_loops_graphs);
  the results gain the odometry_* and pgo_* arrays and a ``pose_graph`` summary section (pose_graph_summary)."""
  if not 1 <= int(top_k) <= TOPK_MAX:
    raise ValueError('top_k must be in [1, %d], got %r' % (TOPK_MAX, top_k))
  top_k = int(top_k)
  poses = np.asarray(poses, np.float64)
  n = len(clouds)
  if poses.shape != (n, 4, 4):
    raise ValueError('poses has shape %s, expected (%d, 4, 4)' % (poses.shape, n))
  register = register or close_loops
  dist, rank, world = _dist()
  eng = infer._engine
  c = past_prefix(poses[:, :2, 3], exclude_frames, exclude_distance)
  local, shares = encode_share(infer, clouds, rank, world)
  full = gather_bank(local, shares) if world > 1 else local
  del local
  # the tensor-core heads' numeric centres from volume 0 on every handle, before the operand copies are built
  eng.calibrate(full[0])
  infer._set_bank(full)
  bank = infer._bank
  r_lo, r_hi = split_rows(c, world)[rank]
  top_ov, top_idx, top_yaw = search(eng, bank, c, top_k, r_lo, r_hi)
  truth = ground_truth(clouds, poses, np.arange(r_lo, r_hi), c[r_lo:r_hi], top_idx, eng.Wf, local=world > 1)
  part = (top_ov, top_idx, top_yaw, truth['best'], truth['top_overlap'], truth['top_yaw_bin'])
  if register:
    reg = register_records(eng, clouds, poses, np.arange(r_lo, r_hi), top_idx, top_yaw)
    reg_keys = sorted(reg)
    part += tuple(reg[key] for key in reg_keys)
  if close_loops:
    odo = register_odometry(eng, clouds, poses, np.arange(r_lo, r_hi))
    odo_keys = sorted(odo)
    part += tuple(odo[key] for key in odo_keys)
  if world > 1:
    parts = [None] * world if rank == 0 else None
    dist.gather_object(part, parts, dst=0)
    if rank != 0:
      return None
    part = tuple(np.concatenate([p[f] for p in parts]) for f in range(len(part)))
  top_ov, top_idx, top_yaw, gt_best, gt_top, gt_bin = part[:6]
  summary, curve = metrics(top_ov, top_idx, gt_top, gt_best, gt_overlap)
  t = summary['f1_max_threshold']
  tp_rows = true_positives_at(top_ov, top_idx, gt_top, t, gt_overlap) if np.isfinite(t) else np.zeros(0, np.int64)
  d_yaw = yaw_errors(eng, bank, tp_rows, top_idx[tp_rows, 0], gt_bin[tp_rows, 0], eng.Wf)
  summary.update(
      scans=n, pairs=int(c.sum()), exclude_frames=exclude_frames, exclude_distance=exclude_distance,
      gt_overlap=gt_overlap, world_size=world, true_positives_at_f1_max=int(tp_rows.size),
      yaw_error_mean=float(d_yaw.mean()) if d_yaw.size else float('nan'),
      yaw_error_max=float(d_yaw.max()) if d_yaw.size else float('nan'),
      yaw_error_rms=float(np.sqrt(np.mean(d_yaw * d_yaw))) if d_yaw.size else float('nan'))
  results = {'c': c, 'top_overlap': top_ov, 'top_index': top_idx, 'top_yaw': top_yaw, 'gt_top_overlap': gt_top,
             'gt_top_yaw_bin': gt_bin, 'gt_best': gt_best, 'positive': gt_best > gt_overlap,
             'true_positive_rows': tp_rows, 'yaw_error': d_yaw}
  results.update({'curve_' + key: v for key, v in curve.items()})
  if register:
    reg = dict(zip(reg_keys, part[6:6 + len(reg_keys)]))
    results.update({'registration_' + key: v for key, v in reg.items()})
    summary['registration'] = registration_summary(top_ov, top_idx, gt_top, gt_best, tp_rows, reg['error'],
                                                   reg['inlier_fraction'], gt_overlap, min_inlier_fraction)
  if close_loops:
    odo = dict(zip(odo_keys, part[6 + len(reg_keys):]))
    results.update({'odometry_' + key: v for key, v in odo.items()})
    masks = loop_sets(top_ov, top_idx, gt_top, reg['inlier_fraction'], t, gt_overlap, min_inlier_fraction)
    pgo = close_loops_graphs(eng, odo['pose'], top_idx, reg['pose'][:, 0], masks)
    results.update({'pgo_' + key: v for key, v in pgo.items()})
    summary['pose_graph'] = pose_graph_summary(pgo, odo, poses, gt_top, gt_overlap)
  if out_dir is not None:
    os.makedirs(out_dir, exist_ok=True)
    save_npz(os.path.join(out_dir, 'lcd_results.npz'), results)
    with open(os.path.join(out_dir, 'lcd_summary.json'), 'w') as f:
      json.dump(summary, f, indent=1, sort_keys=True)
  return summary, results


# ---- the command line ---------------------------------------------------------------------------------------
def parse_args(argv):
  p = argparse.ArgumentParser(prog='python -m overlapnet_b200.lcd_eval',
                              description='Loop-closure precision-recall of a model over a whole sequence.')
  p.add_argument('config', nargs='?', default='config/demo.yml', help='YAML file with a Demo3 section')
  p.add_argument('--top-k', type=int, default=5, help='records kept per query, 1..%d (default 5)' % TOPK_MAX)
  p.add_argument('--exclude-frames', type=int, default=100, help='the most recent frames skipped (default 100)')
  p.add_argument('--exclude-distance', type=float, default=50.0, help='metres of travel skipped (default 50)')
  p.add_argument('--gt-overlap', type=float, default=0.3, help='ground-truth overlap of a true loop (default 0.3)')
  p.add_argument('--precision', default='f16_tc', choices=('f16_tc', 'fp32'))
  p.add_argument('--register', action='store_true',
                 help='register each top record by ICP on the GPU, from the yaw seed and from the identity')
  p.add_argument('--close-loops', action='store_true',
                 help='also register the odometry by ICP and optimize pose graphs over five loop sets (implies '
                      '--register)')
  p.add_argument('--min-inlier-fraction', type=float, default=0.3,
                 help='with --register: the inlier fraction a verified loop reaches (default 0.3)')
  args = p.parse_args(argv)
  if not 1 <= args.top_k <= TOPK_MAX:
    p.error('--top-k must be in [1, %d], got %d' % (TOPK_MAX, args.top_k))
  if not 0.0 <= args.min_inlier_fraction <= 1.0:
    p.error('--min-inlier-fraction must be in [0, 1], got %g' % args.min_inlier_fraction)
  args.register = args.register or args.close_loops
  return args


def network_config(config):
  """The network config of a demo.yml dict's Demo3 section, refused when it uses class probabilities."""
  from .config import load_config
  net = load_config(config['Demo3']['network_config'])
  if net.get('use_class_probabilities', False):
    raise Exception('lcd_eval: the network config uses class probabilities, which would need a .label file per '
                    'scan; only geometric configs are evaluated from raw scans')
  return net


def main(argv=None):
  from . import gt
  from .config import load_config
  from .gt_files import kitti_poses_in_lidar
  from .infer import Infer
  from .preprocess import _read_scan, load_files
  logging.basicConfig(level=logging.INFO, format='%(message)s')
  args = parse_args(sys.argv[1:] if argv is None else argv)
  config = load_config(args.config)
  net = network_config(config)
  d = config['Demo3']
  world = int(os.environ.get('WORLD_SIZE', '1'))
  if world > 1:
    local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local_rank)
    torch.distributed.init_process_group('nccl', device_id=torch.device('cuda', local_rank))
  scan_paths = load_files(d['scan_folder'])
  poses = kitti_poses_in_lidar(gt.load_poses(d['poses_file']), gt.load_calib(d['calib_file']))
  clouds = [(lambda p=p: _read_scan(p)) for p in scan_paths]
  for key, default in (('use_depth', True), ('use_normals', True), ('use_class_probabilities', False),
                       ('use_class_probabilities_pca', False), ('use_intensity', False)):
    net.setdefault(key, default)
  net.setdefault('infer_seqs', d.get('infer_seqs', ''))
  net.setdefault('data_root_folder', '')
  infer = Infer(net, precision=args.precision)
  out_dir = os.path.join(net.get('experiments_path', '/tmp'), net.get('testname', 'experiment_test'))
  res = evaluate_clouds(infer, clouds, poses, args.top_k, args.exclude_frames, args.exclude_distance,
                        args.gt_overlap, out_dir, args.register, args.min_inlier_fraction, args.close_loops)
  if res is not None:
    s = res[0]
    logger.info('Loop closure over %d scans, %d queries, %d positive (ground-truth overlap > %g), %d pairs scored',
                s['scans'], s['queries'], s['positives'], s['gt_overlap'], s['pairs'])
    logger.info('  average precision:              %f', s['average_precision'])
    logger.info('  F1max:                          %f at overlap >= %f', s['f1_max'], s['f1_max_threshold'])
    logger.info('  precision / recall at > %g:    %f / %f', s['operating_point'], s['precision_at_operating_point'],
                s['recall_at_operating_point'])
    logger.info('  recall@1 / recall@%d:            %f / %f', s['k'], s['recall_at_1'], s['recall_at_k'])
    logger.info('  yaw error of the %d true positives at F1max: mean %f, max %f, RMS %f bins',
                s['true_positives_at_f1_max'], s['yaw_error_mean'], s['yaw_error_max'], s['yaw_error_rms'])
    if 'registration' in s:
      r = s['registration']
      logger.info('  registration of the %d true positives: success %f from the yaw seed, %f from the identity '
                  '(< %g m, < %g deg); yaw seed median %f m / %f deg', r['true_positives'], r['success_rate_yaw'],
                  r['success_rate_identity'], r['success_translation_m'], r['success_rotation_deg'],
                  r['median_error_translation_m_yaw'], r['median_error_rotation_deg_yaw'])
      logger.info('  precision / recall at > %g with inlier fraction >= %g: %f / %f', s['operating_point'],
                  r['min_inlier_fraction'], r['precision_at_operating_point_verified'],
                  r['recall_at_operating_point_verified'])
    if 'pose_graph' in s:
      pgs = s['pose_graph']
      o = pgs['odometry']
      logger.info('  odometry: %d ICP steps, median error %f m / %f deg, max %f m / %f deg, %d degenerate, %d with '
                  'too few inliers', o['steps'], o['median_error_translation_m'], o['median_error_rotation_deg'],
                  o['max_error_translation_m'], o['max_error_rotation_deg'], o['degenerate'], o['too_few_inliers'])
      b = pgs['error_before']
      logger.info('  trajectory error of the odometry: RMSE %f m / %f deg, max %f m / %f deg',
                  b['translation_rmse_m'], b['rotation_rmse_deg'], b['translation_max_m'], b['rotation_max_deg'])
      for name, gs in pgs['graphs'].items():
        a = gs['error_after']
        logger.info('  pose graph %-11s %4d loops (%d correct), kept %d correct / %d incorrect: RMSE %f m / %f deg, '
                    'max %f m / %f deg, %s after %d iterations', name, gs['loops'], gs['correct_loops'],
                    gs['kept_correct'], gs['kept_incorrect'], a['translation_rmse_m'], a['rotation_rmse_deg'],
                    a['translation_max_m'], a['rotation_max_deg'], gs['status'], gs['iterations'])
    logger.info('  written to %s', out_dir)
  if world > 1:
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()
  return res


if __name__ == '__main__':
  main()
