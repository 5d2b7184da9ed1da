"""`lcd_eval --close-loops` without a GPU: parsing, the loop sets, the graphs built from the results' arrays, and the
``pose_graph`` summary on crafted arrays."""
import numpy as np

from oracle import pose_graph as P
from overlapnet_b200 import lcd_eval
from overlapnet_b200._cabi import ICP_STATUS, PGO_STATUS


def test_close_loops_implies_register():
  a = lcd_eval.parse_args(['--close-loops'])
  assert a.close_loops and a.register
  a = lcd_eval.parse_args([])
  assert not a.close_loops and not a.register
  a = lcd_eval.parse_args(['--register'])
  assert a.register and not a.close_loops


def crafted():
  # rows 0..5: rows 0, 1 have no record; the others' top records, scores, truth and inlier fractions
  top_index = np.array([[-1, -1], [-1, -1], [0, 1], [1, 0], [0, 2], [2, 1]])
  top_overlap = np.array([[-1, -1], [-1, -1], [0.9, 0.1], [0.35, 0.2], [0.25, 0.1], [0.5, 0.4]], np.float32)
  gt_top = np.array([[-1, -1], [-1, -1], [0.8, 0.0], [0.1, 0.0], [0.6, 0.0], [0.05, 0.0]])
  frac = np.array([[np.nan] * 2, [np.nan] * 2, [0.6, 0.1], [0.5, 0.1], [0.9, 0.1], [0.2, 0.1]])
  return top_index, top_overlap, gt_top, frac


def test_loop_sets():
  top_index, top_overlap, gt_top, frac = crafted()
  m = lcd_eval.loop_sets(top_overlap, top_index, gt_top, frac, f1_threshold=0.5, gt_overlap=0.3,
                         min_inlier_fraction=0.3)
  assert tuple(m) == lcd_eval.PGO_GRAPHS
  assert m['odometry'].tolist() == [False] * 6
  assert m['verified'].tolist() == [False, False, True, True, False, False]     # s > 0.3 and fraction >= 0.3
  assert m['f1_max'].tolist() == [False, False, True, False, False, True]       # s >= 0.5
  assert m['all_records'].tolist() == [False, False, True, True, True, True]
  assert m['true_loops'].tolist() == [False, False, True, False, True, False]   # ground truth > 0.3
  none = lcd_eval.loop_sets(top_overlap, top_index, gt_top, frac, f1_threshold=float('nan'))
  assert not none['f1_max'].any()


def test_loop_graphs_and_summary():
  rng = np.random.default_rng(0)
  top_index, top_overlap, gt_top, frac = crafted()
  n = 6
  gt = np.empty((n, 4, 4))
  gt[0] = np.eye(4)
  for k in range(1, n):
    gt[k] = gt[k - 1] @ P.update(np.eye(4), [0, 0, 0.1, 1.0, 0, 0])
  odo = np.full((n, 4, 4), np.nan)
  odo[1:] = np.linalg.solve(gt[:-1], gt[1:])
  loop_pose = np.full((n, 4, 4), np.nan)
  for r in range(2, n):
    loop_pose[r] = np.linalg.solve(gt[top_index[r, 0]], gt[r])
  masks = lcd_eval.loop_sets(top_overlap, top_index, gt_top, frac, 0.5)
  graphs = lcd_eval.loop_graphs(odo, top_index, loop_pose, masks)
  assert len(graphs) == 5
  for g, name in zip(graphs, lcd_eval.PGO_GRAPHS):
    rows = np.flatnonzero(masks[name])
    assert g['edges'][n - 1:].tolist() == [[top_index[r, 0], r] for r in rows]
    np.testing.assert_allclose(g['poses'], gt, atol=1e-12)          # composed exact odometry from the identity
  # the summary on crafted optimizer outputs: graph 4 (true loops) keeps both loops, graph 3 keeps one wrong one
  G = 5
  pgo = {'poses': np.broadcast_to(gt, (G, n, 4, 4)).copy(), 'loop_mask': np.stack([masks[k] for k in lcd_eval.PGO_GRAPHS]),
         'loop_scale': np.full((G, n), np.nan), 'loop_chi2': np.full((G, n), np.nan),
         'status': np.array([PGO_STATUS['converged']] * 4 + [PGO_STATUS['stalled']], np.int32),
         'iterations': np.arange(G, dtype=np.int32), 'cost': np.zeros((G, 2))}
  pgo['poses'][2, 3, :3, 3] += [0.0, 0.3, 0.4]
  pgo['loop_scale'][3, 2:] = [0.9, 0.6, 0.95, 0.1]
  pgo['loop_scale'][4, [2, 4]] = [0.99, 0.4]
  odometry = {'pose': odo, 'status': np.array([-1, 0, 0, ICP_STATUS['degenerate'], 1, ICP_STATUS['too_few_inliers']],
                                              np.int32),
              'error': np.array([[np.nan, np.nan], [0.1, 1.0], [0.2, 2.0], [0.3, 3.0], [0.4, 4.0], [0.5, 5.0]])}
  s = lcd_eval.pose_graph_summary(pgo, odometry, gt, gt_top, 0.3)
  o = s['odometry']
  assert (o['steps'], o['degenerate'], o['too_few_inliers']) == (5, 1, 1)
  assert o['median_error_translation_m'] == 0.3 and o['max_error_rotation_deg'] == 5.0
  assert s['error_before']['translation_max_m'] < 1e-9
  a = s['graphs']['all_records']
  assert (a['loops'], a['correct_loops'], a['kept_correct'], a['kept_incorrect']) == (4, 2, 2, 1)
  t = s['graphs']['true_loops']
  assert (t['loops'], t['correct_loops'], t['kept_correct'], t['kept_incorrect']) == (2, 2, 1, 0)
  assert t['status'] == 'stalled' and t['iterations'] == 4
  assert abs(s['graphs']['f1_max']['error_after']['translation_max_m'] - 0.5) < 1e-12
