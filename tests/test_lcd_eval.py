"""Host logic of the loop-closure evaluation (overlapnet_b200.lcd_eval): the candidate prefix against demo 3's
gating, the precision-recall metrics against a brute-force loop over the thresholds, the row split and the CLI's
refusals."""
import os

import numpy as np
import pytest

from overlapnet_b200 import lcd, lcd_eval


def _golden_traj():
  from conftest import GOLDEN
  return np.load(os.path.join(GOLDEN, 'lcd_demo3.npz'))['traj']


@pytest.mark.parametrize('frames,dist', [(100, 50), (10, 5.0), (3, 0.5), (0, 0.0)])
def test_past_prefix_restates_the_time_and_distance_rules(frames, dist):
  traj = _golden_traj()
  c = lcd_eval.past_prefix(traj, frames, dist)
  L = lcd_eval.travelled_distance(traj)
  huge = (np.zeros(2), 1e12, 1e12, 0.0)                        # an ellipse that contains every point
  for i in range(len(traj)):
    want = lcd.gate_candidates(i, traj, list(L), huge, frames, dist)
    assert np.array_equal(want, np.arange(c[i])), (i, c[i], want)
  assert np.all(np.diff(L) >= 0)
  if frames == 100:
    assert c.max() > 0 and c[:101].max() == 0


def test_travelled_distance_is_the_detectors():
  traj = _golden_traj()[:50]

  class Null:
    def infer_multiple(self, idx, refs):
      return None
  det = lcd.LoopClosureDetector(Null())
  for i in range(len(traj)):
    det.step(i, traj[i], np.eye(6))
  assert np.array_equal(lcd_eval.travelled_distance(traj), np.asarray(det.traj_length, float))


def brute_metrics(top_ov, top_idx, gt_top, gt_best, gt_overlap=0.3):
  """The definitions, one threshold at a time."""
  q = top_idx[:, 0] >= 0
  s = top_ov[q, 0].astype(np.float64)
  correct = gt_top[q, 0] > gt_overlap
  correct_k = ((top_idx[q] >= 0) & (gt_top[q] > gt_overlap)).any(1)
  pos = gt_best[q] > gt_overlap
  npos = pos.sum()
  P, R = [], []
  for t in sorted(set(s.tolist()), reverse=True):
    d = s >= t
    tp, fp = int((d & correct).sum()), int((d & ~correct).sum())
    P.append(tp / (tp + fp) if tp + fp else 1.0)
    R.append(tp / npos if npos else float('nan'))
  out = {'P': np.array(P), 'R': np.array(R)}
  if npos:
    ap, prev = 0.0, 0.0
    for p, r in zip(P, R):
      ap += (r - prev) * p
      prev = r
    f1 = [2 * p * r / (p + r) if p + r > 0 else 0.0 for p, r in zip(P, R)]
    out.update(ap=ap, f1=max(f1), thr=sorted(set(s.tolist()), reverse=True)[int(np.argmax(f1))],
               r1=(pos & correct).sum() / npos, rk=(pos & correct_k).sum() / npos)
  op = s > 0.3
  out['op_p'] = (op & correct).sum() / op.sum() if op.sum() else 1.0
  out['op_r'] = (op & correct).sum() / npos if npos else float('nan')
  return out


def random_records(rng, rows, k, c_max, tie_levels=None, all_positive=None):
  c = rng.integers(0, c_max + 1, rows)
  top_ov = np.full((rows, k), -1.0, np.float32)
  top_idx = np.full((rows, k), -1, np.int32)
  gt_top = np.full((rows, k), -1.0)
  for r in range(rows):
    m = min(k, c[r])
    v = rng.random(m).astype(np.float32)
    if tie_levels:
      v = (np.floor(v * tie_levels) / tie_levels).astype(np.float32)
    top_ov[r, :m] = np.sort(v)[::-1]
    top_idx[r, :m] = rng.permutation(c[r])[:m]
    gt_top[r, :m] = rng.random(m)
  gt_best = np.where(c > 0, np.maximum(gt_top.max(1), rng.random(rows) * 0.6), -1.0)
  if all_positive is False:
    gt_top = np.minimum(gt_top, 0.2)
    gt_best = np.minimum(gt_best, 0.2)
  return top_ov, top_idx, gt_top, gt_best


@pytest.mark.parametrize('seed,k,c_max,ties,pos', [(0, 5, 40, None, None), (1, 32, 10, 4, None),
                                                    (2, 1, 3, 3, None), (3, 8, 5, None, False),
                                                    (4, 5, 100, 2, None)])
def test_metrics_equal_the_brute_force_loop(seed, k, c_max, ties, pos):
  rng = np.random.default_rng(seed)
  top_ov, top_idx, gt_top, gt_best = random_records(rng, 300, k, c_max, ties, pos)
  s, curve = lcd_eval.metrics(top_ov, top_idx, gt_top, gt_best)
  b = brute_metrics(top_ov, top_idx, gt_top, gt_best)
  assert np.allclose(curve['precision'], b['P'], rtol=0, atol=1e-12)
  assert np.allclose(curve['recall'], b['R'], rtol=0, atol=1e-12, equal_nan=True)
  assert np.allclose(s['precision_at_operating_point'], b['op_p']) and \
      np.allclose(s['recall_at_operating_point'], b['op_r'], equal_nan=True)
  if pos is False:
    assert s['positives'] == 0 and np.isnan(s['average_precision']) and np.isnan(s['f1_max'])
  else:
    assert s['positives'] > 0
    assert abs(s['average_precision'] - b['ap']) < 1e-12 and abs(s['f1_max'] - b['f1']) < 1e-12
    assert s['f1_max_threshold'] == b['thr']
    assert abs(s['recall_at_1'] - b['r1']) < 1e-12 and abs(s['recall_at_k'] - b['rk']) < 1e-12
  assert s['queries'] == int((top_idx[:, 0] >= 0).sum())


def test_metrics_when_every_query_is_declared():
  top_ov = np.array([[0.9], [0.9], [0.9]], np.float32)
  top_idx = np.array([[0], [1], [2]], np.int32)
  gt_top = np.array([[0.5], [0.1], [0.4]])
  gt_best = np.array([0.5, 0.6, 0.4])
  s, curve = lcd_eval.metrics(top_ov, top_idx, gt_top, gt_best)
  assert curve['threshold'].tolist() == [np.float32(0.9)]
  assert curve['tp'].tolist() == [2] and curve['fp'].tolist() == [1]
  assert s['average_precision'] == pytest.approx(2 / 3 * 2 / 3)
  assert s['precision_at_operating_point'] == pytest.approx(2 / 3) and s['recall_at_1'] == pytest.approx(2 / 3)


def test_metrics_refuse_a_poisoned_score():
  with pytest.raises(ValueError, match='NaN'):
    lcd_eval.metrics(np.array([[np.nan]], np.float32), np.array([[0]]), np.array([[0.5]]), np.array([0.5]))


@pytest.mark.parametrize('world', [1, 2, 3, 7])
def test_split_rows_balances_the_pairs(world):
  c = lcd_eval.past_prefix(_golden_traj(), 100, 50)
  parts = lcd_eval.split_rows(c, world)
  assert parts[0][0] == 0 and parts[-1][1] == len(c)
  assert all(a[1] == b[0] for a, b in zip(parts, parts[1:]))
  sums = [int(c[lo:hi].sum()) for lo, hi in parts]
  assert max(sums) - min(sums) <= 2 * int(c.max())


def test_cli_refuses_k_outside_1_to_32(capsys):
  for k in ('0', '33', '-1'):
    with pytest.raises(SystemExit):
      lcd_eval.parse_args(['demo.yml', '--top-k', k])
  assert lcd_eval.parse_args(['demo.yml', '--top-k', '32']).top_k == 32
  with pytest.raises(ValueError, match='top_k'):
    lcd_eval.evaluate_clouds(None, [], np.zeros((0, 4, 4)), top_k=33)


def test_cli_refuses_semantic_configs(tmp_path):
  net = tmp_path / 'network.yml'
  net.write_text('use_class_probabilities: True\nuse_class_probabilities_pca: False\n')
  demo = tmp_path / 'demo.yml'
  demo.write_text('Demo3:\n  network_config: "%s"\n  poses_file: p\n  calib_file: c\n  scan_folder: s\n' % net)
  with pytest.raises(Exception, match='class probabilities'):
    lcd_eval.main([str(demo)])
