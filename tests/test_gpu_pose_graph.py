"""Robust pose-graph optimization on the GPU (ovn_pgo_optimize_host) against the float64 model (oracle/pose_graph.py):
the cost, chi2, scales and gradient at the input, the LM trace against an oracle replay, the known answer and the
robust kernel, sizes up to a KITTI 00 chain, bit-identical graphs in any batch and handle, and the refusals."""
import numpy as np
import pytest

from oracle import pose_graph as P
from overlapnet_b200 import pose_graph as pg, synth
from overlapnet_b200._cabi import PGO_STATUS
from overlapnet_b200.engine import Engine
from overlapnet_b200.pose_graph import trajectory_error

pytestmark = pytest.mark.gpu

CTA_WARPS = 8           # k_pgo_graphs' warps, one chain segment each (DESIGN section 4)


@pytest.fixture(scope='module')
def eng():
  e = Engine(precision='fp32', max_batch_scans=1, max_batch_pairs=1)
  yield e
  e.close()


def rot_err(A, B):
  return np.abs(P.log_so3(np.swapaxes(A[..., :3, :3], -1, -2) @ B[..., :3, :3])).max()


def test_zero_iterations_evaluate_at_the_input(eng):
  g, _ = synth.pose_graph_scene(200, 15, seed=2, n_false=3, init_noise=(0.5, 0.05))
  r = eng.pose_graph([g], {'max_iterations': 0}, want_gradient=True)[0]
  F, chi2, s, grad, _ = P.linearize(g, g['poses'], P.DEFAULTS['phi'])
  assert r['iterations'] == 0 and r['initial_cost'] == r['final_cost']
  np.testing.assert_array_equal(r['poses'], g['poses'])
  assert abs(r['final_cost'] - F) <= 1e-12 * F
  np.testing.assert_allclose(r['chi2'], chi2, rtol=1e-12, atol=0)
  np.testing.assert_allclose(r['scale'], s, rtol=1e-12, atol=0)
  assert np.abs(r['gradient'] - grad).max() <= 1e-10 * np.abs(grad).max()
  assert abs(r['max_gradient'] - np.abs(grad[1:]).max()) <= 1e-10 * np.abs(grad).max()


def test_the_trace_follows_an_oracle_replay(eng):
  g, _ = synth.pose_graph_scene(300, 20, seed=5, n_false=4, init_noise=(0.1, 0.02))
  r = eng.pose_graph([g], want_trace=True)[0]
  t = r['trace']
  assert r['status'] == PGO_STATUS['converged'] and len(t['cost']) == r['iterations']
  ref = P.optimize(g)
  assert [bool(a) for a in t['accepted']] == [bool(a) for _, _, a in ref['trace']]
  np.testing.assert_allclose(t['lambda'], [lam for _, lam, _ in ref['trace']], rtol=0, atol=0)
  costs, _ = P.replay(g, t['lambda'], t['accepted'])
  np.testing.assert_allclose(t['cost'], costs, rtol=1e-9, atol=1e-20)
  assert np.abs(r['poses'][:, :3, 3] - ref['poses'][:, :3, 3]).max() < 1e-6
  assert rot_err(r['poses'], ref['poses']) < 1e-8
  print('trace: %d trials, %d accepted, %d CG iterations' % (r['iterations'], r['accepted'], r['cg_iterations']))


def test_known_answer_and_false_loops(eng):
  clean, gt = synth.pose_graph_scene(300, 20, seed=1)
  dirty, _ = synth.pose_graph_scene(300, 20, seed=1, n_false=5)
  rc, rd, rl = eng.pose_graph([clean, dirty, dirty], None)[:2] + eng.pose_graph([dirty], {'phi': float('inf')})
  assert rc['final_cost'] < 1e-16
  e = trajectory_error(rc['poses'], gt)
  assert e['translation_max_m'] < 1e-8 and np.deg2rad(e['rotation_max_deg']) < 1e-9
  s = rd['scale'][299:]
  assert np.all(s[:20] > 0.9) and np.all(s[20:] < 0.1), s
  ed = trajectory_error(rd['poses'], gt)
  assert ed['translation_max_m'] - e['translation_max_m'] < 1e-3
  assert trajectory_error(rl['poses'], gt)['translation_max_m'] > 10 * max(ed['translation_max_m'], 1e-3)


SIZES = [(2, 0), (CTA_WARPS - 2, 1), (CTA_WARPS + 3, 2), (3 * CTA_WARPS + 6, 3), (1101, 40), (4541, 200)]


@pytest.mark.parametrize('n,loops', SIZES)
def test_sizes_converge_to_the_oracle(eng, n, loops):
  g, gt = synth.pose_graph_scene(n, loops, seed=n, min_gap=min(10, n - 1))
  r = eng.pose_graph([g], want_gradient=True)[0]
  ref = P.optimize(g)
  assert r['status'] == PGO_STATUS['converged'], r
  assert ref['status'] == 'converged'
  assert np.abs(r['poses'][:, :3, 3] - ref['poses'][:, :3, 3]).max() < 1e-6
  assert rot_err(r['poses'], ref['poses']) < 1e-8
  print('n %d, %d loops: %d trials, %d CG iterations' % (n, loops, r['iterations'], r['cg_iterations']))


def bits(x):
  return np.ascontiguousarray(x).view(np.uint8)


def test_a_graph_has_the_same_bits_in_any_batch_and_handle(eng):
  g, _ = synth.pose_graph_scene(500, 30, seed=7, n_false=2)
  others = [synth.pose_graph_scene(50 + 37 * k, 3 + k, seed=20 + k)[0] for k in range(6)]
  alone = eng.pose_graph([g], want_gradient=True, want_trace=True)[0]
  e2 = Engine(precision='fp32', max_batch_scans=1, max_batch_pairs=1)
  try:
    runs = [e2.pose_graph([g], want_gradient=True, want_trace=True)[0]]
  finally:
    e2.close()
  for pos in (0, 3, 6):
    batch = others[:pos] + [g] + others[pos:]
    runs.append(eng.pose_graph(batch, want_gradient=True, want_trace=True)[pos])
  for r in runs:
    for key in ('poses', 'chi2', 'scale', 'gradient'):
      assert np.array_equal(bits(r[key]), bits(alone[key])), key
    for key in ('cost', 'lambda', 'accepted', 'cg_iterations'):
      assert np.array_equal(bits(r['trace'][key]), bits(alone['trace'][key])), key
    for key in ('status', 'iterations', 'accepted', 'cg_iterations', 'final_cost', 'lambda', 'max_gradient'):
      assert r[key] == alone[key], key


def _packed(g):
  return dict(node_off=np.array([0, g['poses'].shape[0]]), edge_off=np.array([0, g['edges'].shape[0]]),
              poses=g['poses'], edges=g['edges'], measurements=g['measurements'], weights=g['weights'])


def test_refusals_return_the_error_and_write_nothing(eng):
  from test_pose_graph import REFUSALS
  g, _ = synth.pose_graph_scene(12, 2, seed=0)
  cases = {k: _packed(f(g)) for k, f in REFUSALS.items()}
  base = _packed(g)
  cases['bad offsets'] = dict(base, node_off=np.array([1, 12]))
  for key, value in (('phi', 0.0), ('phi', float('nan')), ('lambda0', 1e13), ('lambda_min', 0.0), ('cg_tol', -1.0),
                     ('max_iterations', 1001), ('max_iterations', -1), ('max_cg_iterations', 0),
                     ('max_cg_iterations', 10001), ('step_tol', float('inf'))):
    cases['%s=%r' % (key, value)] = dict(base, params=pg.default_params({key: value}))
  for name, c in cases.items():
    c = dict(c)
    prm = c.pop('params', pg.default_params())
    n, e = int(np.asarray(c['poses']).reshape(-1, 16).shape[0]), int(np.asarray(c['edges']).reshape(-1, 2).shape[0])
    G = len(c['node_off']) - 1
    sentinel = {'poses': np.full((n, 4, 4), 7.0), 'result': np.zeros(G, [('initial_cost', 'f8'), ('final_cost', 'f8'),
                ('lambda', 'f8'), ('max_gradient', 'f8'), ('status', 'i4'), ('iterations', 'i4'), ('accepted', 'i4'),
                ('cg_iterations', 'i4')]), 'chi2': np.full(e, 7.0), 'scale': np.full(e, 7.0),
                'gradient': np.full((n, 6), 7.0), 'trace': None}
    sentinel['result']['status'] = 77
    out = eng.pose_graph_raw(c['node_off'], c['edge_off'], c['poses'], c['edges'], c['measurements'], c['weights'],
                             prm, outputs=sentinel)
    assert out['rc'] == -1, name
    assert np.all(out['poses'] == 7.0) and np.all(out['chi2'] == 7.0) and np.all(out['scale'] == 7.0), name
    assert np.all(out['gradient'] == 7.0) and np.all(out['result']['status'] == 77), name
  # the handle stays usable
  assert eng.pose_graph([g])[0]['status'] == PGO_STATUS['converged']


# ---- lcd_eval --close-loops on a street-scene drive --------------------------------------------------------------
DRIVE_STEP = 1.25           # metres between scans
CLOSE_EVAL = dict(top_k=3, exclude_frames=40, exclude_distance=40.0)


def street_drive_poses():
  """One lap around the city block [0, 40]^2 of the street scene along its roads, one scan across to the square
  inset 1.5 m, then 70 m of a second lap along it, at most DRIVE_STEP metres per scan (185 scans)."""
  import math
  from icp_cases import rz
  poses = []
  for off, length in ((0.0, 160.0), (1.5, 70.0)):
    side_len = 40 - 2 * off
    if off:
      poses.append(rz(math.radians(315.0), (0.75, 0.75, 1.73)))
    for k in range(int(length / DRIVE_STEP)):
      s = k * DRIVE_STEP
      side, u = int(s // side_len), s % side_len
      x, y, yaw = [(off + u, off, 0.0), (40 - off, off + u, 90.0), (40 - off - u, 40 - off, 180.0),
                   (off, 40 - off - u, 270.0)][side]
      poses.append(rz(math.radians(yaw), (x, y, 1.73)))
  return np.array(poses)


def street_drive_clouds(poses):
  return [synth.street_scene_cloud(T, seed=11, noise=0.02) for T in poses]


@pytest.fixture(scope='module')
def drive(tmp_path_factory):
  import copy
  import os
  from oracle import network as N
  from overlapnet_b200 import weights as W
  from test_gpu_icp import MODEL
  root = str(tmp_path_factory.mktemp('lcd_close_loops'))
  poses = street_drive_poses()
  w = N.glorot_weights(4, MODEL, seed=5)
  wpath = os.path.join(root, 'weights.npz')
  W.save_npz(wpath, w)
  cfg = {'pretrained_weightsfilename': wpath, 'use_depth': True, 'use_normals': True,
         'use_class_probabilities': False, 'use_class_probabilities_pca': False, 'use_intensity': False,
         'data_root_folder': root, 'infer_seqs': '07', 'batch_size': 4, 'model': copy.deepcopy(MODEL)}
  return street_drive_clouds(poses), poses, cfg


def _close_loops_rank(rank, world, port, cfg, out_dir):
  import copy
  import os
  import torch
  import torch.distributed as dist
  from overlapnet_b200 import lcd_eval
  from overlapnet_b200.infer import Infer
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  torch.cuda.set_device(0)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  try:
    poses = street_drive_poses()
    lcd_eval.evaluate_clouds(Infer(copy.deepcopy(cfg)), street_drive_clouds(poses), poses, out_dir=out_dir,
                             close_loops=True, **CLOSE_EVAL)
  except Exception:
    import traceback
    with open(os.path.join(os.path.dirname(out_dir), 'rank%d.err' % rank), 'w') as f:
      f.write(traceback.format_exc())
    raise
  finally:
    dist.destroy_process_group()


def test_close_loops_on_a_street_drive(drive, tmp_path):
  import copy
  import math
  import os
  import torch.multiprocessing as mp
  from overlapnet_b200 import lcd_eval
  from overlapnet_b200.infer import Infer
  from test_gpu_icp import _free_port
  clouds, poses, cfg = drive
  assert len(poses) <= 200 and np.all(np.linalg.norm(np.diff(poses[:, :3, 3], axis=0), axis=1) <= DRIVE_STEP + 1e-9)
  runs = {}
  for name, kw in (('plain', {}), ('register', {'register': True}), ('close', {'close_loops': True})):
    runs[name] = lcd_eval.evaluate_clouds(Infer(copy.deepcopy(cfg)), clouds, poses, out_dir=str(tmp_path / name),
                                          **CLOSE_EVAL, **kw)
  (s0, plain), (s1, reg), (s2, res) = runs['plain'], runs['register'], runs['close']
  # without the flag nothing changes; with it, everything --register writes is unchanged
  for key, v in reg.items():
    assert np.array_equal(bits(v), bits(res[key])), key
  for key, v in plain.items():
    assert np.array_equal(bits(v), bits(res[key])), key
  assert set(res) - set(reg) == {'odometry_error', 'odometry_pose', 'odometry_status', 'pgo_poses', 'pgo_loop_mask',
                                 'pgo_loop_scale', 'pgo_loop_chi2', 'pgo_status', 'pgo_iterations', 'pgo_cost'}
  assert set(s2) == set(s1) | {'pose_graph'}
  for k in s1:
    assert s1[k] == s2[k] or (isinstance(s1[k], float) and math.isnan(s1[k]) and math.isnan(s2[k])), k
  # pgo_poses are what pose_graph.optimize gives on the graphs rebuilt from the results' arrays
  masks = {name: res['pgo_loop_mask'][g] for g, name in enumerate(lcd_eval.PGO_GRAPHS)}
  graphs = lcd_eval.loop_graphs(res['odometry_pose'], res['top_index'], res['registration_pose'][:, 0], masks)
  want = pg.optimize(Infer(copy.deepcopy(cfg))._engine, graphs)
  for g, r in enumerate(want):
    assert np.array_equal(bits(res['pgo_poses'][g]), bits(r['poses'])), g
    assert res['pgo_status'][g] == r['status'] and res['pgo_iterations'][g] == r['iterations']
  assert masks['true_loops'].any() and not masks['odometry'].any()
  # ground truth only selects the true loops: the odometry edges are the ICP steps
  assert np.array_equal(graphs[0]['measurements'], res['odometry_pose'][1:])
  print('pose_graph summary:', s2['pose_graph'])
  # two gloo ranks write the one-rank results byte for byte
  two = str(tmp_path / 'two')
  try:
    mp.spawn(_close_loops_rank, args=(2, _free_port(), cfg, two), nprocs=2, join=True)
  finally:
    for r in range(2):
      err = tmp_path / ('rank%d.err' % r)
      if err.exists():
        print(err.read_text())
  with open(os.path.join(str(tmp_path / 'close'), 'lcd_results.npz'), 'rb') as f1, \
      open(os.path.join(two, 'lcd_results.npz'), 'rb') as f2:
    assert f1.read() == f2.read()
