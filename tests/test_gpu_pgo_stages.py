"""Every stage of the pose-graph optimizer (k_pgo_graphs) read back by Engine.pose_graph_workspace and checked against
the float64 stage model (oracle/pgo_stages.py, whose docstring derives each gate): the edges' chi2, s, M and q, the
node gather, the preconditioner's factor and its two substitutions, the matvec with the loop edges, the PCG
recurrences and stop, the trial poses, the trial cost and the LM decisions.  Trial 1 at CG iteration c is the run
with max_iterations = 1 and max_cg_iterations = c; trial k is a fresh run from trial k - 1's poses and lambda."""
import ctypes as C

import numpy as np
import pytest

from oracle import pgo_stages as S
from oracle import pose_graph as P
from overlapnet_b200 import pose_graph as pg, synth
from overlapnet_b200._cabi import OvnError, PGO_ARRAYS, lib
from overlapnet_b200.engine import Engine

pytestmark = pytest.mark.gpu

WORST = {}          # stage -> largest err / bound seen, printed at the end of the module


@pytest.fixture(scope='module')
def eng():
  e = Engine(precision='fp32', max_batch_scans=1, max_batch_pairs=1)
  yield e
  e.close()
  print('\nlargest err / bound per stage: ' + ', '.join('%s %.3g' % kv for kv in sorted(WORST.items())))


def note(stage, gate):
  WORST[stage] = max(WORST.get(stage, 0.0), gate['worst'])
  assert gate['worst'] <= 1, (stage, gate)


def rz(a):
  R = np.eye(4)
  R[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
  return R


def with_loops(n, loops, seed, **kw):
  """synth's drive of n nodes with the given loop edges (exact measurements), initial poses perturbed"""
  g, gt = synth.pose_graph_scene(n, 0, seed=seed, **kw)
  loops = np.array(loops, np.int64).reshape(-1, 2)
  Z = np.linalg.solve(gt[loops[:, 0]], gt[loops[:, 1]])
  h = pg.chain_graph(g['measurements'][:n - 1], (loops, Z))
  h['poses'] = g['poses']
  return h


def branch_graph():
  """a straight drive with identity rotations (so chain residuals are exactly 0, sn = 0) and loops whose residual
  angles sit around the Log branch (pi - PI_BRANCH), the J_l^-1 series (SERIES_BELOW), near pi and at pi"""
  n = 12
  T = np.stack([np.eye(4)] * n)
  T[:, 0, 3] = np.arange(n, dtype=np.float64)
  odo = np.linalg.solve(T[:-1], T[1:])
  angles = [np.pi - 0.005, np.pi - 0.0099, np.pi - 0.0101, 0.0099, 0.0101, 0.5, np.pi]
  loops = [(k, k + 3) for k in range(len(angles))]
  Z = np.stack([np.linalg.solve(T[a], T[b]) @ rz(-t) for (a, b), t in zip(loops, angles)])
  g = pg.chain_graph(odo, (np.array(loops), Z))
  g['poses'] = T
  return g, n - 1 + len(angles) - 1          # the loop at exactly pi is not gated


def km_graph():
  g = with_loops(57, [(3, 40), (10, 50), (0, 30)], seed=4)
  T0 = rz(0.7)
  T0[:3, 3] = [700.0, -650.0, 30.0]
  g['poses'] = T0 @ g['poses']
  return g


CASES = {
    'n2': lambda: (synth.pose_graph_scene(2, 0, seed=2)[0], {}),
    'n3_gauge_loop': lambda: (with_loops(3, [(0, 2)], seed=3), {}),
    'n9_adjacent_separators': lambda: (with_loops(9, [(3, 5), (8, 1)], seed=9), {}),
    'n10_gauge': lambda: (with_loops(10, [(0, 5), (2, 9)], seed=10), {}),
    'n17_parallel': lambda: (with_loops(17, [(5, 6), (7, 6)], seed=17), {}),
    'n18_duplicate_reversed': lambda: (with_loops(18, [(2, 13), (2, 13), (16, 4)], seed=18), {}),
    'n57_segment_separators_csr': lambda: (with_loops(
        57, [(8, 12), (7, 21)] + [(30, k) for k in range(57) if k not in (29, 30, 31)][:44], seed=57), {}),
    'n57_lam1e-12': lambda: (with_loops(57, [(3, 40), (20, 50)], seed=5), {'lambda0': 1e-12}),
    'n57_lam1': lambda: (with_loops(57, [(3, 40), (20, 50)], seed=5), {'lambda0': 1.0}),
    'n57_lam1e6': lambda: (with_loops(57, [(3, 40), (20, 50)], seed=5), {'lambda0': 1e6}),
    'n57_km': lambda: (km_graph(), {}),
    'n300_false_loops': lambda: (synth.pose_graph_scene(300, 20, seed=5, n_false=4,
                                                        init_noise=(0.1, 0.02))[0], {}),
    'n300_phi_inf': lambda: (synth.pose_graph_scene(300, 20, seed=5, n_false=4, init_noise=(0.1, 0.02))[0],
                             {'phi': float('inf')}),
    'n1101_chain': lambda: (synth.pose_graph_scene(1101, 0, seed=1101)[0], {}),
    'branches': lambda: (branch_graph()[0], {}),
}


def run(eng, g, prm, **over):
  p = dict(prm, **over)
  return eng.pose_graph([g], p, want_gradient=True, want_trace=True)[0]


def ws(eng, *names):
  return [eng.pose_graph_workspace(k) for k in names]


def n_loops(g):
  return len(g['edges']) - (len(g['poses']) - 1)


@pytest.mark.parametrize('name', list(CASES))
def test_trial_one_stage_by_stage(eng, name):
  g, prm = CASES[name]()
  n, ed = len(g['poses']), g['edges']
  phi = prm.get('phi', P.DEFAULTS['phi'])
  lam = prm.get('lambda0', P.DEFAULTS['lambda0'])
  skip = None
  if name == 'branches':
    skip = np.zeros(len(ed), bool)
    skip[branch_graph()[1]] = True
  # the input: edges and gather
  r0 = run(eng, g, prm, max_iterations=0)
  T, M, q, Hd, gn = ws(eng, 'T', 'M', 'q', 'Hd', 'gn')
  assert np.array_equal(T, g['poses'])
  note('edge', S.edge_gate(g, T, phi, r0['chi2'], r0['scale'], M, q, skip))
  note('gather', S.gather_gate(M, q, Hd, gn, ed, n))
  # trial 1 with every CG iteration it needs
  r1 = run(eng, g, prm, max_iterations=1)
  count = int(r1['trace']['cg_iterations'][0])
  assert r1['iterations'] == 1 and count == r1['cg_iterations']
  Ld, Ls, Lk, Tt, x = ws(eng, 'Ld', 'Ls', 'Lk', 'Tt', 'x')
  if count == 0:
    assert not np.any(gn[1:])
    return
  f = S.factor_gate(Ld, Ls, Lk, Hd, M, lam, n)
  assert f['structure']
  note('factor', f)
  note('update', S.update_gate(T, x, Tt))
  note('cost', S.cost_gate(g, Tt, phi, r1['trace']['cost'][0]))
  assert bool(r1['trace']['accepted'][0]) == bool(r1['trace']['cost'][0] < r0['final_cost'])
  # CG iteration c from the runs capped at c - 2, c - 1 and c
  runs = {}

  def cap(c):
    if c not in runs:
      if c == 0:
        z = np.zeros((n, 6))
        runs[0] = {'x': z, 'r': np.concatenate([z[:1], -gn[1:]])}
      else:
        run(eng, g, prm, max_iterations=1, max_cg_iterations=c)
        runs[c] = dict(zip(('x', 'r', 'z', 'p', 'Ap', 'y'), ws(eng, 'x', 'r', 'z', 'p', 'Ap', 'y')))
    return runs[c]
  for c in sorted({1, 2, 3, max(1, count // 2), count} & set(range(1, count + 1))):
    cur, prev = cap(c), cap(c - 1)
    note('apply', S.apply_gate(Ld, Ls, Lk, prev['r'], cur['y'], cur['z'], n))
    note('matvec', S.matvec_gate(Hd, M, ed, lam, cur['p'], cur['Ap'], n))
    if c == 1:
      gate = S.pcg_gate(n, prev['r'], cur['z'], cur['p'], cur['Ap'], prev['x'], cur['x'], cur['r'])
      if n_loops(g) == 0 or all(k[0] == 0 or k[1] == 0 for k in ed[n - 1:]):
        note('one CG iteration', S.one_iteration_gate(Ld, Ls, Lk, Hd, M, ed, lam, gn, cur['z'], gate['alpha'],
                                                      cur['r'], n))
    else:
      pp = cap(c - 2)
      gate = S.pcg_gate(n, prev['r'], cur['z'], cur['p'], cur['Ap'], prev['x'], cur['x'], cur['r'],
                        p_prev2=prev['p'], r_prev2=pp['r'], z_prev2=prev['z'])
    note('pcg', gate)
  # the stop: every c when there are few, else the last two
  cs = range(1, count + 1) if count <= 40 else (count - 1, count)
  norms = {c: float(np.linalg.norm(cap(c)['r'][1:])) for c in cs}
  ok, ties = S.cg_stop(norms, gn, P.DEFAULTS['cg_tol'], count, P.DEFAULTS['max_cg_iterations'])
  assert ok, (name, count, norms)
  # exact arithmetic needs at most 12 L + 1 iterations; reported, not gated: at lam = 1e-12 an H100 took 21 of 25
  L = n_loops(g)
  print('%s: trial 1 took %d CG iterations (12 L + 1 = %d for L = %d loops), %d near-ties' % (
      name, count, 12 * L + 1, L, ties))


def test_restarted_trials_are_the_original_trials(eng):
  g, _ = synth.pose_graph_scene(300, 20, seed=5, n_false=4, init_noise=(0.1, 0.02))
  full = run(eng, g, {})
  t = full['trace']
  K = len(t['cost'])
  assert K >= 4 and S.lm_gate(t, P.DEFAULTS['lambda_min'])
  for k in sorted({2, K // 2, K}):
    before = run(eng, g, {}, max_iterations=k - 1)
    again = run(eng, dict(g, poses=before['poses']), {}, max_iterations=1, lambda0=float(t['lambda'][k - 1]))
    for key in ('cost', 'lambda', 'accepted', 'cg_iterations'):
      assert np.array_equal(S.bits_equal(again['trace'][key][:1].astype(np.float64),
                                         t[key][k - 1:k].astype(np.float64))['frac'], 0.0), (k, key)
    assert bool(again['trace']['accepted'][0]) == bool(again['trace']['cost'][0] < again['initial_cost'])
    T, M, q, Hd, gn, Ld, Ls, Lk, Tt, x = ws(eng, 'T', 'M', 'q', 'Hd', 'gn', 'Ld', 'Ls', 'Lk', 'Tt', 'x')
    if again['trace']['accepted'][0]:
      T = before['poses']                # M, q, Hd and gn are those of the new T now
      r0 = run(eng, dict(g, poses=T), {}, max_iterations=0)
      M, q, Hd, gn = ws(eng, 'M', 'q', 'Hd', 'gn')
      assert r0['initial_cost'] == again['initial_cost']
    note('factor', S.factor_gate(Ld, Ls, Lk, Hd, M, float(t['lambda'][k - 1]), 300))
    note('update', S.update_gate(T, x, Tt))
    note('cost', S.cost_gate(g, Tt, P.DEFAULTS['phi'], again['trace']['cost'][0]))
    print('trial %d of %d: %d CG iterations (12 L + 1 = %d)' % (k, K, again['cg_iterations'], 12 * 24 + 1))


def defined(name, n, E):
  """the positions ovn_pgo_copy_workspace defines for a graph of n nodes"""
  if name in ('M', 'q'):
    return np.ones(E, bool)
  m = np.zeros(n, bool)
  if name in ('T', 'Tt', 'Hd', 'gn'):
    m[:] = True
    return m
  m[1:] = True
  P_ = S.separators(n)
  if name == 'Ls':
    m[P_[1:-1]] = False
    m[n - 1] = False
  if name == 'Lk':
    m[:P_[1] + 1 if len(P_) > 2 else n] = False
  return m


def test_a_graph_reads_back_the_same_alone_and_in_a_batch(eng):
  g = with_loops(57, [(8, 12), (7, 21), (0, 30)], seed=57)
  others = [synth.pose_graph_scene(20 + 41 * k, 2 + k, seed=30 + k)[0] for k in range(6)]
  eng.pose_graph([g])
  alone = {k: eng.pose_graph_workspace(k) for k in PGO_ARRAYS}
  eng.pose_graph(others[:3] + [g] + others[3:])
  n, E = len(g['poses']), len(g['edges'])
  for k in PGO_ARRAYS:
    got = eng.pose_graph_workspace(k, graph=3)
    m = defined(k, n, E)
    assert np.array_equal(S.bits_equal(got[m], alone[k][m])['frac'], 0.0), k


def test_readback_refusals(eng):
  L = lib()
  fresh = Engine(precision='fp32', max_batch_scans=1, max_batch_pairs=1)
  try:
    with pytest.raises(OvnError, match='no successful'):
      fresh.pose_graph_workspace('T')
  finally:
    fresh.close()
  g, _ = synth.pose_graph_scene(12, 2, seed=0)
  eng.pose_graph([g, g])
  out = np.empty(12 * 16)
  ptr = out.ctypes.data_as(C.c_void_p)
  assert L.ovn_pgo_copy_workspace(eng._h, 0, 1, ptr) == 0
  for array, graph in ((15, 0), (-1, 0), (0, 2), (0, -1)):
    assert L.ovn_pgo_copy_workspace(eng._h, array, graph, ptr) == -1, (array, graph)
  assert L.ovn_pgo_copy_workspace(eng._h, 0, 0, None) == -1
  with pytest.raises(OvnError):
    eng.pose_graph_workspace('x', graph=2)
  # a refused call invalidates the record
  bad = pg.default_params({'phi': 0.0})
  node_off, edge_off = np.array([0, 12]), np.array([0, len(g['edges'])])
  rc = eng.pose_graph_raw(node_off, edge_off, g['poses'], g['edges'], g['measurements'], g['weights'], bad)['rc']
  assert rc == -1
  assert L.ovn_pgo_copy_workspace(eng._h, 0, 0, ptr) == -1
  with pytest.raises(OvnError, match='no successful'):
    eng.pose_graph_workspace('T')
  eng.pose_graph([g])
  assert eng.pose_graph_workspace('T').shape == (12, 4, 4)
