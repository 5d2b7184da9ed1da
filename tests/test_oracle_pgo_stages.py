"""The pose-graph stage model (oracle/pgo_stages.py) on the CPU: its NumPy restatement of the kernel's gather, factor,
substitutions and matvec passes every gate against the exact sparse model, and each mutant of those stages exceeds
its gate (a mutant factor that meets a non-positive pivot is rejected too: the kernel would return
OVN_PGO_FAILED)."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

from oracle import pgo_stages as S
from oracle import pose_graph as P
from overlapnet_b200 import synth

# (n, loops): the separator layouts of the GPU file, with loops where the graph has room
CASES = [(2, 0), (3, 0), (9, 1), (10, 2), (17, 3), (18, 0), (57, 5), (300, 20)]


def kernel_edges(g, phi=25.0):
  """M (upper triangle mirrored, as the kernel writes it) and q of every edge at the graph's poses"""
  ed = g['edges']
  e, A = P.jacobian(g['poses'][ed[:, 0]], g['poses'][ed[:, 1]], g['measurements'])
  _, chi2, s, _, _ = P.linearize(g, g['poses'], phi)
  d = s * s
  M = d[:, None, None] * np.einsum('kri,kr,krj->kij', A, g['weights'], A)
  M = np.triu(M) + np.swapaxes(np.triu(M, 1), 1, 2)
  q = d[:, None] * np.einsum('kri,kr,kr->ki', A, g['weights'], e)
  return M, q, chi2, s


def case(n, loops, lam=1e-6):
  g, _ = synth.pose_graph_scene(n, loops, seed=n, min_gap=min(3, n - 1), n_false=1 if loops else 0)
  M, q, chi2, s = kernel_edges(g)
  Hd, gn = S.gather(M, q, g['edges'], n)
  r = np.zeros((n, 6))
  r[1:] = -gn[1:]
  return dict(g=g, n=n, M=M, q=q, chi2=chi2, s=s, Hd=Hd, gn=gn, r=r, lam=lam, ed=g['edges'])


@pytest.mark.parametrize('n,loops', CASES)
def test_the_restatement_passes_every_gate(n, loops):
  c = case(n, loops)
  Hd, M, lam, ed = c['Hd'], c['M'], c['lam'], c['ed']
  # the gather equals the oracle's gradient, and Hd + the chain is the oracle's H
  _, _, _, grad, H = P.linearize(c['g'], c['g']['poses'], 25.0)
  assert np.abs(c['gn'] - grad).max() <= 1e-12 * np.abs(grad).max()
  A = S.system(Hd, M, ed, 0.0, n)
  assert abs(A - H[6:, 6:]).max() <= 1e-12 * abs(H).max()
  assert S.gather_gate(M, c['q'], Hd, c['gn'], ed, n)['worst'] == 0
  Ld, Ls, Lk = S.factor(Hd, M, lam, n)
  f = S.factor_gate(Ld, Ls, Lk, Hd, M, lam, n)
  assert f['structure'] and f['worst'] <= 1, f
  y, z = S.apply(Ld, Ls, Lk, c['r'], n)
  assert S.apply_gate(Ld, Ls, Lk, c['r'], y, z, n)['worst'] <= 1
  zex = spla.spsolve(S.preconditioner(Hd, M, lam, n).tocsc(), c['r'][1:].ravel())
  assert np.abs(z[1:].ravel() - zex).max() <= 1e-8 * np.abs(zex).max()
  Ap = S.matvec(Hd, M, ed, lam, z, n)
  assert S.matvec_gate(Hd, M, ed, lam, z, Ap, n)['worst'] <= 1
  # one exact PCG step: x_1 = alpha z_0, r_1 = r_0 - alpha A z_0
  rz = np.dot(c['r'][1:].ravel(), z[1:].ravel())
  alpha = rz / np.dot(z[1:].ravel(), Ap[1:].ravel())
  x1, r1 = alpha * z, c['r'] - alpha * Ap
  x0 = np.zeros((n, 6))
  assert S.pcg_gate(n, c['r'], z, z, Ap, x0, x1, r1)['worst'] <= 1
  if loops == 0:
    assert S.one_iteration_gate(Ld, Ls, Lk, Hd, M, ed, lam, c['gn'], z, alpha, r1, n)['worst'] <= 1
  e = S.edge_gate(c['g'], c['g']['poses'], 25.0, c['chi2'], c['s'], M, c['q'])
  assert e['worst'] <= 1, e


def _rejected(gate):
  return not gate['worst'] <= 1


# mutants run where the code they break runs: segments with a left separator and interior nodes
MUTANT_CASES = [(10, 2), (57, 5), (300, 20)]


@pytest.mark.parametrize('n,loops', MUTANT_CASES)
@pytest.mark.parametrize('mutant', S.MUTANTS_FACTOR)
def test_factor_mutants_exceed_the_gate(n, loops, mutant):
  c = case(n, loops)
  try:
    Ld, Ls, Lk = S.factor(c['Hd'], c['M'], c['lam'], n, mutant)
  except np.linalg.LinAlgError:
    print('%s, n %d: a non-positive pivot' % (mutant, n))
    return
  g = S.factor_gate(Ld, Ls, Lk, c['Hd'], c['M'], c['lam'], n)
  print('%s, n %d: %.3g of %d elements over the gate' % (mutant, n, g['frac'], g['n']))
  assert _rejected(g) and g['frac'] > 0


@pytest.mark.parametrize('n,loops', MUTANT_CASES)
def test_apply_mutant_exceeds_the_gate(n, loops):
  c = case(n, loops)
  Ld, Ls, Lk = S.factor(c['Hd'], c['M'], c['lam'], n)
  y, z = S.apply(Ld, Ls, Lk, c['r'], n, 'no_sR_coupling')
  g = S.apply_gate(Ld, Ls, Lk, c['r'], y, z, n)
  print('no_sR_coupling, n %d: forward %.3g, backward %.3g over the gate' % (n, g['fwd']['frac'], g['bwd']['frac']))
  assert _rejected(g)


@pytest.mark.parametrize('n,loops', MUTANT_CASES)
def test_matvec_mutant_exceeds_the_gate(n, loops):
  c = case(n, loops)
  v = np.random.default_rng(n).normal(size=(n, 6))
  Ap = S.matvec(c['Hd'], c['M'], c['ed'], c['lam'], v, n, 'wrong_loop_end')
  g = S.matvec_gate(c['Hd'], c['M'], c['ed'], c['lam'], v, Ap, n)
  print('wrong_loop_end, n %d: %.3g of %d elements over the gate' % (n, g['frac'], g['n']))
  assert _rejected(g) and g['frac'] > 0


@pytest.mark.parametrize('n,loops', MUTANT_CASES)
@pytest.mark.parametrize('mutant', S.MUTANTS_GATHER)
def test_gather_mutants_break_the_bits(n, loops, mutant):
  c = case(n, loops)
  Hd, gn = S.gather(c['M'], c['q'], c['ed'], n, mutant)
  g = S.gather_gate(c['M'], c['q'], Hd, gn, c['ed'], n)
  print('%s, n %d: Hd %.3g, gn %.3g of the elements differ' % (mutant, n, g['Hd']['frac'], g['gn']['frac']))
  assert _rejected(g)


def test_cg_stop_rule():
  g = np.zeros((3, 6))
  g[1:] = 1.0
  thr = 1e-12 * np.sqrt(12.0)
  assert S.cg_stop({1: 1.0, 2: 2 * thr, 3: 0.5 * thr}, g, 1e-12, 3, 100) == (True, 0)
  assert S.cg_stop({1: 1.0, 2: 0.5 * thr, 3: 0.5 * thr}, g, 1e-12, 3, 100)[0] is False      # stopped late
  assert S.cg_stop({1: 1.0, 2: 2 * thr}, g, 1e-12, 2, 100)[0] is False                     # stopped early
  assert S.cg_stop({1: 1.0, 2: 2 * thr}, g, 1e-12, 2, 2) == (True, 0)                       # at the cap
  assert S.cg_stop({1: 1.0, 2: thr * (1 + 1e-16)}, g, 1e-12, 2, 100) == (True, 1)           # a near-tie is not judged


def test_lm_schedule_and_separators():
  assert S.lm_gate({'lambda': [1e-6, 1e-7, 1e-6], 'accepted': [1, 0, 1]}, 1e-12)
  assert not S.lm_gate({'lambda': [1e-6, 1e-5], 'accepted': [1, 1]}, 1e-12)
  assert S.lm_gate({'lambda': [1e-12, 1e-12], 'accepted': [1, 1]}, 1e-12)
  assert S.separators(2) == [0, 2] and S.separators(3) == [0, 1, 3]
  assert S.separators(9) == [0, 1, 2, 3, 4, 5, 6, 7, 9]
  assert S.separators(10) == [0, 2, 4, 6, 8, 10] and S.separators(18) == [0, 3, 6, 9, 12, 15, 18]
  assert S.separators(1101) == [0] + [138 * q for q in range(1, 8)] + [1101]
