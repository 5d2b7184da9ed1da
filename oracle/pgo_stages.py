"""Float64 stage model of the pose-graph optimizer (k_pgo_graphs, csrc/pose_graph.cu) and the gates each stage read
back by ovn_pgo_copy_workspace (Engine.pose_graph_workspace) must pass.  Test infrastructure only; it builds on
oracle/pose_graph.py.

The kernel's layout.  Over the free nodes 1 .. n-1 a separator sits every len = ceil((n - 1) / 8) nodes, at q len for
q = 1 .. Q while q len < n - 1; segment w (w = 0 .. Q) is the nodes strictly between P[w] and P[w + 1], with P[0] = 0
and P[Q + 1] = n.  The preconditioner is the block tridiagonal Ã = blocktridiag(Hd_i + lam diag(Hd_i), -M_i) over
nodes 1 .. n-1 (chain edge i joins i and i + 1); the system is A = H + lam diag(H), which adds each loop edge's -M_k
at (a, b) and (b, a).  The factor L̂ is lower triangular in nested-dissection order (every segment's nodes in order,
then the separators in order): Ld_j on the diagonal, Ls_j at (j + 1, j) inside a segment and at (sR, last node),
Lk_j at (sL, j) for the nodes of segments 1 .. Q (the spikes), and Lk_s at (s_q, s_{q-1}) for separators q >= 2.

Notation: u = 2^-53, gamma(k) = k u / (1 - k u).  Every bound below is first order in u; the long double reference
(64-bit significand on x86, more elsewhere) adds at most 2^-11 of it, covered by the factor REF = 1 + 2^-10.

Gates (err / bound <= 1 everywhere, per element):

  edge      chi2, s, M, q at the GPU's T against oracle.pose_graph.jacobian / rho in long double.  edge_model
            propagates absolute rounding bounds through the kernel's formulas: u = Ta_R^T ta + tZ (4 terms, gamma(4)),
            RC (3 terms, gamma(3)), tC (gamma(3) plus RC's and u's), R_E = RC Tb_R (gamma(3) plus RC's), t_E = RC tb + tC
            (gamma(4) plus the others': with translations of hundreds of metres this is a cancelling difference whose
            absolute error, not its size, sets the bound).  Log: |dphi| <= 9 max(1, th / (2 sin th)) eps_R + 8 u th,
            with eps_R the largest bound of R_E (the antisymmetric formula amplifies by th / sn, sn = 2 sin th; the
            symmetric branch above pi - PI_BRANCH by at most 9).  J_l^-1: |dJ| <= 1.5 |dphi| + gamma(8) |J| since
            |dJ/dphi| <= 1/2 + 2 c th + |c'| th^2 <= 1.3 for th <= pi.  A: products of 3 terms, gamma(3) plus the
            inputs'.  chi2: sum w (2 |e| de + de^2) + gamma(7) chi2.  s = phi / (phi + chi2): s (dchi2 / (phi + chi2)
            + 3 u); d = s^2.  M = d A^T W A and q = d A^T W e: d sum w (dA |A| + |A| dA) + gamma(7) d sum w |A| |A|
            + dd sum w |A| |A| (|e| and de in place of the second |A| and dA for q).  On the chain (and phi = inf)
            s = 1 exactly.
  gather    Hd, gn: the kernel's sums in float64 in its order (chain (i - 1, i), chain (i, i + 1), loops in edge
            order, from +0.0) of the GPU's own M and q: pure adds and exact +-1 products, so bit-exact.
  factor    Ld lower triangular, positive diagonal, upper part exactly 0; |P Ã P^T - L̂ L̂^T| <= gamma(2 K + 12)
            |L̂| |L̂^T| componentwise over the union of both patterns, fill positions (Ã = 0) included.  K = 6 times
            the most blocks in a row of L̂ (a separator's row: Ld, Lk to the previous separator, the left segment's last
            Ls and the right segment's spikes), so K bounds every inner product the kernel accumulates, in any order;
            + 4 covers the subtractions of the Schur sums, the sqrt and the division; the damped diagonal's two
            roundings are <= gamma(2) |Ã_ii| <= gamma(2) (|L̂||L̂^T|)_ii; doubling covers numpy's own L̂ L̂^T.
  apply     y and z = M^-1 r from the GPU's L̂ and r: |r - L̂ ŷ| <= gamma(2 K + 12) |L̂| |ŷ| and |ŷ - L̂^T ẑ| <=
            gamma(2 K + 12) |L̂^T| |ẑ| (triangular solves are componentwise backward stable with the same K); this does
            not depend on the conditioning.
  matvec    Ap against A p from the GPU's Hd, M and p: <= gamma(2 m + 2) (|A| |p|)_i with m the row's nonzeros plus
            the damping term (the kernel's and numpy's sums each of at most m + 1 terms).
  pcg       x_c = x_{c-1} + alpha p_{c-1}, r_c = r_{c-1} - alpha Ap and p_{c-1} = z_{c-1} + beta p_{c-2}, alpha and
            beta recomputed from the GPU's vectors: 3 u (|out| + |coef term|) + e_coef |coef term|, with e_coef =
            2 gamma(N) (sum |a_i b_i| / |a . b| of each dot product) + 4 u, N = 6 (n - 1) (the kernel's block sum and
            numpy's dot each).  p_0 = z_0 exactly.
  cg stop   ||r_c|| <= cg_tol ||g|| first at the GPU's count, except within gamma(N + 2) (||r|| + cg_tol ||g||) of the
            threshold (near-ties, counted).
  update    Tt against oracle update(T, x) in long double: node 0 bit-identical; rows of nodes 1 .. n-1 within
            gamma(28) (sum_k |T_kj| + |v_i| [j = 3]): R(omega) is exact to 24 u absolute (sqrt, division, sin / cos
            of 2 ulp, 1 - cos, K^2), and each entry of R T + v is a 4-term sum.
  cost      the trial's F against evaluate(Tt) in long double: 1/2 sum rho' dchi2 + gamma(E) F (edge_model's dchi2).
  decisions accepted == (Ft < F), F the cost the trial started from, and lam_{k+1} = max(lam_k / 10, lam_min)
            or 10 lam_k: bit-exact.
  one CG    loop-free, the preconditioner is the system, so after one iteration |r_1| <= (e_alpha + gamma(3 K + 20))
            (|L̂| |L̂^T| |z_0| + |A| |z_0| + |g|): the backward errors of the factor and the two solves, the matvec and
            the update of r, with z_0 = p_0.  With L loops A - Ã has rank <= 12 L, so exact arithmetic needs at most
            12 L + 1 iterations.
"""
import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp

from . import pose_graph as P

U = 2.0 ** -53
WARPS = 8               # k_pgo_graphs' warps: one chain segment each
REF = 1.0 + 2.0 ** -10
LD = np.longdouble
MUTANTS_FACTOR = ('spike_dropped', 'fill_transposed', 'no_dLL', 'no_dRR', 'separators_undamped',
                  'separators_shifted')
MUTANTS_APPLY = ('no_sR_coupling',)
MUTANTS_MATVEC = ('wrong_loop_end',)
MUTANTS_GATHER = ('loop_sign_swapped', 'order_changed')


def gamma(k):
  return k * U / (1 - k * U)


def separators(n):
  """P = [0, s_1 .. s_Q, n] as the kernel places them"""
  m = n - 1
  ln = (m + WARPS - 1) // WARPS
  return [0] + [q * ln for q in range(1, WARPS + 1) if q * ln < n - 1] + [n]


def segments(P):
  """(a, b, sL, sR) of segment w = 0 .. Q: its nodes are a .. b - 1; sL / sR are None at the ends"""
  Q = len(P) - 2
  return [(P[w] + 1, P[w + 1], P[w] if w >= 1 else None, P[w + 1] if w + 1 <= Q else None) for w in range(Q + 1)]


def nd_order(n, P=None):
  """the free nodes 1 .. n-1 in nested-dissection order"""
  P = separators(n) if P is None else P
  return [j for a, b, _, _ in segments(P) for j in range(a, b)] + P[1:-1]


def _damp(B, lam):
  return B + np.diag(lam * np.diag(B))


def _blocks(n, entries):
  """sparse [6(n-1)]^2 over nodes 1 .. n-1 from {(i, j): 6x6 block}"""
  rows, cols, vals = [], [], []
  ii, jj = np.meshgrid(np.arange(6), np.arange(6), indexing='ij')
  for (i, j), B in entries.items():
    rows.append(6 * (i - 1) + ii.ravel())
    cols.append(6 * (j - 1) + jj.ravel())
    vals.append(np.asarray(B, np.float64).ravel())
  if not rows:
    return sp.csr_matrix((6 * (n - 1), 6 * (n - 1)))
  return sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))),
                       shape=(6 * (n - 1), 6 * (n - 1))).tocsr()


def preconditioner(Hd, M, lam, n):
  """Ã over nodes 1 .. n-1 (natural order)"""
  ent = {(i, i): _damp(Hd[i], lam) for i in range(1, n)}
  for i in range(1, n - 1):
    ent[(i + 1, i)] = -M[i]
    ent[(i, i + 1)] = -M[i].T
  return _blocks(n, ent)


def system(Hd, M, edges, lam, n):
  """A = H + lam diag(H) over nodes 1 .. n-1 from the diagonal blocks Hd and every edge's M"""
  A = preconditioner(Hd, M, lam, n).tolil()
  for k in range(n - 1, len(edges)):
    a, b = int(edges[k][0]), int(edges[k][1])
    if a >= 1 and b >= 1:
      A[6 * (a - 1):6 * a, 6 * (b - 1):6 * b] -= M[k]
      A[6 * (b - 1):6 * b, 6 * (a - 1):6 * a] -= M[k]
  return A.tocsr()


# ---- the kernel's stages restated in NumPy (mutants are built on these) -------------------------------------------
def gather(M, q, edges, n, mutant=None):
  """Hd [n, 6, 6], gn [n, 6]: the kernel's per-node sums in its order"""
  assert mutant in (None,) + MUTANTS_GATHER
  Hd, g = np.zeros((n, 6, 6)), np.zeros((n, 6))
  loops = range(n - 1, len(edges))

  def add_loops():
    for k in loops:
      a, b = int(edges[k][0]), int(edges[k][1])
      Hd[a] += M[k]
      Hd[b] += M[k]
      sa, sb = (1.0, -1.0) if mutant == 'loop_sign_swapped' else (-1.0, 1.0)
      g[a] += sa * q[k]
      g[b] += sb * q[k]
  if mutant == 'order_changed':
    add_loops()
  Hd[1:] += M[:n - 1]
  g[1:] += q[:n - 1]
  Hd[:n - 1] += M[:n - 1]
  g[:n - 1] -= q[:n - 1]
  if mutant != 'order_changed':
    add_loops()
  return Hd, g


def _trsm(L, B):
  """B L^-T"""
  return sla.solve_triangular(L, B.T, lower=True).T


def factor(Hd, M, lam, n, mutant=None):
  """Ld, Ls, Lk [n, 6, 6] as the kernel factors Ã (positions it never writes are NaN)"""
  assert mutant in (None,) + MUTANTS_FACTOR
  P = separators(n)
  if mutant == 'separators_shifted':
    P = [0] + [s + 1 for s in P[1:-1]] + [n]
  Q = len(P) - 2
  Ld, Ls, Lk = (np.full((n, 6, 6), np.nan) for _ in range(3))
  dLL, dRR, fill = {}, {}, {}
  for w, (a, b, sL, sR) in enumerate(segments(P)):
    dL = np.zeros((6, 6))
    F = -M[sL] if sL is not None and a < b else None
    Lp = None
    for j in range(a, b):
      D = _damp(Hd[j], lam)
      if j > a:
        D = D - Lp @ Lp.T
      L = np.linalg.cholesky(D)
      Ld[j] = L
      if sL is not None:
        F = _trsm(L, F)
        Lk[j] = 0.0 if mutant == 'spike_dropped' else F
        dL = dL + F @ F.T
      if j + 1 < n:
        Tm = _trsm(L, -M[j])
        Ls[j] = Tm
        if sL is not None:
          F = -(F @ Tm.T).T if mutant == 'fill_transposed' else -(F @ Tm.T)
        Lp = Tm
    dLL[w] = dL
    if a < b and sR is not None:
      dRR[w] = Lp @ Lp.T
      if sL is not None:
        fill[w] = F
    elif sL is not None and sR is not None:
      fill[w] = -M[sL]
  Lprev = None
  for qq in range(1, Q + 1):
    s = P[qq]
    D = Hd[s].copy() if mutant == 'separators_undamped' else _damp(Hd[s], lam)
    if P[qq - 1] + 1 < s and mutant != 'no_dRR':
      D -= dRR[qq - 1]
    if s + 1 < P[qq + 1] and mutant != 'no_dLL':
      D -= dLL[qq]
    if qq >= 2:
      Tm = _trsm(Lprev, fill[qq - 1].T)
      Lk[s] = Tm
      D -= Tm @ Tm.T
    Lprev = Ld[s] = np.linalg.cholesky(D)
  return Ld, Ls, Lk


def apply(Ld, Ls, Lk, v, n, mutant=None):
  """(y, z): the kernel's forward and back substitutions of v [n, 6] through its factor"""
  assert mutant in (None,) + MUTANTS_APPLY
  P = separators(n)
  Q = len(P) - 2
  segs = segments(P)
  y, z = np.full((n, 6), np.nan), np.full((n, 6), np.nan)
  cL, cR = np.zeros((Q + 1, 6)), np.zeros((Q + 1, 6))
  for w, (a, b, sL, sR) in enumerate(segs):
    for j in range(a, b):
      t = v[j] - (Ls[j - 1] @ y[j - 1] if j > a else 0.0)
      y[j] = sla.solve_triangular(Ld[j], t, lower=True)
      if sL is not None:
        cL[w] += Lk[j] @ y[j]
    if a < b and sR is not None and mutant != 'no_sR_coupling':
      cR[w] = Ls[b - 1] @ y[b - 1]
  for qq in range(1, Q + 1):
    s = P[qq]
    t = v[s] - (cR[qq - 1] + cL[qq]) - (Lk[s] @ y[P[qq - 1]] if qq >= 2 else 0.0)
    y[s] = sla.solve_triangular(Ld[s], t, lower=True)
  for qq in range(Q, 0, -1):
    s = P[qq]
    t = y[s] - (Lk[P[qq + 1]].T @ z[P[qq + 1]] if qq < Q else 0.0)
    z[s] = sla.solve_triangular(Ld[s], t, lower=True, trans='T')
  for a, b, sL, sR in segs:
    for j in range(b - 1, a - 1, -1):
      t = y[j].copy()
      if j < b - 1:
        t -= Ls[j].T @ z[j + 1]
      elif sR is not None and mutant != 'no_sR_coupling':
        t -= Ls[j].T @ z[sR]
      if sL is not None:
        t -= Lk[j].T @ z[sL]
      z[j] = sla.solve_triangular(Ld[j], t, lower=True, trans='T')
  return y, z


def matvec(Hd, M, edges, lam, v, n, mutant=None):
  """Ap [n, 6] (node 0 NaN) as the kernel forms (H + lam diag(H)) v"""
  assert mutant in (None,) + MUTANTS_MATVEC
  out = np.full((n, 6), np.nan)
  nbr = [[] for _ in range(n)]
  for k in range(n - 1, len(edges)):
    a, b = int(edges[k][0]), int(edges[k][1])
    nbr[a].append((k, a if mutant == 'wrong_loop_end' else b))
    nbr[b].append((k, a))
  for i in range(1, n):
    o = Hd[i] @ v[i] + lam * np.diag(Hd[i]) * v[i]
    if i - 1 >= 1:
      o -= M[i - 1] @ v[i - 1]
    if i + 1 <= n - 1:
      o -= M[i] @ v[i + 1]
    for k, j in nbr[i]:
      if j != 0:
        o -= M[k] @ v[j]
    out[i] = o
  return out


# ---- assembly and gates -------------------------------------------------------------------------------------------
def assemble(Ld, Ls, Lk, n):
  """(L̂ sparse lower triangular in nested-dissection order, the order, K) from the defined positions only"""
  P = separators(n)
  order = nd_order(n, P)
  pos = {j: t for t, j in enumerate(order)}
  ent, rowblocks = {}, {j: 1 for j in order}
  for w, (a, b, sL, sR) in enumerate(segments(P)):
    for j in range(a, b):
      ent[(j, j)] = Ld[j]
      if j + 1 < b:
        ent[(j + 1, j)] = Ls[j]
        rowblocks[j + 1] += 1
      elif sR is not None:
        ent[(sR, j)] = Ls[j]
        rowblocks[sR] += 1
      if sL is not None:
        ent[(sL, j)] = Lk[j]
        rowblocks[sL] += 1
  for qq, s in enumerate(P[1:-1], 1):
    ent[(s, s)] = Ld[s]
    if qq >= 2:
      ent[(s, P[qq - 1])] = Lk[s]
      rowblocks[s] += 1
  L = _blocks(n, {(pos[i] + 1, pos[j] + 1): B for (i, j), B in ent.items()})
  return L, order, 6 * max(rowblocks.values())


def _perm(n, order):
  return np.concatenate([6 * (j - 1) + np.arange(6) for j in order])


def _vec(v, n, order):
  """v [n, 6] -> the free nodes in `order`, flattened"""
  return np.asarray(v)[order].reshape(-1)


def ratio(err, bound):
  """{'worst': max err / bound, 'frac': fraction over the bound, 'n': elements} (0 / 0 = 0)"""
  err, bound = np.abs(np.asarray(err, np.float64)).ravel(), np.asarray(bound, np.float64).ravel()
  with np.errstate(divide='ignore', invalid='ignore'):
    r = np.where(err == 0, 0.0, err / np.where(bound > 0, bound, 0.0)) if err.size else np.zeros(0)
    over = ~(err <= bound)
  return {'worst': float(r.max()) if r.size else 0.0, 'frac': float(over.mean()) if r.size else 0.0,
          'n': int(err.size)}


def _sparse_ratio(D, B):
  """ratio of |D| to B over the union of their patterns"""
  S = (abs(D) + B).tocoo()
  err = np.asarray(abs(D).tocsr()[S.row, S.col]).ravel()
  bnd = np.asarray(B.tocsr()[S.row, S.col]).ravel()
  return ratio(err, bnd)


def factor_gate(Ld, Ls, Lk, Hd, M, lam, n):
  """the factor's gates: Ld's structure, and the componentwise backward error of L̂ L̂^T against P Ã P^T"""
  Lt = Ld[1:]
  upper = np.triu(np.ones((6, 6), bool), 1)
  structure = bool(np.all(Lt[:, upper] == 0) and np.all(np.diagonal(Lt, axis1=1, axis2=2) > 0))
  L, order, K = assemble(Ld, Ls, Lk, n)
  p = _perm(n, order)
  At = preconditioner(Hd, M, lam, n)[p][:, p]
  aL = abs(L)
  g = _sparse_ratio(L @ L.T - At, gamma(2 * K + 12) * (aL @ aL.T))
  return dict(g, structure=structure, K=K)


def apply_gate(Ld, Ls, Lk, r, y, z, n):
  """the two substitutions' componentwise backward errors from the GPU's L̂, r, y and z"""
  L, order, K = assemble(Ld, Ls, Lk, n)
  rv, yv, zv = _vec(r, n, order), _vec(y, n, order), _vec(z, n, order)
  gm = gamma(2 * K + 12)
  fwd = ratio(rv - L @ yv, gm * (abs(L) @ np.abs(yv)))
  bwd = ratio(yv - L.T @ zv, gm * (abs(L).T @ np.abs(zv)))
  return {'fwd': fwd, 'bwd': bwd, 'worst': max(fwd['worst'], bwd['worst']), 'K': K}


def matvec_gate(Hd, M, edges, lam, p, Ap, n):
  A = system(Hd, M, edges, lam, n)
  pv = np.asarray(p)[1:].reshape(-1)
  m = np.diff(A.indptr) + 1
  return ratio(np.asarray(Ap)[1:].reshape(-1) - A @ pv, (2 * m + 2) * U / (1 - (2 * m + 2) * U) * (abs(A) @ np.abs(pv)))


def bits_equal(a, b):
  """{'worst': 0 or inf, 'frac': fraction of elements whose bits differ}"""
  a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
  diff = a.view(np.uint64) != b.view(np.uint64)
  return {'worst': float('inf') if diff.any() else 0.0, 'frac': float(diff.mean()), 'n': int(diff.size)}


def gather_gate(M, q, Hd, gn, edges, n):
  rH, rg = gather(M, q, edges, n)
  h, g = bits_equal(Hd, rH), bits_equal(gn, rg)
  return {'Hd': h, 'gn': g, 'worst': max(h['worst'], g['worst'])}


def _dot_cond(a, b):
  d = float(np.dot(a, b))
  return np.sum(np.abs(a * b)) / abs(d) if d != 0 else np.inf


def pcg_gate(n, r_prev, z_prev, p_prev, Ap, x_prev, x, r, p_prev2=None, r_prev2=None, z_prev2=None):
  """iteration c from the GPU's vectors [n, 6] (node 0 ignored): r_prev = r_{c-1}, z_prev = z_{c-1}, p_prev =
  p_{c-1}, Ap = A p_{c-1}, x_prev = x_{c-1}; x, r = x_c, r_c.  With p_prev2 = p_{c-2}, r_prev2, z_prev2 (c >= 2)
  also p_{c-1} = z_{c-1} + beta p_{c-2}; without (c = 1) p_0 == z_0 bit for bit."""
  f = lambda v: np.asarray(v)[1:].reshape(-1)  # noqa: E731
  rp, zp, pp, ap, xp, xc, rc = map(f, (r_prev, z_prev, p_prev, Ap, x_prev, x, r))
  N = rp.size
  alpha = float(np.dot(rp, zp)) / float(np.dot(pp, ap))
  e_a = 2 * gamma(N) * (_dot_cond(rp, zp) + _dot_cond(pp, ap)) + 4 * U
  out = {'alpha': alpha}
  out['x'] = ratio(xc - (xp + alpha * pp), 3 * U * (np.abs(xc) + np.abs(alpha * pp)) + e_a * np.abs(alpha * pp))
  out['r'] = ratio(rc - (rp - alpha * ap), 3 * U * (np.abs(rc) + np.abs(alpha * ap)) + e_a * np.abs(alpha * ap))
  if p_prev2 is None:
    out['p'] = bits_equal(pp, zp)
  else:
    pq, rq, zq = map(f, (p_prev2, r_prev2, z_prev2))
    beta = float(np.dot(rp, zp)) / float(np.dot(rq, zq))
    e_b = 2 * gamma(N) * (_dot_cond(rp, zp) + _dot_cond(rq, zq)) + 4 * U
    out['p'] = ratio(pp - (zp + beta * pq), 3 * U * (np.abs(pp) + np.abs(beta * pq)) + e_b * np.abs(beta * pq))
    out['beta'] = beta
  out['worst'] = max(out[k]['worst'] for k in ('x', 'r', 'p'))
  return out


def cg_stop(r_norms, g, cg_tol, count, max_cg):
  """whether the kernel stopped where ||r_c|| <= cg_tol ||g|| first holds: r_norms = {c: ||r_c||} (numpy's, from the
  GPU's r_c) for any c in 1 .. count.  Returns (ok, ties): a comparison within the norms' rounding of the threshold
  is a tie and is not judged."""
  gv = np.asarray(g)[1:].reshape(-1)
  N = gv.size
  thr = cg_tol * float(np.sqrt(np.dot(gv, gv)))
  ties, ok = 0, True
  for c, rn in r_norms.items():
    if abs(rn - thr) <= gamma(N + 2) * (rn + thr):
      ties += 1
      continue
    below = rn <= thr
    if c < count and below:
      ok = False
    if c == count and not below and count < max_cg:
      ok = False
  return ok, ties


def one_iteration_gate(Ld, Ls, Lk, Hd, M, edges, lam, g, z0, alpha, r1, n):
  """loop-free: |r_1| <= (e_alpha + gamma(3 K + 20)) (|L̂||L̂^T||z_0| + |A||z_0| + |g|) componentwise"""
  L, order, K = assemble(Ld, Ls, Lk, n)
  p = _perm(n, order)
  A = system(Hd, M, edges, lam, n)
  zv, gv = np.asarray(z0)[1:].reshape(-1), np.asarray(g)[1:].reshape(-1)
  aL = abs(L)
  LL = np.empty_like(zv)
  LL[p] = aL @ (aL.T @ np.abs(zv[p]))
  N = zv.size
  Az = A @ zv
  e_a = 2 * gamma(N) * (_dot_cond(gv, zv) + _dot_cond(zv, Az)) + 4 * U
  return ratio(np.asarray(r1)[1:].reshape(-1), (e_a + gamma(3 * K + 20)) * (LL + abs(A) @ np.abs(zv) + np.abs(gv)))


def _ld_graph(graph):
  return {'edges': np.asarray(graph['edges'], np.int64), 'measurements': np.asarray(graph['measurements'], LD),
          'weights': np.asarray(graph['weights'], LD)}


def _hat_abs(v):
  """|hat(v)| of magnitudes v [..., 3]"""
  return np.abs(P.hat(v))


def edge_model(graph, T, phi):
  """The long double reference and the kernel's first-order rounding bounds of every edge at the poses T [n, 4, 4]:
  a dict of chi2, s, M [E, 6, 6], q [E, 6] (long double) and dchi2, ds, dM, dq, de (float64 bounds)."""
  ed = np.asarray(graph['edges'], np.int64)
  n, E = T.shape[0], ed.shape[0]
  Ta, Tb, Z = (np.asarray(x, np.float64) for x in (T[ed[:, 0]], T[ed[:, 1]], graph['measurements']))
  w = np.asarray(graph['weights'], np.float64)
  e, A = P.jacobian(Ta.astype(LD), Tb.astype(LD), Z.astype(LD))
  wl = w.astype(LD)
  chi2 = np.sum(wl * e * e, -1)
  loop = np.arange(E) >= n - 1
  _, s = P.rho(chi2, loop, phi)
  d = s * s
  M = d[:, None, None] * np.einsum('kri,kr,krj->kij', A, wl, A)
  q = d[:, None] * np.einsum('kri,kr,kr->ki', A, wl, e)
  # magnitudes and absolute rounding bounds of the kernel's intermediates
  ZR, Zt, TaR, ta, TbR, tb = (np.abs(x) for x in (Z[:, :3, :3], Z[:, :3, 3], Ta[:, :3, :3], Ta[:, :3, 3],
                                                  Tb[:, :3, :3], Tb[:, :3, 3]))
  ZRt = np.swapaxes(ZR, 1, 2)
  mv = lambda Mx, v: np.einsum('kij,kj->ki', Mx, v)  # noqa: E731
  m_u = mv(np.swapaxes(TaR, 1, 2), ta) + Zt
  d_u = gamma(4) * m_u
  m_RC = ZRt @ np.swapaxes(TaR, 1, 2)
  d_RC = gamma(3) * m_RC
  m_tC = mv(ZRt, m_u)
  d_tC = gamma(3) * m_tC + mv(ZRt, d_u)
  m_RE = m_RC @ TbR
  d_RE = gamma(3) * m_RE + d_RC @ TbR
  m_tE = mv(m_RC, tb) + m_tC
  d_tE = gamma(4) * m_tE + mv(d_RC, tb) + d_tC
  ef = np.abs(e.astype(np.float64))
  th = np.sqrt(np.sum(ef[:, :3] ** 2, -1))
  with np.errstate(divide='ignore', invalid='ignore'):
    amp = np.where(th <= np.pi - P.PI_BRANCH + 1e-9, np.where(th > 0, th / (2 * np.sin(th)), 0.5), 1.0)
  d_rot = 9 * np.maximum(1.0, amp) * d_RE.reshape(E, 9).max(-1) + 8 * U * th
  de = np.concatenate([np.repeat(d_rot[:, None], 3, 1), d_tE], 1)
  chif = np.sum(w * ef * ef, -1)
  dchi2 = np.sum(w * (2 * ef * de + de * de), -1) + gamma(7) * chif
  sf = s.astype(np.float64)
  ds = np.where(loop & ~np.isinf(phi), sf * (dchi2 / (phi + chif) + 3 * U), 0.0) if not np.isinf(phi) else \
      np.zeros(E)
  df = sf * sf
  dd = 2 * sf * ds + U * df
  c = 1 / np.pi ** 2 + 1e-3
  mK = _hat_abs(ef[:, :3])
  mJ = np.eye(3) + 0.5 * mK + c * (mK @ mK)
  dJ = 1.5 * d_rot[:, None, None] + gamma(8) * mJ
  mS_v = m_tC + ef[:, 3:]
  dS_v = d_tC + d_tE + U * mS_v
  mA, dA = np.zeros((E, 6, 6)), np.zeros((E, 6, 6))
  mA[:, :3, :3] = mJ @ m_RC
  dA[:, :3, :3] = dJ @ m_RC + mJ @ d_RC + gamma(3) * mJ @ m_RC
  mA[:, 3:, :3] = _hat_abs(mS_v) @ m_RC
  dA[:, 3:, :3] = _hat_abs(dS_v) @ m_RC + _hat_abs(mS_v) @ d_RC + gamma(3) * mA[:, 3:, :3]
  mA[:, 3:, 3:] = m_RC
  dA[:, 3:, 3:] = d_RC
  AwA = np.einsum('kri,kr,krj->kij', mA, w, mA)
  dM = df[:, None, None] * (np.einsum('kri,kr,krj->kij', dA, w, mA) + np.einsum('kri,kr,krj->kij', mA, w, dA)) + \
      (gamma(7) * df + dd)[:, None, None] * AwA
  Awe = np.einsum('kri,kr,kr->ki', mA, w, ef)
  dq = df[:, None] * (np.einsum('kri,kr,kr->ki', dA, w, ef) + np.einsum('kri,kr,kr->ki', mA, w, de)) + \
      (gamma(7) * df + dd)[:, None] * Awe
  return {'chi2': chi2, 's': s, 'M': M, 'q': q, 'dchi2': REF * dchi2, 'ds': REF * ds, 'dM': REF * dM,
          'dq': REF * dq, 'de': REF * de, 'rho_prime': df}


def _diff(a, ref):
  return (np.asarray(a, LD) - np.asarray(ref, LD)).astype(np.float64)


def edge_gate(graph, T, phi, chi2, s, M, q, skip=None):
  """the GPU's chi2, s, M, q at T against edge_model; `skip` [E] bool: edges not gated (e.g. exactly at pi).  M must
  also be symmetric bit for bit (the kernel writes each entry to both positions)."""
  m = edge_model(graph, T, phi)
  keep = np.ones(len(chi2), bool) if skip is None else ~np.asarray(skip)
  out = {'chi2': ratio(_diff(chi2, m['chi2'])[keep], m['dchi2'][keep]),
         's': ratio(_diff(s, m['s'])[keep], m['ds'][keep]),
         'M': ratio(_diff(M, m['M'])[keep], m['dM'][keep]),
         'q': ratio(_diff(q, m['q'])[keep], m['dq'][keep]),
         'symmetric': bits_equal(M, np.swapaxes(M, 1, 2))}
  out['worst'] = max(v['worst'] for v in out.values())
  return out


def update_gate(T, x, Tt):
  """Tt = update(T, x) over nodes 1 .. n-1, node 0 unchanged"""
  ref = P.update(np.asarray(T[1:], LD), np.asarray(x[1:], LD))
  T1 = np.abs(np.asarray(T[1:], np.float64))
  bound = np.zeros_like(T1)
  bound[:, :3, :] = np.sum(np.abs(T1[:, :3, :]), 1)[:, None, :]
  bound[:, :3, 3] += np.abs(np.asarray(x[1:, 3:], np.float64))
  g = ratio(_diff(Tt[1:, :3], ref[:, :3]), gamma(28) * bound[:, :3])
  node0 = bits_equal(Tt[:1], T[:1])
  bottom = bits_equal(Tt[1:, 3], np.broadcast_to([0.0, 0.0, 0.0, 1.0], Tt[1:, 3].shape))
  return {'rows': g, 'node0': node0, 'bottom': bottom, 'worst': max(g['worst'], node0['worst'], bottom['worst'])}


def cost_gate(graph, Tt, phi, cost):
  """the trial's F at Tt against evaluate in long double"""
  F, _, _ = P.evaluate(_ld_graph(graph), np.asarray(Tt, LD), phi)
  m = edge_model(graph, np.asarray(Tt, np.float64), phi)
  E = len(graph['edges'])
  bound = 0.5 * np.sum(m['rho_prime'] * m['dchi2']) + gamma(E) * float(F)
  return ratio(_diff(cost, F), bound)


def lm_gate(trace, lambda_min):
  """the lambda schedule of a trace, bit-exact: lam_{k+1} = max(lam_k / 10, lambda_min) after an accepted trial,
  10 lam_k after a rejected one (each decision is gated against its own F by the restarted trials)"""
  lam, acc = trace['lambda'], trace['accepted']
  return all((max(lam[k] / 10.0, lambda_min) if acc[k] else lam[k] * 10.0) == lam[k + 1] for k in range(len(lam) - 1))
