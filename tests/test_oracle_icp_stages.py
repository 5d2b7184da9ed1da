"""The ICP stage gates (oracle/icp_stages.py) on the CPU: a NumPy restatement of k_icp_pairs passes every gate, each
planted defect exceeds its gate, and the bin classifier (oracle/gt.bin_candidates) calls bin edges ambiguous and
everything else certain."""
import numpy as np
import pytest

from icp_cases import kitti_pair, pixel_centre_image
from oracle import gt as G
from oracle import icp
from oracle import icp_stages as I
from oracle import projection as P
from overlapnet_b200 import gt
from overlapnet_b200.registration import seed_pose

GEOM = icp.geometry()


def images(points):
  r, v, _, _ = P.range_projection(np.asarray(points, np.float32))
  return v.astype(np.float32), P.gen_normal_map(r, v).astype(np.float32)


@pytest.fixture(scope='module')
def kitti30():
  L, R, T = kitti_pair(30.0, (1.5, -1.0, 0.1))
  vt, nt = images(L)
  vs, ns = images(R)
  return vs, ns, vt, nt, seed_pose(gt.yaw_bin(np.eye(4), T, 360), 360)


def _run(case, k, prm=None, mutant=None):
  vs, ns, vt, nt, T = case
  prm = dict(icp.DEFAULTS, **(prm or {}))
  st = I.restate_iteration(T, k, prm, GEOM, vs, ns, vt, nt, mutant)
  return I.check_iteration(T, k, prm, GEOM, vs, ns, vt, nt, st), st


def _passes(rep):
  return (rep['unexplained'] == 0 and rep['sums'] <= 1 and rep['pose'] <= 1 and rep['decision'] == 0
          and rep['fields'] == 0)


# ---- the restatement passes --------------------------------------------------------------------------------------
def test_restatement_passes_every_gate(kitti30):
  vs, ns, vt, nt, T = kitti30
  prm = dict(icp.DEFAULTS)
  worst = {}
  for k in range(4):
    rep, st = _run((vs, ns, vt, nt, T), k)
    assert _passes(rep), (k, rep)
    for key in ('sums', 'pose', 'ambiguous'):
      worst[key] = max(worst.get(key, 0), rep[key])
    T = st['pose']
  print('restatement: sums <= %.3f, pose <= %.3g of their bounds, %d ambiguous pixels'
        % (worst['sums'], worst['pose'], worst['ambiguous']))
  assert worst['sums'] > 0                     # the restatement's sums do round


def test_sums_gate_weights():
  # thread 0 has pixels 0, 384, 768: its first term 3 roundings (product + 2 adds), the second 3, the third 2;
  # warp 0 then adds 5 + 11, warp 11 (pixel 383) 5 + 1
  w = I.weights(np.array([0, 384, 768, 383]), 1000)
  assert w.tolist() == [3 + 16, 3 + 16, 2 + 16, 1 + 6]


# ---- mutants exceed their gates -----------------------------------------------------------------------------------
@pytest.mark.parametrize('mutant', ['cos_unrotated', 'atan2_plus', 'schedule_advanced'])
def test_association_mutants_exceed_the_gate(kitti30, mutant):
  rep, _ = _run(kitti30, 0, mutant=mutant)
  print(mutant, rep)
  assert rep['unexplained'] > 0


@pytest.mark.parametrize('mutant', ['sums_float32', 'chain_drop_last', 'cross_reversed'])
def test_sums_mutants_exceed_the_gate(kitti30, mutant):
  rep, _ = _run(kitti30, 0, mutant=mutant)
  print(mutant, rep)
  assert rep['sums'] > 1


def test_pivot_without_the_trace_factor_exceeds_the_gate():
  # H = diag(1e5, 1, 1, 1, 1, 1e-9): the last pivot is below 1e-12 tr (~1e-7) but above 1e-12
  S = np.zeros(29)
  r, c = np.triu_indices(6)
  diag = [1e5, 1.0, 1.0, 1.0, 1.0, 1e-9]
  for k, (i, j) in enumerate(zip(r, c)):
    if i == j:
      S[k] = diag[i]
  S[21:27] = 1e-3
  S[27] = 1000
  prm = dict(icp.DEFAULTS)
  m = I.model_step(S, 0.3, prm)
  assert m['status'] == icp.DEGENERATE and not m['tie']
  mutated = I.model_step(S, 0.3, prm, 'pivot_no_trace')['status']
  assert I.decision_gate(m, icp.MAX_ITERATIONS if mutated is None else mutated)[0] == 1
  assert I.decision_gate(m, icp.DEGENERATE) == (0, 0)


def test_early_convergence_exceeds_the_gate():
  # the exact known answer: every pixel associates to itself, g = 0, d = 0; at d_k = d_start > d_end the kernel goes on
  v, n = pixel_centre_image(GEOM)
  case = (v, n, v, n, np.eye(4))
  rep, st = _run(case, 0)
  assert _passes(rep) and st['status'] == icp.MAX_ITERATIONS and st['inliers'] == GEOM['H'] * GEOM['W']
  rep, st = _run(case, 0, mutant='converge_early')
  assert st['status'] == icp.CONVERGED and rep['decision'] == 1


def test_known_answer_converges_at_once_with_the_identity():
  v, n = pixel_centre_image(GEOM)
  rep, st = _run((v, n, v, n, np.eye(4)), 0, dict(d_start=0.3, d_end=0.3))
  assert _passes(rep) and rep['ambiguous'] == 0
  assert st['status'] == icp.CONVERGED and np.array_equal(st['pose'], np.eye(4))
  assert np.all(st['system'][21:27] == 0) and st['system'][28] == 0


def test_rank_five_planes_are_degenerate():
  v, n = pixel_centre_image(GEOM, nz=False)
  rep, st = _run((v, n, v, n, np.eye(4)), 0)
  assert _passes(rep) and st['status'] == icp.DEGENERATE and not rep['tie']


# ---- the bin classifier ---------------------------------------------------------------------------------------------
def _edge_points(g, yaws, pitches, depth=10.0):
  yaws, pitches = np.asarray(yaws, np.float64), np.asarray(pitches, np.float64)
  return (depth * np.cos(pitches) * np.cos(-yaws), depth * np.cos(pitches) * np.sin(-yaws), depth * np.sin(pitches))


def _yaw_edge(k, W):
  return np.pi * (2.0 * k / W - 1.0)


def _exact_edges(bin_of, approx, width=1e-9):
  """per approximate edge, the least float64 angle whose bin (``bin_of``) differs from the bin width below it:
  bisection over the ordered bit patterns of positive and negative doubles alike"""
  key = lambda a: np.where(a >= 0, a.view(np.int64), -(np.abs(a).view(np.int64)))
  unkey = lambda k: np.where(k >= 0, k, -k).view(np.float64) * np.where(k >= 0, 1.0, -1.0)
  lo, hi = key(approx - width), key(approx + width)
  base = bin_of(approx - width)
  while np.any(hi - lo > 1):
    mid = lo + (hi - lo) // 2
    same = bin_of(unkey(mid)) == base
    lo = np.where(same, mid, lo)
    hi = np.where(same, hi, mid)
  return unkey(hi)


@pytest.mark.parametrize('geometry', [icp.geometry(), icp.geometry(32, 2048, 15.0, -15.0),
                                      icp.geometry(128, 1024, 2.0, -24.9)])
def test_classifier_edges_are_ambiguous_and_the_rest_certain(geometry):
  g = geometry
  W, H = g['W'], g['H']
  ks = np.array([1, 2, W // 3, W - W // 3, W - 2, W - 1])
  down = abs(g['fov_down'] / 180.0 * np.pi)
  fov = down + abs(g['fov_up'] / 180.0 * np.pi)
  rows = np.arange(1, H)
  ye = _exact_edges(lambda a: G.angle_bins(a, np.zeros_like(a), g)[0], _yaw_edge(ks, W))
  pe = _exact_edges(lambda a: -G.angle_bins(np.zeros_like(a), a, g)[1], (1.0 - rows / H) * fov - down)
  for step in (-np.inf, None, np.inf):                        # the edge's angle and its neighbours by nextafter
    y = ye if step is None else np.nextafter(ye, step)
    p = pe if step is None else np.nextafter(pe, step)
    c = G.angle_candidates(y, np.full(y.size, 0.01), g)
    assert np.all(c['amb_x']) and np.all(np.abs(c['alt_x'] - c['bx']) == 1) and not np.any(c['amb_y'])
    assert np.all(np.minimum(c['bx'], c['alt_x']) == ks - 1) and np.all(c['bx'] == (ks if step != -np.inf else ks - 1))
    c = G.angle_candidates(np.full(p.size, 0.3), p, g)
    assert np.all(c['amb_y']) and np.all(np.abs(c['alt_y'] - c['by']) == 1) and not np.any(c['amb_x'])
    assert np.all(np.minimum(c['by'], c['alt_y']) == rows - 1)
    assert np.all(c['by'] == (rows - 1 if step != -np.inf else rows))
  for d in (1e-9, -1e-9):                                    # 1e-9 rad away: certain
    c = G.angle_candidates(ye + d, np.full(ks.size, 0.01), g)
    assert not np.any(c['amb_x']) and np.array_equal(c['bx'], ks if d > 0 else ks - 1)
    c = G.angle_candidates(np.full(rows.size, 0.3), pe + d, g)
    assert not np.any(c['amb_y'])
  # next to yaw 0 the + 1.0 of the bin rounds away far more than 3 ulp of the angle: certain even on the edge
  c = G.angle_candidates(_yaw_edge(np.array([W // 2 + 1]), W), np.array([0.01]), g)
  assert not c['amb_x'][0]
  # and through the points: a point on an edge's ray is ambiguous where its float64 angle is that close
  x, y, z = _edge_points(g, ye, np.full(ks.size, 0.01))
  c = G.bin_candidates(x, y, z, g)
  _, _, yaw, _ = G.range_angles(x, y, z, g)
  near = np.abs(yaw - ye) <= np.spacing(np.abs(ye))
  assert np.count_nonzero(near) >= 3 and np.all(c['amb_x'][near])


def test_classifier_at_the_azimuth_seam():
  g = GEOM
  W = g['W']
  # the edges next to the seam: a one-bin shift between bins 0 and 1, and W - 2 and W - 1
  for k, lo in ((1, 0), (W - 1, W - 2)):
    c = G.angle_candidates(np.array([_yaw_edge(k, W)]), np.array([0.0]), g)
    assert c['amb_x'][0] and {int(c['bx'][0]), int(c['alt_x'][0])} == {lo, lo + 1}
  # on the seam itself the sign of y decides, exactly: +0 -> yaw -pi -> bin 0, -0 -> yaw +pi -> bin W - 1
  c = G.bin_candidates(np.array([-10.0, -10.0, -10.0]), np.array([0.0, -0.0, -1e-300]), np.zeros(3), g)
  assert c['bx'].tolist() == [0, W - 1, W - 1] and not np.any(c['amb_x'])


def test_classifier_matches_the_model_bins():
  rng = np.random.default_rng(1)
  x, y, z = rng.normal(size=(3, 100000)) * 20
  c = G.bin_candidates(x, y, z, GEOM)
  keep, bx, by = icp.bins_f64(x, y, z, GEOM)
  assert np.array_equal(keep, c['keep']) and np.array_equal(bx[keep], c['bx'][keep])
  amb = c['amb_x'] | c['amb_y']
  print('random points: %d of %d ambiguous' % (np.count_nonzero(amb), amb.size))
  assert np.count_nonzero(amb) < 20


def test_explain_range_image_accepts_only_explained_pixels():
  g = G.geometry(64, 900, 3.0, -25.0, 50.0, f32=False)
  W = g['W']
  ks = np.arange(1, W, 7)
  x, y, z = _edge_points(g, _yaw_edge(ks, W), np.full(ks.size, 0.01))
  vertex = np.stack([x, y, z, np.ones_like(x)], 1)
  img = G.range_image_f64(vertex)
  bad, amb, uncertain = G.explain_range_image(vertex, img, g)
  assert bad == 0 and amb > 0 and np.count_nonzero(uncertain) >= amb
  # the other candidate of an ambiguous point is also explained; a wrong depth or a lost point is not
  c = G.bin_candidates(x, y, z, g)
  i = int(np.flatnonzero(c['amb_x'])[0])
  moved = img.copy().reshape(-1)
  moved[c['by'][i] * W + c['alt_x'][i]] = moved[c['by'][i] * W + c['bx'][i]]
  moved[c['by'][i] * W + c['bx'][i]] = -1
  assert G.explain_range_image(vertex, moved.reshape(img.shape), g)[0] == 0
  wrong = img.copy()
  wrong[img > 0] = np.nextafter(wrong[img > 0], np.float32(np.inf))
  assert G.explain_range_image(vertex, wrong, g)[0] == np.count_nonzero(img > 0)
  far = vertex.copy()
  far[:, :3] *= 2.0                                            # still in range, every point now certain
  certain = G.bin_candidates(far[:, 0], far[:, 1], far[:, 2], g)
  lost = G.range_image_f64(far).reshape(-1)
  j = int(np.flatnonzero(~(certain['amb_x'] | certain['amb_y']))[0])
  lost[certain['by'][j] * W + certain['bx'][j]] = -1
  assert G.explain_range_image(far, lost.reshape(img.shape), g)[0] >= 1
