"""Every image and head geometry the handle accepts, on the GPU, against the oracles (tests/test_geometry.py
pins the oracles themselves at these geometries):

A. projection, normals, semantic gather and the fused preprocess bit-exact at other image sizes and fovs, and
   the points whose bin the projection's fast path decides closest to its margin;
B. the fp32 leg and heads at other (leg_output_width, conv1size), and the yaw known answer at those widths;
C. head-only and whole-network training gradients at other head geometries;
D. the tensor-core and fp32 legs at other layer-1 strides."""
import functools
import math

import numpy as np
import pytest
import torch

import train_leg_oracle as TL
import train_oracle as T
from oracle import network as N
from oracle import projection as P
from overlapnet_b200 import synth
from overlapnet_b200._cabi import OvnError
from overlapnet_b200.engine import HEAD_LAYERS, Engine
from test_geometry import HEAD_GEOMETRIES, MODEL, head_model, image_size
from test_gpu_network import check_yaw

pytestmark = pytest.mark.gpu


def bits(a):
  a = np.ascontiguousarray(a)
  return a.view(np.uint32) if a.dtype == np.float32 else a


def _idx(a, dev):
  return torch.from_numpy(np.ascontiguousarray(a, np.int32)).to(dev)


# ---- A. projection -----------------------------------------------------------------------------------------
# (H, W, fov_up, fov_down): a partial last tile row (60 rows, tiles are 8 x 32), both tails, an image narrower
# than the gather tile's 33-pixel halo, a wide image at a symmetric fov, a tall image at a narrow fov, control
PROJ_GEOMETRIES = [(60, 900, 3.0, -25.0), (37, 457, 3.0, -25.0), (16, 20, 3.0, -25.0), (32, 2048, 15.0, -15.0),
                   (128, 1024, 2.0, -24.9), (64, 900, 3.0, -25.0)]


@functools.lru_cache(maxsize=None)
def _clouds():
  """The seeded clouds of test_gpu_projection.py::test_oracle_parity_synthetic_batch, the empty and the
  1-point cloud included, and per-point class probabilities."""
  clouds = [synth.kitti_like_cloud(20 + s, n_points=n, zero_points=z)
            for s, (n, z) in enumerate([(124668, 0), (60000, 11), (33, 1), (5000, 0)])]
  clouds.insert(2, np.zeros((0, 4), np.float32))
  clouds.append(np.array([[2.0, 1.0, -0.2, 0.7]], np.float32))
  probs = [synth.random_probs(300 + i, c.shape[0]) for i, c in enumerate(clouds)]
  return clouds, probs


def _proj_engine(H, W, fu, fd, use=None):
  return Engine(use=use, model=MODEL, precision='fp32', max_batch_scans=8, max_batch_pairs=1, proj_H=H, proj_W=W,
                fov_up=fu, fov_down=fd)


@pytest.mark.parametrize('H,W,fu,fd', PROJ_GEOMETRIES)
def test_projection_matches_oracle_at_geometry(H, W, fu, fd):
  clouds, probs = _clouds()
  eng = _proj_engine(H, W, fu, fd)
  dev = eng.device
  batch = eng.upload_clouds(clouds)
  out = eng.project(batch)
  nrm = eng.normals(out['range'], out['vertex']).cpu().numpy()
  out = {k: v.cpu().numpy() for k, v in out.items()}
  idx_inf = eng.project(batch, max_range=float('inf'), want=('idx',))['idx']
  prob_all = torch.from_numpy(np.concatenate(probs)).to(dev)
  sem = eng.semantic(idx_inf, prob_all, batch.offsets).cpu().numpy()
  idx_inf = idx_inf.cpu().numpy()
  x4 = eng.preprocess(batch).cpu().numpy()
  eng.close()
  eng25 = _proj_engine(H, W, fu, fd, use={'use_intensity': True, 'use_class_probabilities': True})
  assert eng25.C == 25
  x25 = eng25.preprocess(eng25.upload_clouds(clouds), prob_all.to(eng25.device)).cpu().numpy()
  eng25.close()
  for i, c in enumerate(clouds):
    rng, vert, inten, idx = P.range_projection(c, fu, fd, H, W)
    assert np.array_equal(bits(out['range'][i]), bits(rng)), i
    assert np.array_equal(bits(out['vertex'][i]), bits(vert)), i
    assert np.array_equal(bits(out['intensity'][i]), bits(inten)), i
    assert np.array_equal(out['idx'][i], idx), i
    normal = P.gen_normal_map(rng, vert, H, W)
    assert np.array_equal(bits(nrm[i]), bits(normal)), i
    assert np.array_equal(idx_inf[i], P.range_projection(c, fu, fd, H, W, max_range=np.inf)[3]), i
    assert np.array_equal(bits(sem[i]), bits(P.gen_semantic_image(c, probs[i], H, W, fu, fd))), i
    assert np.array_equal(bits(x4[i]), bits(P.pack_input(rng, normal))), i
    # the fused path gathers the probabilities with the configured max_range's index (projection.cu)
    prob_img = np.full((H, W, 20), -1, np.float32)
    prob_img[idx >= 0] = probs[i][idx[idx >= 0]]
    assert np.array_equal(bits(x25[i]), bits(P.pack_input(rng, normal, prob_img, inten))), i
  assert (out['idx'][0] >= 0).sum() > 0.1 * H * W          # the big cloud covers the image


def fast_path_margins(H, W, fov_up, fov_down):
  """The margins of projection.cu's make_params: twice the worst-case distance between the fast estimate and
  the exact pre-floor value, never below 1e-3 (x) / 1e-4 (y).  Mirrors bound_x / bound_y (DESIGN.md section 4)."""
  ulp32 = lambda a: 2.0 ** (math.frexp(a)[1] - 24)
  pi, e24 = math.pi, 2.0 ** -24
  fu = float(np.float32(fov_up)) / 180.0 * pi
  fd = float(np.float32(fov_down)) / 180.0 * pi
  bx = W / (2 * pi) * 3.5 * ulp32(pi) + 0.5 * W * 3.5 * e24 + ulp32(W)
  fov = abs(fd) + abs(fu)
  pmax = max(abs(fu), abs(fd)) * (1 + 1e-6)
  by = (H / fov * (2.5 * ulp32(pmax) + pmax * e24 + 0.5 * ulp32(abs(fd)) + 0.5 * ulp32(pmax + abs(fd)))
        + H * 4 * e24 + ulp32(H))
  return float(np.float32(max(1e-3, 2 * bx))), float(np.float32(max(1e-4, 2 * by)))


def _point(tau_y, tau_x, H, W, fu, fd, rho=10.0):
  """float32 points whose pre-floor bins are close to (tau_y, tau_x), by inverting utils.py:90-95 in float64."""
  fu_r, fd_r = fu / 180.0 * np.pi, fd / 180.0 * np.pi
  fov = abs(fu_r) + abs(fd_r)
  pitch = (1.0 - np.asarray(tau_y) / H) * fov - abs(fd_r)
  yaw = (2.0 * np.asarray(tau_x) / W - 1.0) * np.pi
  pts = np.empty((np.size(tau_x), 4), np.float32)
  pts[:, 0] = rho * np.cos(pitch) * np.cos(yaw)
  pts[:, 1] = -rho * np.cos(pitch) * np.sin(yaw)
  pts[:, 2] = rho * np.sin(pitch)
  pts[:, 3] = 0.5
  return pts


def _band_cloud(axis, H, W, fu, fd, m):
  """Points whose exact float32 pre-floor value along ``axis`` lies between 1x and 3x the margin m from a bin
  edge, on both sides, each in a pixel of its own; the other coordinate sits mid-bin."""
  n_other, n_edge = (H, W) if axis == 'x' else (W, H)
  edges = np.arange(2, n_edge - 1, 2)                          # bins k-1 and k of edge k are no other edge's
  lanes = [(j + 1) * n_other // 5 for j in range(4)]           # 4 rows (x band) or columns (y band)
  deltas = np.array([1.25, 1.75, 2.25, 2.75]) * m
  tau_e, tau_o = [], []
  for lane, d in zip(lanes, deltas):
    for sign in (1.0, -1.0):
      tau_e.append(edges + sign * d)
      tau_o.append(np.full(edges.shape, lane + 0.5))
  tau_e, tau_o = np.concatenate(tau_e), np.concatenate(tau_o)
  pts = _point(tau_o, tau_e, H, W, fu, fd) if axis == 'x' else _point(tau_e, tau_o, H, W, fu, fd)
  _, ty, tx = P.projection_prefloor(pts, fu, fd, H, W)
  t, o = (tx, ty) if axis == 'x' else (ty, tx)
  t, o = t.astype(np.float64), o.astype(np.float64)
  k = np.rint(t)
  dist = np.abs(t - k)
  keep = (dist >= m) & (dist <= 3 * m) & (np.abs(k - np.rint(tau_e)) == 0) & (np.floor(o) == np.floor(tau_o))
  assert keep.mean() > 0.9, keep.mean()
  return pts[keep]


# the default geometry, a wide image and the largest one tested (1024 x 16384: margins 0.011 / 1.4e-3)
@pytest.mark.parametrize('H,W,fu,fd', [(64, 900, 3.0, -25.0), (128, 4096, 2.0, -24.9), (1024, 16384, 2.0, -24.9)])
def test_projection_bins_next_to_the_fast_path_margin(H, W, fu, fd):
  """Only points within a few margins of a bin edge are decided by the fast estimate with little to spare; a
  margin smaller than the estimate's error puts them in the wrong bin.  Both sides of every other edge."""
  mx, my = fast_path_margins(H, W, fu, fd)
  if (H, W) == (64, 900):
    assert (mx, my) == (float(np.float32(1e-3)), float(np.float32(1e-4)))
  clouds = [_band_cloud('x', H, W, fu, fd, mx), _band_cloud('y', H, W, fu, fd, my)]
  eng = Engine(model=MODEL, precision='fp32', max_batch_scans=2, max_batch_pairs=1, proj_H=H, proj_W=W,
               fov_up=fu, fov_down=fd)
  out = eng.project(eng.upload_clouds(clouds), want=('range', 'idx'))
  out = {k: v.cpu().numpy() for k, v in out.items()}
  eng.close()
  for i, c in enumerate(clouds):
    rng, _, _, idx = P.range_projection(c, fu, fd, H, W)
    assert (idx >= 0).sum() == c.shape[0]                     # one point per pixel: none hides another
    bad = np.argwhere(out['idx'][i] != idx)
    assert bad.size == 0, ('xy'[i], bad[:10].tolist(), len(bad))
    assert np.array_equal(bits(out['range'][i]), bits(rng))


# ---- B. fp32 network at other head geometries ----------------------------------------------------------------
@pytest.mark.parametrize('wf,s', HEAD_GEOMETRIES)
def test_fp32_network_matches_oracle_at_head_geometry(wf, s):
  model = head_model(wf, s)
  H, W = image_size(model, wf)
  w = N.glorot_weights(4, model, seed=0, leg_out_width=wf)
  x = synth.range_like_images(1000 + wf + s, 3, 4, H=H, W=W)
  fv_ref = N.leg_forward(x, w, model)[:, 0]
  eng = Engine(model=model, precision='fp32', max_batch_scans=2, max_batch_pairs=4, proj_H=H, proj_W=W)
  assert eng.Wf == wf
  eng.load_weights(w)
  fv = eng.leg(torch.from_numpy(x).to(eng.device)).cpu().numpy()          # 3 scans > max_batch_scans = 2
  err = np.abs(fv - fv_ref).max() / np.abs(fv_ref).max()
  print('\n[geometry] fp32 leg Wf=%d: max rel err %.2e' % (wf, err))
  assert err <= 2e-5, err
  rng = np.random.default_rng(wf + s)
  bank_np = np.stack([fv_ref[0], fv_ref[1], fv_ref[2],
                      np.roll(fv_ref[2], 37, axis=0) + np.abs(rng.normal(0, 0.01, fv_ref[2].shape)).astype(np.float32),
                      np.roll(fv_ref[0], -100, axis=0), fv_ref[1] * np.float32(0.5) + fv_ref[0] * np.float32(0.5)])
  left = np.array([0, 1, 2, 3, 4, 5, 5, 3], np.int32)                      # 8 pairs > max_batch_pairs = 4
  right = np.array([5, 5, 5, 5, 5, 5, 0, 2], np.int32)
  _, _, _, z0 = N.heads_forward(bank_np[left][:, None], bank_np[right][:, None], w, model, batch=2, return_logit=True)
  w = N.spread_dense(w, z0, target_std=1.5)
  eng.load_weights(w)
  ov_ref, yaw_ref, corr_ref = N.heads_forward(bank_np[left][:, None], bank_np[right][:, None], w, model, batch=2)
  bank = torch.from_numpy(bank_np).to(eng.device)
  ov, yaw, corr = eng.heads(bank, torch.from_numpy(left), torch.from_numpy(right), want_corr=True)
  ov, yaw, corr = ov.cpu().numpy(), yaw.cpu().numpy(), corr.cpu().numpy()
  print('[geometry] heads Wf=%d s=%d: max |overlap - oracle| %.2e (overlaps %.2f..%.2f)'
        % (wf, s, np.abs(ov - ov_ref).max(), ov_ref.min(), ov_ref.max()))
  assert np.abs(ov - ov_ref).max() <= 1e-3
  assert ov_ref.max() - ov_ref.min() > 0.25
  assert corr.shape == (8, wf)
  assert np.abs(corr - corr_ref).max() / np.abs(corr_ref).max() <= 1e-5
  check_yaw(yaw, yaw_ref, corr_ref)
  # pair 7: LEFT = roll(RIGHT, 37) + noise, i.e. RIGHT = roll(LEFT, -37): argmax = (37 - Wf//2) mod Wf
  assert yaw_ref[7] == 180 - (37 - wf // 2) % wf and yaw[7] == yaw_ref[7]
  ov1, yaw1, _ = eng.heads_1vsN(bank, bank[5], cand_idx=torch.arange(6, dtype=torch.int32))
  assert np.array_equal(ov1.cpu().numpy(), ov[:6]) and np.array_equal(yaw1.cpu().numpy(), yaw[:6])
  ov2, yaw2, _ = eng.heads_1vsN(bank, bank[5], n_cand=4)
  assert np.array_equal(ov2.cpu().numpy(), ov[:4]) and np.array_equal(yaw2.cpu().numpy(), yaw[:4])
  eng.check()
  eng.close()


@pytest.mark.parametrize('wf,s', [(225, 15), (405, 27)])
def test_yaw_shift_known_answer_at_other_widths(wf, s):
  """R = roll(L, shift) for every shift of the width: the yaw is the reference's 180 - argmax, with
  argmax = (-shift - Wf//2) mod Wf (infer.py:158 subtracts from 180 whatever the width)."""
  model = head_model(wf, s)
  H, W = image_size(model, wf)
  eng = Engine(model=model, precision='fp32', max_batch_scans=1, max_batch_pairs=wf, proj_H=H, proj_W=W)
  eng.load_weights(N.glorot_weights(4, model, seed=1, leg_out_width=wf))
  base = synth.feature_volumes(3, 1, width=wf)[0, 0]
  shifts = np.arange(-(wf // 2), wf - wf // 2)
  rolled = np.stack([np.roll(base, k, axis=0) for k in shifts])
  corr_ref = N.correlation_head(np.repeat(base[None, None], len(shifts), 0), rolled[:, None])
  _, want = N.readout(np.zeros(len(shifts)), corr_ref)
  assert want.tolist() == (180 - (-shifts - wf // 2) % wf).tolist()
  bank = torch.from_numpy(np.concatenate([base[None], rolled])).to(eng.device)
  left = torch.zeros(len(shifts), dtype=torch.int32)
  right = torch.arange(1, len(shifts) + 1, dtype=torch.int32)
  _, yaw, _ = eng.heads(bank, left, right)
  eng.close()
  got = yaw.cpu().numpy()
  assert np.array_equal(got, want), (got[:5].tolist(), want[:5].tolist())


# ---- C. training at other head geometries --------------------------------------------------------------------
TRAIN_GEOMETRIES = [(225, 15), (360, 12)]
N_PAIRS = 4


def _relu_margin(pre):
  """Smallest |pre-activation| relative to the layer's largest."""
  a = np.abs(np.asarray(pre, np.float64))
  return float(a.min() / a.max())


def _head_relu_margins(l, r, w, model):
  """The oracle's c_conv2 / c_conv3 pre-activations (float64) of the pairs (l, r) of (n, Wf, 128) volumes."""
  x = N.delta_layer(torch.as_tensor(l, dtype=torch.float64)[:, None],
                    torch.as_tensor(r, dtype=torch.float64)[:, None]).permute(0, 3, 1, 2)
  out = {}
  for name, _, stride, _, act in N.head_layers(model):
    k, b = w[name]
    x = N._conv(x, k, b, stride, False, torch.float64)
    if act == 'relu':
      out[name] = _relu_margin(x)
      x = torch.relu(x)
  return out


def _leg_relu_margins(x_nhwc, w, model):
  x = torch.as_tensor(x_nhwc, dtype=torch.float64).permute(0, 3, 1, 2)
  out = {}
  for name, _, stride, _ in N.leg_layers(model):
    k, b = w[name]
    x = N._conv(x, k, b, stride, False, torch.float64)
    out[name] = _relu_margin(x)
    x = torch.relu(x)
  return out


@functools.lru_cache(maxsize=None)
def _train_setup(wf, s):
  """Images, the fp32 leg's volumes, Glorot weights with the Dense layer rescaled to a logit spread of 1.5,
  targets above every prediction and orientations over [0, Wf)."""
  model = head_model(wf, s)
  H, W = image_size(model, wf)
  w = N.glorot_weights(4, model, seed=0, leg_out_width=wf)
  x = synth.range_like_images(77, 6, 4, H=H, W=W)
  eng = Engine(model=model, precision='fp32', max_batch_scans=6, max_batch_pairs=4, proj_H=H, proj_W=W)
  eng.load_weights(w)
  fv = eng.leg(torch.from_numpy(x).to(eng.device)).cpu().numpy()
  eng.close()
  # The pairs are the first N_PAIRS of a fixed order whose head ReLU inputs (c_conv2 / c_conv3) all lie further
  # than 1e-6 of the layer's largest from 0; the head gradients are compared element by element, and a mask
  # that fp32 and float64 decide differently would fail them for a reason of its own
  left, right = [], []
  for i, j in ((i, j) for d in range(1, 6) for i in range(6) for j in [(i + d) % 6]):
    if min(_head_relu_margins(fv[[i]], fv[[j]], w, model).values()) > 1e-6:
      left.append(i); right.append(j)
    if len(left) == N_PAIRS:
      break
  assert len(left) == N_PAIRS, (left, right)
  left, right = np.array(left, np.int32), np.array(right, np.int32)
  _, _, _, z = N.heads_forward(fv[left][:, None], fv[right][:, None], w, model, return_logit=True)
  w = N.spread_dense(w, z, target_std=1.5)
  ov_ref, _, _ = N.heads_forward(fv[left][:, None], fv[right][:, None], w, model)
  rng = np.random.default_rng(5)
  gt_ov = (ov_ref + rng.uniform(0.15, 0.35, N_PAIRS)).astype(np.float32)
  gt_or = rng.integers(0, wf, N_PAIRS).astype(np.int32)
  return model, w, x, fv, left, right, gt_ov, gt_or


def _train_engine(wf, s, w, maxp=4):
  model = head_model(wf, s)
  H, W = image_size(model, wf)
  eng = Engine(model=model, precision='fp32', max_batch_scans=6, max_batch_pairs=maxp, proj_H=H, proj_W=W)
  eng.load_weights(w)
  return eng


def _compare(got, ref, names, tol):
  for name in names:
    for i, part in enumerate(('kernel', 'bias')):
      g, r = got[name][i], ref[name][i]
      assert g.shape == r.shape
      err = float(np.abs(g - r).max()) / float(np.abs(r).max())
      print('%s %s: max|g - g_ref| / max|g_ref| = %.2e' % (name, part, err))
      assert np.abs(r).max() > 0 and err <= tol(name), (name, part, err)


@pytest.mark.parametrize('wf,s', TRAIN_GEOMETRIES)
@pytest.mark.parametrize('n', [1, 4])
def test_head_gradients_match_oracle_at_head_geometry(wf, s, n):
  model, w, x, fv, left, right, gt_ov, gt_or = _train_setup(wf, s)
  l, r = left[:n], right[:n]
  margins = _head_relu_margins(fv[l], fv[r], w, model)
  print('head ReLU margins', margins)
  assert min(margins.values()) > 1e-6, margins
  eng = _train_engine(wf, s, w)
  bank = torch.from_numpy(fv).to(eng.device)
  loss = eng.head_gradients(bank, _idx(l, eng.device), _idx(r, eng.device), gt_ov[:n], gt_or[:n], 0.7)
  grads = eng.get_gradients()
  eng.close()
  ref_loss, ref = T.losses_and_gradients(fv[l], fv[r], w, gt_ov[:n], gt_or[:n], 0.7, model)
  print('losses gpu %s oracle %s' % (loss, ref_loss))
  for got, exp in zip(loss, ref_loss):
    assert abs(got - exp) <= 1e-5 * abs(exp), (loss, ref_loss)
  _compare(grads, ref, HEAD_LAYERS, lambda name: 1e-4)


@pytest.mark.parametrize('wf,s', TRAIN_GEOMETRIES)
@pytest.mark.parametrize('n', [1, 4])
def test_net_gradients_match_oracle_at_head_geometry(wf, s, n):
  model, w, x, fv, left, right, gt_ov, gt_or = _train_setup(wf, s)
  l, r = left[:n], right[:n]
  head = _head_relu_margins(fv[l], fv[r], w, model)
  assert min(head.values()) > 1e-6, head
  # A leg layer has 1e5 - 1e6 pre-activations per image, so its smallest |pre-activation| is commonly 1e-8 - 1e-6
  # of its largest.  A leg mask flip changes one term of a weight-gradient sum over every pixel; the 1e-3 bound
  # of the leg layers absorbs it (test_gpu_train_leg.py measured 5e-5 with s_conv3a), and an exact tie would not.
  leg = _leg_relu_margins(x[np.unique(np.concatenate([l, r]))], w, model)
  print('ReLU margins', head, leg)
  assert min(leg.values()) > 1e-9, leg
  eng = _train_engine(wf, s, w)
  dev = eng.device
  loss, dfv = eng.net_gradients(torch.from_numpy(x).to(dev), _idx(l, dev), _idx(r, dev), gt_ov[:n], gt_or[:n], 0.7,
                                fv_grad=True)
  grads = eng.get_gradients(eng.layers)
  eng.close()
  ref_loss, ref, ref_dfv = TL.losses_and_gradients(x[l], x[r], w, gt_ov[:n], gt_or[:n], 0.7, model,
                                                   fv=np.concatenate([fv[l], fv[r]]))
  print('losses gpu %s oracle %s' % (loss, ref_loss))
  for got, exp in zip(loss, ref_loss):
    assert abs(got - exp) <= 1e-5 * abs(exp), (loss, ref_loss)
  dfv = dfv.cpu().numpy()
  assert dfv.shape == ref_dfv.shape == (2, n, wf, 128)
  err = float(np.abs(dfv - ref_dfv).max()) / float(np.abs(ref_dfv).max())
  print('dL/d(volumes): %.2e' % err)
  assert err <= 1e-4
  assert sorted(grads) == sorted(ref)
  _compare(grads, ref, TL.layer_names(model), lambda name: 1e-4 if name in HEAD_LAYERS else 1e-3)


def test_net_gradients_pair_limit_at_width_225():
  """One call launches np * Wf * (Wf / s) rows of c_conv1, 64 per CTA, on grid.y (<= 65 535), and np * (Wf / s)
  CTAs of k_delta_dgrad on grid.z: at (225, 15) that is min(65535 * 64 // 3375, 65535 // 15) = 1242 pairs."""
  wf, s = 225, 15
  limit = min(65535 * 64 // (wf * (wf // s)), 65535 // (wf // s))
  assert limit == 1242
  model, w, x, fv, left, right, gt_ov, gt_or = _train_setup(wf, s)
  eng = _train_engine(wf, s, w, maxp=limit + 1)
  dev = eng.device
  big = np.arange(limit + 1, dtype=np.int32) % 6
  with pytest.raises(OvnError, match='OVN_ERR_CAPACITY.*%d pairs' % limit):
    eng.net_gradients(torch.from_numpy(x).to(dev), _idx(big, dev), _idx(big[::-1].copy(), dev),
                      np.full(limit + 1, 0.5, np.float32), np.zeros(limit + 1, np.int32), 0.7)
  eng.close()


# ---- D. legs at other layer-1 strides ------------------------------------------------------------------------
@pytest.mark.parametrize('strides', [[1, 1], [1, 2], [2, 1]])
def test_legs_match_oracle_at_layer1_strides(strides):
  model = dict(MODEL, strides_layer1=strides)
  H, W = image_size(model, 360)
  w = N.glorot_weights(4, model, seed=6)
  x = synth.range_like_images(31 + strides[0] + 2 * strides[1], 5, 4, H=H, W=W)
  ref = N.leg_forward(x, w, model)[:, 0]
  scale = np.abs(ref).max()
  engs = {key: Engine(model=model, precision=prec, max_batch_scans=m, max_batch_pairs=5, proj_H=H, proj_W=W)
          for key, prec, m in (('tc5', 'f16_tc', 5), ('tc1', 'f16_tc', 1), ('fp32', 'fp32', 5))}
  for e in engs.values():
    e.load_weights(w)
  xt = torch.from_numpy(x).to(engs['tc5'].device)
  fv = {k: e.leg(xt) for k, e in engs.items()}
  errs = {k: float(np.abs(v.cpu().numpy() - ref).max() / scale) for k, v in fv.items()}
  between = (fv['tc5'] - fv['tc1']).abs().max().item() / scale
  print('\n[geometry] strides %s (%d x %d): leg rel err %s, 1 vs 5 scans %.2e' % (strides, H, W, errs, between))
  # one scan per call is K-sliced, five are one accumulation chain per layer (tests/test_gpu_network.py, LEG_TC_TOL_*)
  assert errs['tc1'] <= 2e-5 and errs['tc5'] <= 1e-4 and errs['fp32'] <= 2e-5, errs
  assert between <= 1e-4
  # the tensor-core heads once on these volumes
  tc = engs['tc5']
  bank_np = fv['tc5'].cpu().numpy()
  left, right = np.array([0, 1, 2, 3, 4], np.int32), np.array([1, 2, 3, 4, 0], np.int32)
  _, _, _, z = N.heads_forward(bank_np[left][:, None], bank_np[right][:, None], w, model, batch=2, return_logit=True)
  w = N.spread_dense(w, z, target_std=1.5)
  tc.load_weights(w)
  ov_ref, yaw_ref, corr_ref = N.heads_forward(bank_np[left][:, None], bank_np[right][:, None], w, model, batch=2)
  ov, yaw, _ = tc.heads(fv['tc5'], torch.from_numpy(left), torch.from_numpy(right))
  tc.check()
  # The tensor-core heads see only the volumes, whatever the strides; on the volumes of the [1, 2] leg one pair
  # was 1.28e-3 from the float64 oracle on an H100 (the others within 1e-3), so this bound is 2e-3
  err = float(np.abs(ov.cpu().numpy() - ov_ref).max())
  print('[geometry] f16_tc heads on strides %s volumes: max |overlap - oracle| %.2e' % (strides, err))
  assert err <= 2e-3
  check_yaw(yaw.cpu().numpy(), yaw_ref, corr_ref)
  for e in engs.values():
    e.close()
