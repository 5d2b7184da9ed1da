"""Overlap-based Monte Carlo localization: a LiDAR scan stream localized in a map of keyframe scans, with the
network's overlap and yaw as the observation model and the particle filter on the GPU (DESIGN.md section 7).

  python -m overlapnet_b200.mcl [config/demo.yml] [--keyframe-stride S] [--particles N] [--runs R]
                                [--sigma-overlap 0.1] [--sigma-yaw-deg 10] [--cell 0.5] [--max-distance 5]
                                [--converged-m 2] [--virtual-spacing G [--render-sources 8] [--render-radius R]
                                [--render surfels [--surfel-kappa 1] [--max-splat 8]]]

The model:
  map         K keyframes, each a scan encoded once (Infer.encode_clouds), calibrated on keyframe 0 and kept
              resident, with its planar pose (x_k, y_k, theta_k = atan2(R10, R00)).  ``MapIndex`` rasterises the
              keyframes' bounding box grown by max_distance: each cell holds the keyframe nearest to its centre
              within max_distance (ties to the lowest index), else -1.
  virtual     with a virtual spacing G, the map frames are instead the points of a G-metre lattice within
              max_distance of the keyframes (virtual_map.lattice), each rendered on the GPU from its M nearest
              keyframe clouds within the render radius and encoded; the raster holds the nearest lattice frame
              within G of each cell centre.  ``--render surfels`` renders them from the keyframes' surfels (oriented
              disks, DESIGN.md section 7, "Surfel renders") instead of their points.
  particles   (x, y, theta) with a log-weight, float64, on the device (Engine.mcl_*).
  step        predict (odometry + noise, raster lookup, the touched keyframes listed on the device), the heads on
              LEFT = touched keyframes, RIGHT = the query (ovn_heads_1vsN), update (likelihood, normalisation,
              systematic resampling below rho N effective particles).
  evaluation  keyframes are frames 0, S, 2S, ...; queries the frames = S // 2 mod S, in order; odometry is the
              planar relative pose of consecutive queries.  Per run (seed r of 0..R-1): the estimates, position and
              yaw errors, ESS and n_touched, and the convergence step: the first step after which the position error
              stays below converged_m.

Configs with class probabilities are refused, as in lcd_eval.  Results go to ``<experiments_path>/<testname>``:
``mcl_results.npz`` and ``mcl_summary.json``."""
import argparse
import json
import logging
import math
import os
import sys

import numpy as np
import torch

from ._cabi import SURFEL_MAX_SPLAT, OvnError

logger = logging.getLogger('overlapnet_b200.mcl')

# None of these is tuned on KITTI.  render_sources = 8 comes from the synthetic street-scene study of DESIGN.md
# section 7.
DEFAULTS = dict(cell=0.5, max_distance=5.0, sigma_overlap=0.1, sigma_yaw_deg=10.0, rho=0.5, init_radius=1.0,
                motion_sigma=(0.1, 0.1, math.radians(1.0)), render_sources=8)
MAX_RENDER_SOURCES = 64


# ---- geometry -----------------------------------------------------------------------------------------------
def wrap_pi(a):
  """Angles into (-pi, pi], as the filter wraps them."""
  r = np.fmod(np.asarray(a, np.float64) + np.pi, 2 * np.pi)
  r = np.where(r <= 0.0, r + 2 * np.pi, r)
  return r - np.pi


def planar(poses):
  """(n, 3) x, y, theta = atan2(R10, R00) of (n, 4, 4) poses."""
  poses = np.asarray(poses, np.float64)
  return np.stack([poses[:, 0, 3], poses[:, 1, 3], np.arctan2(poses[:, 1, 0], poses[:, 0, 0])], 1)


def odometry(p):
  """(n, 3) planar relative poses of consecutive rows of ``p`` (n, 3), each in the previous frame; row 0 is zero."""
  p = np.asarray(p, np.float64)
  out = np.zeros_like(p)
  d = p[1:, :2] - p[:-1, :2]
  c, s = np.cos(p[:-1, 2]), np.sin(p[:-1, 2])
  out[1:, 0] = c * d[:, 0] + s * d[:, 1]
  out[1:, 1] = -s * d[:, 0] + c * d[:, 1]
  out[1:, 2] = wrap_pi(p[1:, 2] - p[:-1, 2])
  return out


def split_sequence(n, stride):
  """(keyframes, queries): frames 0, S, 2S, ... and the frames = S // 2 mod S, for a sequence of n frames."""
  stride = int(stride)
  if stride < 2:
    raise ValueError('the keyframe stride must be at least 2, so that no query is a keyframe; got %d' % stride)
  return np.arange(0, n, stride), np.arange(stride // 2, n, stride)


def convergence_step(err, threshold):
  """The first step t with err[t'] < threshold for every t' >= t, -1 when the last error is not below it."""
  bad = np.flatnonzero(~(np.asarray(err, np.float64) < threshold))
  if bad.size == 0:
    return 0
  return -1 if bad[-1] == len(err) - 1 else int(bad[-1] + 1)


class MapIndex:
  """The raster of the nearest keyframe within ``max_distance`` of each cell centre (ties: lowest index).  Cell
  (r, c) covers [x0 + c cell, x0 + (c + 1) cell) x [y0 + r cell, y0 + (r + 1) cell)."""

  def __init__(self, keyframes_xy, cell=0.5, max_distance=5.0):
    from scipy.spatial import cKDTree
    xy = np.asarray(keyframes_xy, np.float64).reshape(-1, 2)
    if xy.shape[0] < 1:
      raise ValueError('a map needs at least one keyframe')
    if not (cell > 0 and max_distance >= 0):
      raise ValueError('cell must be > 0 and max_distance >= 0')
    self.cell, self.max_distance = float(cell), float(max_distance)
    lo = xy.min(0) - max_distance
    hi = xy.max(0) + max_distance
    self.x0, self.y0 = float(lo[0]), float(lo[1])
    self.cols = max(1, int(math.ceil((hi[0] - lo[0]) / cell)))
    self.rows = max(1, int(math.ceil((hi[1] - lo[1]) / cell)))
    cx = self.x0 + (np.arange(self.cols) + 0.5) * cell
    cy = self.y0 + (np.arange(self.rows) + 0.5) * cell
    centres = np.stack(np.meshgrid(cx, cy), -1).reshape(-1, 2)
    k = min(8, xy.shape[0])
    d, idx = cKDTree(xy).query(centres, k=k, distance_upper_bound=max_distance * (1 + 1e-9) + 1e-12)
    d, idx = d.reshape(-1, k), idx.reshape(-1, k)
    # the exact distances of the candidates, so that equal distances tie and go to the lowest index
    valid = idx < xy.shape[0]
    safe = np.where(valid, idx, 0)
    diff = xy[safe] - centres[:, None, :]
    d2 = np.where(valid, diff[..., 0] ** 2 + diff[..., 1] ** 2, np.inf)
    best = d2.min(1)
    cand = np.where(d2 == best[:, None], safe, np.iinfo(np.int64).max).min(1)
    ok = np.isfinite(best) & (best <= max_distance ** 2)
    self.raster = np.where(ok, cand, -1).astype(np.int32).reshape(self.rows, self.cols)


# ---- the filter ---------------------------------------------------------------------------------------------
class OverlapMCL:
  """Localize a scan stream in the map of ``map_clouds`` ((N, 4) float32 arrays or callables returning one) at the
  LiDAR-frame ``map_poses`` (K, 4, 4), with ``infer``'s network (an overlapnet_b200.Infer).  The map's volumes become
  ``infer``'s resident bank; the particle set lives in its engine.

  With ``virtual_spacing`` G, the map frames are the lattice frames of virtual_map.lattice(map_poses, G,
  max_distance), rendered from their ``render_sources`` nearest keyframe clouds within ``render_radius`` (default:
  the handle's max_range); the raster is MapIndex(lattice xy, cell, max_distance=G).  ``render`` 'surfels' renders
  the lattice frames from the keyframes' surfels, with ``surfel_params`` (a dict overriding Engine.surfel_params's
  defaults).  ``keyframes`` holds the map frames' planar poses either way."""

  def __init__(self, infer, map_clouds, map_poses, cell=DEFAULTS['cell'], max_distance=DEFAULTS['max_distance'],
               sigma_overlap=DEFAULTS['sigma_overlap'], sigma_yaw=math.radians(DEFAULTS['sigma_yaw_deg']),
               rho=DEFAULTS['rho'], motion_sigma=DEFAULTS['motion_sigma'], virtual_spacing=None,
               render_sources=DEFAULTS['render_sources'], render_radius=None, render='points', surfel_params=None):
    from .lcd_eval import encode_share
    self.infer = infer
    self.engine = infer._engine
    map_poses = np.asarray(map_poses, np.float64)
    if len(map_clouds) != map_poses.shape[0]:
      raise ValueError('%d map clouds for %d map poses' % (len(map_clouds), map_poses.shape[0]))
    self.max_distance = float(max_distance)
    self.virtual_spacing = None if virtual_spacing is None else float(virtual_spacing)
    self.sigma_overlap, self.sigma_yaw, self.rho = float(sigma_overlap), float(sigma_yaw), float(rho)
    self.motion_sigma = tuple(float(s) for s in motion_sigma)
    if render not in ('points', 'surfels'):
      raise ValueError("render must be 'points' or 'surfels', got %r" % (render,))
    if render == 'surfels' and self.virtual_spacing is None:
      raise ValueError("render='surfels' needs a virtual_spacing: keyframe maps are not rendered")
    self.render = render
    if self.virtual_spacing is None:
      self.keyframes = planar(map_poses)
      self.index = MapIndex(self.keyframes[:, :2], cell, max_distance)
      bank, _ = encode_share(infer, map_clouds)
    else:
      from . import virtual_map
      if not 1 <= int(render_sources) <= MAX_RENDER_SOURCES:
        raise ValueError('render_sources must be in [1, %d], got %s' % (MAX_RENDER_SOURCES, render_sources))
      self.render_sources = int(render_sources)
      self.render_radius = float(self.engine.cfg.max_range if render_radius is None else render_radius)
      frames = virtual_map.lattice(map_poses, self.virtual_spacing, max_distance)
      self.keyframes = planar(frames)
      self.index = MapIndex(self.keyframes[:, :2], cell, self.virtual_spacing)
      surfels = None
      if render == 'surfels':
        prm = self.engine.surfel_params(surfel_params)
        self.surfel_params = dict(kappa=prm.kappa, c_min=prm.c_min, max_splat=prm.max_splat)
        surfels = self.surfel_params
      bank = virtual_map.encode(infer, map_clouds, map_poses, frames, self.render_sources, self.render_radius,
                                surfels=surfels)
    # the tensor-core heads' numeric centres from keyframe 0, before the operand copies are built (as lcd_eval)
    self.engine.calibrate(bank[0])
    infer._set_bank(bank)
    self.bank = infer._bank
    self.engine.mcl_set_map(self.keyframes, self.index.raster, self.index.x0, self.index.y0, self.index.cell)

  def init_global(self, n, seed, init_radius=DEFAULTS['init_radius']):
    self.engine.mcl_init('global', n, seed, init_radius=init_radius)

  def init_pose(self, pose, sigma, n, seed):
    self.engine.mcl_init('pose', n, seed, pose=pose, sigma=sigma)

  def encode(self, cloud):
    """The query's feature volume [360, 128] on the device."""
    return self.infer.encode_clouds([np.ascontiguousarray(cloud, np.float32)])[0]

  def step(self, cloud, odom):
    """One step with a raw query scan: encode, predict, heads on the touched keyframes, update."""
    return self.step_volume(self.encode(cloud), odom)

  def step_volume(self, query, odom):
    """One step with the query's feature volume."""
    eng, bank = self.engine, self.bank

    def observe(ids):
      ov, yaw, _ = eng.heads_1vsN(bank, query, cand_idx=ids)
      return ov, yaw
    try:
      return self.step_observed(odom, observe)
    except OvnError as refused:
      # The tensor-core heads poison every output while a device error (a non-finite operand) is flagged, until
      # ovn_check reports and clears it: check here, so that the next step's heads are clean again.
      try:
        eng.check()
      except OvnError as flagged:
        raise OvnError('%s; the heads flagged: %s' % (refused, flagged)) from refused
      raise

  def step_observed(self, odom, observe):
    """One step with ``observe(ids)`` -> (overlap [n], yaw [n]) in place of the heads: ``ids`` is the int32 cuda
    tensor of the touched keyframes, ascending; yaw is the heads' 180 - argmax.  Returns the estimate dict."""
    touched, n = self.engine.mcl_predict(odom, self.motion_sigma)
    if n:
      ov, yaw = observe(touched[:n])
      ov = torch.as_tensor(ov, dtype=torch.float32, device=self.engine.device).contiguous()
      yaw = torch.as_tensor(yaw, dtype=torch.int32, device=self.engine.device).contiguous()
    else:
      ov = yaw = None
    return self.engine.mcl_update(ov, yaw, n, self.sigma_overlap, self.sigma_yaw, self.rho)

  def particles(self):
    """[4, N] float64 host array: x, y, theta, log-weight."""
    return self.engine.mcl_particles().cpu().numpy()


# ---- sequence evaluation ------------------------------------------------------------------------------------
def run_errors(est, truth):
  """Position (m) and absolute yaw (rad) errors of (T, 3) estimates against (T, 3) true planar poses."""
  est, truth = np.asarray(est, np.float64), np.asarray(truth, np.float64)
  return np.hypot(est[:, 0] - truth[:, 0], est[:, 1] - truth[:, 1]), np.abs(wrap_pi(est[:, 2] - truth[:, 2]))


def summarize(pos_err, yaw_err, conv, converged_m):
  """Success rate over runs, and the mean / RMS errors of the steps after convergence of the successful runs."""
  conv = np.asarray(conv)
  ok = conv >= 0
  pos = np.concatenate([pos_err[r, conv[r]:] for r in np.flatnonzero(ok)]) if ok.any() else np.zeros(0)
  yaw = np.concatenate([yaw_err[r, conv[r]:] for r in np.flatnonzero(ok)]) if ok.any() else np.zeros(0)
  f = (lambda v, g: float(g(v)) if v.size else float('nan'))
  return {'runs': int(conv.size), 'success_rate': float(ok.mean()) if conv.size else float('nan'),
          'converged_m': float(converged_m),
          'convergence_step_mean': f(conv[ok].astype(float), np.mean),
          'position_error_mean': f(pos, np.mean), 'position_error_rms': f(pos, lambda v: np.sqrt(np.mean(v * v))),
          'yaw_error_mean_deg': f(np.degrees(yaw), np.mean),
          'yaw_error_rms_deg': f(np.degrees(yaw), lambda v: np.sqrt(np.mean(v * v)))}


def evaluate_sequence(infer, clouds, poses, keyframe_stride=5, particles=100000, runs=5, converged_m=2.0,
                      out_dir=None, **filter_args):
  """Localize the queries of a sequence in the map of its keyframes, ``runs`` times with seeds 0..runs-1 from a
  global initialisation.  ``clouds``: (N, 4) float32 arrays or callables, ``poses`` (n, 4, 4) LiDAR-frame poses.
  Returns (summary dict, results dict of arrays); writes mcl_results.npz and mcl_summary.json to ``out_dir``."""
  from .lcd_eval import save_npz
  poses = np.asarray(poses, np.float64)
  if poses.shape != (len(clouds), 4, 4):
    raise ValueError('poses has shape %s, expected (%d, 4, 4)' % (poses.shape, len(clouds)))
  kf, q = split_sequence(len(clouds), keyframe_stride)
  if q.size == 0:
    raise ValueError('no query frame: the sequence has %d frames, the stride is %d' % (len(clouds), keyframe_stride))
  mcl = OverlapMCL(infer, [clouds[i] for i in kf], poses[kf], **filter_args)
  truth = planar(poses[q])
  odom = odometry(truth)
  queries = torch.stack([mcl.encode(clouds[i]() if callable(clouds[i]) else clouds[i]) for i in q])
  T = q.size
  est = np.zeros((runs, T, 3))
  ess = np.zeros((runs, T))
  n_touched = np.zeros((runs, T), np.int64)
  resampled = np.zeros((runs, T), bool)
  for r in range(runs):
    mcl.init_global(particles, r)
    for t in range(T):
      e = mcl.step_volume(queries[t], odom[t])
      est[r, t] = (e['x'], e['y'], e['theta'])
      ess[r, t], n_touched[r, t], resampled[r, t] = e['ess'], e['n_touched'], e['resampled']
  pos_err = np.zeros((runs, T))
  yaw_err = np.zeros((runs, T))
  for r in range(runs):
    pos_err[r], yaw_err[r] = run_errors(est[r], truth)
  conv = np.array([convergence_step(pos_err[r], converged_m) for r in range(runs)], np.int64)
  summary = summarize(pos_err, yaw_err, conv, converged_m)
  summary.update(frames=len(clouds), keyframes=int(kf.size), queries=int(T), keyframe_stride=int(keyframe_stride),
                 particles=int(particles), cell=mcl.index.cell, max_distance=mcl.max_distance,
                 sigma_overlap=mcl.sigma_overlap, sigma_yaw_deg=math.degrees(mcl.sigma_yaw), rho=mcl.rho)
  results = {'keyframes': kf, 'queries': q, 'truth': truth, 'odometry': odom, 'estimate': est,
             'position_error': pos_err, 'yaw_error': yaw_err, 'ess': ess, 'n_touched': n_touched,
             'resampled': resampled, 'convergence_step': conv}
  if mcl.virtual_spacing is not None:
    summary.update(virtual_spacing=mcl.virtual_spacing, render_sources=mcl.render_sources,
                   render_radius=mcl.render_radius, map_frames=int(mcl.keyframes.shape[0]))
    if mcl.render == 'surfels':
      summary.update(render='surfels', surfel_kappa=mcl.surfel_params['kappa'],
                     surfel_c_min=mcl.surfel_params['c_min'], surfel_max_splat=mcl.surfel_params['max_splat'])
    results['map_frames'] = mcl.keyframes
  if out_dir is not None:
    os.makedirs(out_dir, exist_ok=True)
    save_npz(os.path.join(out_dir, 'mcl_results.npz'), results)
    with open(os.path.join(out_dir, 'mcl_summary.json'), 'w') as f:
      json.dump(summary, f, indent=1, sort_keys=True)
  return summary, results


# ---- the command line ---------------------------------------------------------------------------------------
def parse_args(argv):
  p = argparse.ArgumentParser(prog='python -m overlapnet_b200.mcl',
                              description='Overlap-based Monte Carlo localization over a sequence.')
  p.add_argument('config', nargs='?', default='config/demo.yml', help='YAML file with a Demo3 section')
  p.add_argument('--keyframe-stride', type=int, default=5, help='every S-th frame is a keyframe, S >= 2 (default 5)')
  p.add_argument('--particles', type=int, default=100000, help='particles per run (default 100000)')
  p.add_argument('--runs', type=int, default=5, help='runs with seeds 0..R-1 (default 5)')
  p.add_argument('--sigma-overlap', type=float, default=DEFAULTS['sigma_overlap'])
  p.add_argument('--sigma-yaw-deg', type=float, default=DEFAULTS['sigma_yaw_deg'])
  p.add_argument('--cell', type=float, default=DEFAULTS['cell'], help='raster cell in metres (default 0.5)')
  p.add_argument('--max-distance', type=float, default=DEFAULTS['max_distance'],
                 help='metres from a keyframe a cell may be (default 5)')
  p.add_argument('--converged-m', type=float, default=2.0, help='position error of a converged run (default 2)')
  p.add_argument('--precision', default='f16_tc', choices=('f16_tc', 'fp32'))
  p.add_argument('--virtual-spacing', type=float, default=None,
                 help='localize in a map of virtual scans rendered on a lattice of this spacing in metres '
                      '(default: the keyframe scans themselves)')
  p.add_argument('--render-sources', type=int, default=DEFAULTS['render_sources'],
                 help='keyframe clouds rendered into each virtual scan, 1..%d (default %d)'
                      % (MAX_RENDER_SOURCES, DEFAULTS['render_sources']))
  p.add_argument('--render-radius', type=float, default=None,
                 help='metres from a virtual frame a rendered keyframe may be (default: the max_range)')
  p.add_argument('--render', default='points', choices=('points', 'surfels'),
                 help='render the virtual scans from the keyframes\' points or surfels (default points; needs '
                      '--virtual-spacing)')
  p.add_argument('--surfel-kappa', type=float, default=None,
                 help='surfel radius scale, > 0 (default 1, from a synthetic study; not tuned on KITTI)')
  p.add_argument('--max-splat', type=int, default=None,
                 help='pixels a surfel may cover on each side of its centre, 0..%d (default 8)' % SURFEL_MAX_SPLAT)
  args = p.parse_args(argv)
  if args.keyframe_stride < 2:
    p.error('--keyframe-stride must be at least 2, got %d' % args.keyframe_stride)
  if not 1 <= args.particles <= (1 << 24):
    p.error('--particles must be in [1, 2^24], got %d' % args.particles)
  if args.runs < 1:
    p.error('--runs must be at least 1')
  for name in ('sigma_overlap', 'sigma_yaw_deg', 'cell', 'converged_m'):
    if not getattr(args, name) > 0:
      p.error('--%s must be > 0' % name.replace('_', '-'))
  if not args.max_distance >= 0:
    p.error('--max-distance must be >= 0')
  if args.virtual_spacing is not None and not (args.virtual_spacing > 0 and math.isfinite(args.virtual_spacing)):
    p.error('--virtual-spacing must be > 0')
  if not 1 <= args.render_sources <= MAX_RENDER_SOURCES:
    p.error('--render-sources must be in [1, %d], got %d' % (MAX_RENDER_SOURCES, args.render_sources))
  if args.render_radius is not None and not (args.render_radius > 0 and math.isfinite(args.render_radius)):
    p.error('--render-radius must be > 0')
  if args.render == 'surfels' and args.virtual_spacing is None:
    p.error('--render surfels needs --virtual-spacing')
  if (args.surfel_kappa is not None or args.max_splat is not None) and args.render != 'surfels':
    p.error('--surfel-kappa and --max-splat need --render surfels')
  if args.surfel_kappa is not None and not (args.surfel_kappa > 0 and math.isfinite(args.surfel_kappa)):
    p.error('--surfel-kappa must be > 0')
  if args.max_splat is not None and not 0 <= args.max_splat <= SURFEL_MAX_SPLAT:
    p.error('--max-splat must be in [0, %d], got %d' % (SURFEL_MAX_SPLAT, args.max_splat))
  return args


def virtual_args(args):
  """OverlapMCL's virtual-map arguments of the parsed command line: none without --virtual-spacing."""
  if args.virtual_spacing is None:
    return {}
  out = dict(virtual_spacing=args.virtual_spacing, render_sources=args.render_sources,
             render_radius=args.render_radius)
  if args.render == 'surfels':
    prm = {k: v for k, v in (('kappa', args.surfel_kappa), ('max_splat', args.max_splat)) if v is not None}
    out.update(render='surfels', surfel_params=prm)
  return out


def network_config(config):
  """The network config of a demo.yml dict's Demo3 section, refused when it uses class probabilities."""
  from .config import load_config
  net = load_config(config['Demo3']['network_config'])
  if net.get('use_class_probabilities', False):
    raise Exception('mcl: the network config uses class probabilities, which would need a .label file per scan; only '
                    'geometric configs are localized from raw scans')
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
  s, _ = evaluate_sequence(infer, clouds, poses, args.keyframe_stride, args.particles, args.runs, args.converged_m,
                           out_dir, cell=args.cell, max_distance=args.max_distance, sigma_overlap=args.sigma_overlap,
                           sigma_yaw=math.radians(args.sigma_yaw_deg), **virtual_args(args))
  logger.info('MCL over %d frames: %d keyframes, %d queries, %d particles, %d runs', s['frames'], s['keyframes'],
              s['queries'], s['particles'], s['runs'])
  logger.info('  success rate (position error < %g m to the end): %f', s['converged_m'], s['success_rate'])
  logger.info('  after convergence: position error mean %f m, RMS %f m; yaw error mean %f deg, RMS %f deg',
              s['position_error_mean'], s['position_error_rms'], s['yaw_error_mean_deg'], s['yaw_error_rms_deg'])
  logger.info('  written to %s', out_dir)
  return s


if __name__ == '__main__':
  main()
