"""Thin torch-facing wrapper of the C ABI (include/ovn_b200.h).

PyTorch is plumbing here: it owns device memory and streams; every compute step is a call into
libovn_b200.so.  All methods take / return CUDA tensors and are asynchronous on the current torch
stream unless stated otherwise.
"""
import ctypes as C

import numpy as np
import torch

from . import _cabi
from . import weights as _weights
from ._cabi import OvnConfig, OvnError, check, lib

FEAT_C = 128
HEAD_LAYERS = ('c_conv1', 'c_conv2', 'c_conv3', 'overlap_output')


def leg_layers(model=None):
  """Names of the leg layers (generateNet.py:161-217) of a ``model:`` section, input to output: s_conv3a
  only with ``additional_unsymmetric_layer3a``."""
  use3a = bool(dict(model or {}).get('additional_unsymmetric_layer3a', False))
  return tuple(name for name, *_, opt in _weights.LEG_TABLE if use3a or not opt)


def _ptr(t):
  return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def check_probs(probs, n_points, n_prob, what):
  """Refuse per-point class probabilities that do not fit a handle with ``n_prob`` probability channels before
  anything reaches the device: any array on a handle without such channels, and any shape but
  (n_points, n_prob), one row per point.  None is passed through (the library refuses it on a semantic
  handle with OVN_ERR_INVALID_ARG)."""
  if probs is None:
    return None
  if n_prob == 0:
    raise ValueError('%s: class probabilities given, but the handle has no probability channels' % what)
  shape = tuple(probs.shape)
  if shape != (n_points, n_prob):
    raise ValueError('%s: class probabilities of shape %s, expected (%d, %d): one row of %d per point'
                     % (what, shape, n_points, n_prob, n_prob))
  return probs


class _DeviceBlock:
  """A float32 block of device memory the handle owns, as torch.as_tensor takes it (__cuda_array_interface__)."""

  def __init__(self, ptr, shape):
    self.__cuda_array_interface__ = {'data': (int(ptr), False), 'shape': tuple(shape), 'typestr': '<f4',
                                     'strides': None, 'version': 3}


class CloudBatch:
  """Clouds back to back on the device: points [sum N, 4] f32, offsets [n+1] i64 (+ a host copy)."""

  def __init__(self, points, offsets, offsets_host):
    self.points, self.offsets, self.offsets_host = points, offsets, np.asarray(offsets_host, np.int64)
    self.n = int(self.offsets_host.shape[0] - 1)


class Engine:
  """One handle per GPU.  ``use`` = dict of cue flags like the reference's config
  (config/network.yml:20-24); ``model`` = the ``model:`` section (network.yml:64-82)."""

  def __init__(self, use=None, model=None, precision='f16_tc', device=None, max_batch_scans=16,
               max_batch_pairs=1101, proj_H=64, proj_W=900, fov_up=3.0, fov_down=-25.0, max_range=50.0):
    L = lib()
    if not torch.cuda.is_available():
      raise OvnError('no CUDA device: overlapnet_b200 has no CPU fallback')
    self.device = torch.device('cuda', torch.cuda.current_device() if device is None else device)
    use = dict(use or {})
    model = dict(model or {})
    cfg = OvnConfig()
    L.ovn_default_config(C.byref(cfg))
    cfg.proj_H, cfg.proj_W = proj_H, proj_W
    cfg.fov_up_deg, cfg.fov_down_deg, cfg.max_range = fov_up, fov_down, max_range
    cfg.use_depth = int(bool(use.get('use_depth', True)))
    cfg.use_normals = int(bool(use.get('use_normals', True)))
    cfg.use_intensity = int(bool(use.get('use_intensity', False)))
    if use.get('use_class_probabilities', False):
      cfg.n_prob_channels = 3 if use.get('use_class_probabilities_pca', False) else 20
    else:
      cfg.n_prob_channels = 0
    s1 = model.get('strides_layer1', (2, 2))
    cfg.strides_layer1[0], cfg.strides_layer1[1] = int(s1[0]), int(s1[1])
    cfg.additional_unsymmetric_layer3a = int(bool(model.get('additional_unsymmetric_layer3a', False)))
    cfg.leg_output_width = int(model.get('leg_output_width', 360))
    cfg.conv1size = int(model.get('conv1NetworkHead_conv1size', 15))
    cfg.precision = {'fp32': _cabi.PREC_FP32, 'f16_tc': _cabi.PREC_F16_TC}[precision]
    cfg.max_batch_scans = int(max_batch_scans)
    cfg.max_batch_pairs = int(max_batch_pairs)
    self.cfg = cfg
    self.model = model
    self.precision = precision
    self.train_precision = 'fp32'
    self.H, self.W = proj_H, proj_W
    self._h = C.c_void_p(0)
    with torch.cuda.device(self.device):
      st = L.ovn_create(C.byref(cfg), C.byref(self._h))
    if st != 0:
      raise OvnError('ovn_create failed: %s (%s)' % (L.ovn_status_string(st).decode(),
                                                     L.ovn_last_error(None).decode()))
    self.C = L.ovn_input_channels(self._h)
    self.n_prob = int(cfg.n_prob_channels)
    self.Wf = L.ovn_feature_width(self._h)
    self.max_batch_scans = int(max_batch_scans)
    self.max_batch_pairs = int(max_batch_pairs)
    self._pgo_sizes = []      # (n, E) of each graph of the last successful pose_graph call

  def close(self):
    if getattr(self, '_h', None) is not None and self._h.value:
      for a in getattr(self, '_pinned', ()):                      # host_register'ed blocks still pinned
        lib().ovn_host_unregister(self._h, a.ctypes.data_as(C.c_void_p))
      self._pinned = []
      self._shards = {}                                            # ovn_destroy closes and frees the shards
      lib().ovn_destroy(self._h)
      self._h = C.c_void_p(0)

  def __del__(self):
    try:
      self.close()
    except Exception:
      pass

  # ------------------------------------------------------------------------------------------
  def _stream(self):
    return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

  def launch_count(self):
    return int(lib().ovn_launch_count(self._h))

  def check(self):
    """ovn_check: synchronises the current stream and raises OvnError if a kernel flagged an error
    since the last check (index out of range, unprepared resident row, pipeline barrier time-out);
    the affected outputs hold NaN / INT32_MIN."""
    check(self._h, lib().ovn_check(self._h, self._stream()), 'ovn_check')

  def set_feature_center(self, mu=None):
    """Fix the per-channel centre of the fp16 operand copies (None = calibrate at first use)."""
    ptr = None
    if mu is not None:
      mu = np.ascontiguousarray(mu, np.float32).reshape(FEAT_C)
      ptr = mu.ctypes.data_as(C.c_void_p)
    check(self._h, lib().ovn_set_feature_center(self._h, ptr), 'ovn_set_feature_center')

  def peer_signal(self, flag_addrs, value):
    """ovn_peer_signal: one launch stores ``value`` (release.sys) to each peer-mapped flag address."""
    arr = (C.c_uint64 * len(flag_addrs))(*[int(a) for a in flag_addrs])
    check(self._h, lib().ovn_peer_signal(self._h, arr, len(flag_addrs), int(value), self._stream()), 'ovn_peer_signal')

  def peer_wait(self, flags, n, skip, value):
    """ovn_peer_wait: one launch waits until flags[i] >= value for every i < n except ``skip``."""
    check(self._h, lib().ovn_peer_wait(self._h, _ptr(flags), int(n), int(skip), int(value), self._stream()), 'ovn_peer_wait')

  def calibrate(self, volume):
    """ovn_calibrate: derive the three centres of the tensor-core heads from this [360,128] volume."""
    v = volume.to(device=self.device, dtype=torch.float32).contiguous()
    check(self._h, lib().ovn_calibrate(self._h, _ptr(v), self._stream()), 'ovn_calibrate')

  def get_feature_center(self):
    mu = np.zeros(FEAT_C, np.float32)
    is_set = C.c_int32(0)
    check(self._h, lib().ovn_get_feature_center(self._h, mu.ctypes.data_as(C.c_void_p), C.byref(is_set)),
          'ovn_get_feature_center')
    return mu, bool(is_set.value)

  def profile_enable(self, on=True):
    check(self._h, lib().ovn_profile_enable(self._h, int(bool(on))), 'ovn_profile_enable')

  def profile_read(self, kernel):
    """(total milliseconds, launches) of the named kernel since the last read; synchronises."""
    ms, n = C.c_double(0), C.c_int64(0)
    check(self._h, lib().ovn_profile_read(self._h, kernel.encode(), C.byref(ms), C.byref(n)), 'ovn_profile_read')
    return ms.value, int(n.value)

  def load_weights(self, weights):
    """weights: {layer name: (kernel, bias)} in Keras layouts (overlapnet_b200.weights)."""
    L = lib()
    for name, (k, b) in weights.items():
      k = np.ascontiguousarray(k, dtype=np.float32)
      b = np.ascontiguousarray(b, dtype=np.float32)
      dims = (C.c_int64 * k.ndim)(*k.shape)
      check(self._h, L.ovn_set_weights(self._h, name.encode(), k.ctypes.data_as(C.c_void_p), dims, k.ndim,
                                       b.ctypes.data_as(C.c_void_p), b.size), 'ovn_set_weights(%s)' % name)
    check(self._h, L.ovn_finalize_weights(self._h), 'ovn_finalize_weights')

  # ---- clouds --------------------------------------------------------------------------------
  def upload_clouds(self, clouds):
    """list of (N_i, 4) float32 arrays -> CloudBatch (points [sum N, 4] cuda, offsets [n+1] int64)."""
    offs = np.zeros(len(clouds) + 1, np.int64)
    for i, c in enumerate(clouds):
      offs[i + 1] = offs[i] + c.shape[0]
    flat = np.concatenate([np.ascontiguousarray(c, np.float32).reshape(-1, 4) for c in clouds]) if clouds \
        else np.zeros((0, 4), np.float32)
    return CloudBatch(torch.from_numpy(flat).to(self.device), torch.from_numpy(offs).to(self.device), offs)

  def _chunks(self, batch):
    n = batch.n
    for s0 in range(0, n, self.max_batch_scans):
      s1 = min(n, s0 + self.max_batch_scans)
      p0, p1 = int(batch.offsets_host[s0]), int(batch.offsets_host[s1])
      pts = batch.points[p0:p1]
      offs = batch.offsets[s0:s1 + 1] if p0 == 0 else (batch.offsets[s0:s1 + 1] - p0)
      yield s0, s1, p0, p1, pts, offs.contiguous()

  def project(self, batch, max_range=-1.0, want=('range', 'vertex', 'intensity', 'idx')):
    """ovn_project_batch: range_projection (utils.py:59-134) for a CloudBatch."""
    n = batch.n
    dev = self.device
    out = {}
    if 'range' in want: out['range'] = torch.empty((n, self.H, self.W), dtype=torch.float32, device=dev)
    if 'vertex' in want: out['vertex'] = torch.empty((n, self.H, self.W, 4), dtype=torch.float32, device=dev)
    if 'intensity' in want: out['intensity'] = torch.empty((n, self.H, self.W), dtype=torch.float32, device=dev)
    if 'idx' in want: out['idx'] = torch.empty((n, self.H, self.W), dtype=torch.int32, device=dev)
    L = lib()
    for s0, s1, p0, p1, pts, offs in self._chunks(batch):
      sl = {k: v[s0:s1] for k, v in out.items()}
      check(self._h, L.ovn_project_batch(
          self._h, _ptr(pts), _ptr(offs), s1 - s0, p1 - p0, float(max_range),
          _ptr(sl.get('range')), _ptr(sl.get('vertex')), _ptr(sl.get('intensity')), _ptr(sl.get('idx')),
          self._stream()), 'ovn_project_batch')
    return out

  def gt_range(self, batch, pose_ref=None, pose_cur_inv=None, max_range=-1.0):
    """ovn_gt_range_batch: float32 range images of the scans of a CloudBatch after the two float64
    pose products of com_overlap_yaw.py:39-40 (``pose_ref``: (n,4,4) float64 or None, ``pose_cur_inv``:
    (4,4) float64 or None), projected in float64 like the reference's GT generator."""
    n = batch.n
    dev = self.device
    out = torch.empty((n, self.H, self.W), dtype=torch.float32, device=dev)
    pr = None if pose_ref is None else torch.as_tensor(pose_ref, dtype=torch.float64).reshape(n, 16).to(dev).contiguous()
    pc = None if pose_cur_inv is None else torch.as_tensor(pose_cur_inv, dtype=torch.float64).reshape(16).to(dev).contiguous()
    L = lib()
    for s0, s1, p0, p1, pts, offs in self._chunks(batch):
      check(self._h, L.ovn_gt_range_batch(
          self._h, _ptr(pts), _ptr(offs), s1 - s0, p1 - p0, _ptr(pr[s0:s1]) if pr is not None else None, _ptr(pc),
          float(max_range), _ptr(out[s0:s1]), self._stream()), 'ovn_gt_range_batch')
    return out

  def gt_overlap_count(self, ref_ranges, cur_range):
    """ovn_gt_overlap_count: int32 [n + 1]: per reference image the number of pixels with ref > 0 and
    |ref - cur| < 1 (com_overlap_yaw.py:44-45); last entry = number of valid pixels of ``cur_range``."""
    n = ref_ranges.shape[0]
    counts = torch.empty((n + 1,), dtype=torch.int32, device=self.device)
    check(self._h, lib().ovn_gt_overlap_count(self._h, _ptr(ref_ranges), _ptr(cur_range), n, _ptr(counts),
                                             self._stream()), 'ovn_gt_overlap_count')
    return counts

  def gt_scan_radius(self, batch):
    """ovn_gt_scan_radius: float64 [n] = max ||p|| of each scan of a CloudBatch (0 for an empty scan)."""
    out = torch.empty((batch.n,), dtype=torch.float64, device=self.device)
    check(self._h, lib().ovn_gt_scan_radius(self._h, _ptr(batch.points), _ptr(batch.offsets), batch.n, _ptr(out),
                                           self._stream()), 'ovn_gt_scan_radius')
    return out

  def gt_pairs_count(self, batch, pose_ref, radius, cur_ranges, pose_cur_inv, counts=None, n_pruned=None,
                     max_range=-1.0, tile_cur=0, tile_ref=0):
    """ovn_gt_pairs_count: int32 [n_cur, n_ref] ground-truth counts of every (current frame, reference scan)
    pair, each equal to gt_range + gt_overlap_count for that pair.  ``batch``: the reference scans
    (CloudBatch); ``pose_ref`` float64 [n_ref, 4, 4] and ``radius`` (gt_scan_radius) on the device;
    ``cur_ranges`` [n_cur, H, W] the frames' own images; ``pose_cur_inv`` float64 [n_cur, 4, 4] on the device.
    ``counts`` may be a column slice of a wider int32 tensor (rows contiguous); ``n_pruned`` an int64 device
    scalar that receives the number of pairs skipped by the range bound."""
    n_ref, n_cur = batch.n, int(cur_ranges.shape[0])
    if counts is None:
      counts = torch.empty((n_cur, n_ref), dtype=torch.int32, device=self.device)
    assert counts.dtype == torch.int32 and tuple(counts.shape) == (n_cur, n_ref) and counts.stride(1) == 1
    ld = counts.stride(0) if n_cur > 1 else n_ref
    offs = np.ascontiguousarray(batch.offsets_host, np.int64)
    check(self._h, lib().ovn_gt_pairs_count(
        self._h, _ptr(batch.points), offs.ctypes.data_as(C.c_void_p), n_ref, _ptr(pose_ref), _ptr(radius),
        _ptr(cur_ranges), _ptr(pose_cur_inv), n_cur, float(max_range), int(tile_cur), int(tile_ref), _ptr(counts),
        int(ld), _ptr(n_pruned), self._stream()), 'ovn_gt_pairs_count')
    return counts

  def normals(self, rng, vertex):
    n = rng.shape[0]
    out = torch.empty((n, self.H, self.W, 3), dtype=torch.float32, device=self.device)
    check(self._h, lib().ovn_normals_batch(self._h, _ptr(rng), _ptr(vertex), n, _ptr(out), self._stream()),
          'ovn_normals_batch')
    return out

  def semantic(self, idx, probs, offsets):
    n = idx.shape[0]
    ncls = probs.shape[1]
    out = torch.empty((n, self.H, self.W, ncls), dtype=torch.float32, device=self.device)
    check(self._h, lib().ovn_semantic_batch(self._h, _ptr(idx), _ptr(probs), _ptr(offsets), n, ncls, _ptr(out),
                                           self._stream()), 'ovn_semantic_batch')
    return out

  def preprocess(self, batch, probs=None):
    """Fused raw clouds (CloudBatch) -> packed NHWC network input [n, H, W, C]."""
    n = batch.n
    out = torch.empty((n, self.H, self.W, self.C), dtype=torch.float32, device=self.device)
    L = lib()
    for s0, s1, p0, p1, pts, offs in self._chunks(batch):
      pr = probs[p0:p1] if probs is not None else None
      check(self._h, L.ovn_preprocess_batch(self._h, _ptr(pts), _ptr(offs), s1 - s0, p1 - p0, _ptr(pr),
                                            _ptr(out[s0:s1]), self._stream()), 'ovn_preprocess_batch')
    return out

  def preprocess_cues(self, batch, probs=None):
    """ovn_preprocess_cues_batch: raw clouds (CloudBatch) -> packed NHWC network input [n, H, W, C] with every
    channel as the reference's cue files give it: the class probabilities projected at max_range = inf and
    gathered like gen_semantic_data.py:36-46, the other cues at the configured max_range.  ``probs``: [sum N,
    n_prob] float32 (a CUDA tensor or anything torch.as_tensor takes), the points' rows in batch order;
    required iff the handle has probability channels."""
    n_total = int(batch.offsets_host[-1])
    probs = check_probs(probs, n_total, self.n_prob, 'preprocess_cues')
    if probs is not None:
      probs = torch.as_tensor(probs).to(device=self.device, dtype=torch.float32).contiguous()
    out = torch.empty((batch.n, self.H, self.W, self.C), dtype=torch.float32, device=self.device)
    L = lib()
    for s0, s1, p0, p1, pts, offs in self._chunks(batch):
      pr = probs[p0:p1] if probs is not None else None
      check(self._h, L.ovn_preprocess_cues_batch(self._h, _ptr(pts), _ptr(offs), s1 - s0, p1 - p0, _ptr(pr),
                                                 _ptr(out[s0:s1]), self._stream()), 'ovn_preprocess_cues_batch')
    return out

  def _render_chunks(self, batch, entry_offsets, entry_cloud, entry_pose):
    """Host tables of the render, cut into calls of at most max_batch_scans virtual frames: yields (v0, v1,
    offsets, clouds, poses) with the chunk's entry offsets starting at 0."""
    eo = np.ascontiguousarray(entry_offsets, np.int64).reshape(-1)
    ec = np.ascontiguousarray(entry_cloud, np.int32).reshape(-1)
    ep = np.ascontiguousarray(entry_pose, np.float64).reshape(-1, 16)
    if eo.size < 1 or eo[0] != 0 or eo[-1] != ec.size or ep.shape[0] != ec.size:
      raise ValueError('render: entry_offsets [n_virtual + 1] must run from 0 to the number of entries, with one '
                       'cloud and one 4x4 pose per entry')
    n = eo.size - 1
    for v0 in range(0, n, self.max_batch_scans):
      v1 = min(n, v0 + self.max_batch_scans)
      e0, e1 = int(eo[v0]), int(eo[v1])
      yield v0, v1, np.ascontiguousarray(eo[v0:v1 + 1] - e0), np.ascontiguousarray(ec[e0:e1]), \
          np.ascontiguousarray(ep[e0:e1])

  @staticmethod
  def _hp(a):
    return a.ctypes.data_as(C.c_void_p)

  def render(self, batch, entry_offsets, entry_cloud, entry_pose, max_range=-1.0,
             want=('range', 'vertex', 'intensity', 'winner')):
    """ovn_render_batch: range images of virtual frames rendered from the clouds of a CloudBatch.  Virtual frame v
    concatenates, in entry order, the entries [entry_offsets[v], entry_offsets[v + 1]): cloud entry_cloud[e] moved
    by the float64 pose entry_pose[e] (4x4, T_v^-1 T_k).  ``winner`` is the int32 index of each pixel's point in
    that concatenated cloud, -1 where empty.  Calls of max_batch_scans frames."""
    n = int(np.asarray(entry_offsets).reshape(-1).shape[0]) - 1
    dev = self.device
    out = {}
    if 'range' in want: out['range'] = torch.empty((n, self.H, self.W), dtype=torch.float32, device=dev)
    if 'vertex' in want: out['vertex'] = torch.empty((n, self.H, self.W, 4), dtype=torch.float32, device=dev)
    if 'intensity' in want: out['intensity'] = torch.empty((n, self.H, self.W), dtype=torch.float32, device=dev)
    if 'winner' in want: out['winner'] = torch.empty((n, self.H, self.W), dtype=torch.int32, device=dev)
    offs = np.ascontiguousarray(batch.offsets_host, np.int64)
    L = lib()
    for v0, v1, eo, ec, ep in self._render_chunks(batch, entry_offsets, entry_cloud, entry_pose):
      sl = {k: v[v0:v1] for k, v in out.items()}
      check(self._h, L.ovn_render_batch(
          self._h, _ptr(batch.points), self._hp(offs), batch.n, v1 - v0, self._hp(eo), self._hp(ec), self._hp(ep),
          float(max_range), _ptr(sl.get('range')), _ptr(sl.get('vertex')), _ptr(sl.get('intensity')),
          _ptr(sl.get('winner')), self._stream()), 'ovn_render_batch')
    return out

  def render_preprocess(self, batch, entry_offsets, entry_cloud, entry_pose, out=None):
    """ovn_render_preprocess_batch: the render's packed NHWC network input [n_virtual, H, W, C], as preprocess packs
    a projection (``out``: an optional float32 tensor of that shape to write)."""
    n = int(np.asarray(entry_offsets).reshape(-1).shape[0]) - 1
    if out is None:
      out = torch.empty((n, self.H, self.W, self.C), dtype=torch.float32, device=self.device)
    assert out.dtype == torch.float32 and tuple(out.shape) == (n, self.H, self.W, self.C) and out.is_contiguous()
    offs = np.ascontiguousarray(batch.offsets_host, np.int64)
    L = lib()
    for v0, v1, eo, ec, ep in self._render_chunks(batch, entry_offsets, entry_cloud, entry_pose):
      check(self._h, L.ovn_render_preprocess_batch(
          self._h, _ptr(batch.points), self._hp(offs), batch.n, v1 - v0, self._hp(eo), self._hp(ec), self._hp(ep),
          _ptr(out[v0:v1]), self._stream()), 'ovn_render_preprocess_batch')
    return out

  def surfel_params(self, params=None):
    """ovn_surfel_params: ovn_surfel_default_params (kappa 1, c_min 0.5, max_splat 8, from a synthetic study and not
    tuned on KITTI) with the keys of the ``params`` dict overriding them."""
    prm = _cabi.SurfelParams()
    lib().ovn_surfel_default_params(C.byref(prm))
    for k, v in dict(params or {}).items():
      if k not in ('kappa', 'c_min', 'max_splat'):
        raise ValueError('unknown surfel parameter %r (kappa, c_min, max_splat)' % (k,))
      setattr(prm, k, int(v) if k == 'max_splat' else float(v))
    return prm

  def pixel_rays(self):
    """The float64 unit directions [H, W, 3] of the pixel centres at the handle's geometry (virtual_map.pixel_rays), on
    the device; built once per engine."""
    if getattr(self, '_rays', None) is None:
      from .virtual_map import pixel_rays
      self._rays = torch.from_numpy(pixel_rays(self.H, self.W, self.cfg.fov_up_deg, self.cfg.fov_down_deg)).to(
          self.device)
    return self._rays

  def surfels(self, batch, params=None, out=None):
    """ovn_surfels_batch: the surfel banks [n, H, W, 8] float32 of the clouds of a CloudBatch, one slot per pixel of
    their projections: (cx, cy, cz, r, nx, ny, nz, intensity), all zero where the pixel is empty.  Calls of
    max_batch_scans clouds; ``out``: an optional float32 tensor of that shape to write."""
    if out is None:
      out = torch.empty((batch.n, self.H, self.W, _cabi.SURFEL_FLOATS), dtype=torch.float32, device=self.device)
    assert out.dtype == torch.float32 and tuple(out.shape) == (batch.n, self.H, self.W, _cabi.SURFEL_FLOATS) \
        and out.is_contiguous()
    prm = self.surfel_params(params)
    L = lib()
    for s0, s1, p0, p1, pts, offs in self._chunks(batch):
      check(self._h, L.ovn_surfels_batch(self._h, _ptr(pts), _ptr(offs), s1 - s0, p1 - p0, C.byref(prm),
                                         _ptr(out[s0:s1]), self._stream()), 'ovn_surfels_batch')
    return out

  def _surfel_bank(self, surfels):
    assert surfels.dtype == torch.float32 and surfels.is_contiguous() and \
        tuple(surfels.shape[1:]) == (self.H, self.W, _cabi.SURFEL_FLOATS), 'surfels: [n, H, W, 8] float32 expected'
    return int(surfels.shape[0])

  def render_surfels(self, surfels, entry_offsets, entry_cloud, entry_pose, params=None, max_range=-1.0,
                     want=('range', 'vertex', 'intensity', 'winner')):
    """ovn_render_surfels_batch: range images of virtual frames z-buffered from surfel banks (``surfels`` [n, H, W, 8],
    Engine.surfels), with render's entry tables: entry e is bank entry_cloud[e] moved by entry_pose[e].  ``winner`` is
    each pixel's (entry ordinal in its frame) H W + slot, -1 where empty.  ``params``: as surfel_params (only
    max_splat is read here).  Calls of max_batch_scans frames."""
    n = int(np.asarray(entry_offsets).reshape(-1).shape[0]) - 1
    n_clouds = self._surfel_bank(surfels)
    dev = self.device
    out = {}
    if 'range' in want: out['range'] = torch.empty((n, self.H, self.W), dtype=torch.float32, device=dev)
    if 'vertex' in want: out['vertex'] = torch.empty((n, self.H, self.W, 4), dtype=torch.float32, device=dev)
    if 'intensity' in want: out['intensity'] = torch.empty((n, self.H, self.W), dtype=torch.float32, device=dev)
    if 'winner' in want: out['winner'] = torch.empty((n, self.H, self.W), dtype=torch.int32, device=dev)
    prm = self.surfel_params(params)
    rays = self.pixel_rays()
    L = lib()
    for v0, v1, eo, ec, ep in self._render_chunks(None, entry_offsets, entry_cloud, entry_pose):
      sl = {k: v[v0:v1] for k, v in out.items()}
      check(self._h, L.ovn_render_surfels_batch(
          self._h, _ptr(surfels), n_clouds, _ptr(rays), v1 - v0, self._hp(eo), self._hp(ec), self._hp(ep),
          C.byref(prm), float(max_range), _ptr(sl.get('range')), _ptr(sl.get('vertex')), _ptr(sl.get('intensity')),
          _ptr(sl.get('winner')), self._stream()), 'ovn_render_surfels_batch')
    return out

  def render_surfels_preprocess(self, surfels, entry_offsets, entry_cloud, entry_pose, params=None, out=None):
    """ovn_render_surfels_preprocess_batch: the surfel render's packed NHWC network input [n_virtual, H, W, C], as
    preprocess packs a projection (``out``: an optional float32 tensor of that shape to write)."""
    n = int(np.asarray(entry_offsets).reshape(-1).shape[0]) - 1
    n_clouds = self._surfel_bank(surfels)
    if out is None:
      out = torch.empty((n, self.H, self.W, self.C), dtype=torch.float32, device=self.device)
    assert out.dtype == torch.float32 and tuple(out.shape) == (n, self.H, self.W, self.C) and out.is_contiguous()
    prm = self.surfel_params(params)
    rays = self.pixel_rays()
    L = lib()
    for v0, v1, eo, ec, ep in self._render_chunks(None, entry_offsets, entry_cloud, entry_pose):
      check(self._h, L.ovn_render_surfels_preprocess_batch(
          self._h, _ptr(surfels), n_clouds, _ptr(rays), v1 - v0, self._hp(eo), self._hp(ec), self._hp(ep),
          C.byref(prm), _ptr(out[v0:v1]), self._stream()), 'ovn_render_surfels_preprocess_batch')
    return out

  def pack_input(self, depth=None, normal=None, prob=None, intensity=None):
    first = next(t for t in (depth, normal, prob, intensity) if t is not None)
    n = first.shape[0]
    out = torch.empty((n, self.H, self.W, self.C), dtype=torch.float32, device=self.device)
    check(self._h, lib().ovn_pack_input(self._h, _ptr(depth), _ptr(normal), _ptr(prob), _ptr(intensity), n,
                                       _ptr(out), self._stream()), 'ovn_pack_input')
    return out

  def gather_images(self, images, rows, shifts=None, rot=None, out=None):
    """ovn_gather_images: out[i] = images[rows[i]] rolled by shifts[i] columns with its normals rotated by
    rot[i] = (cos theta, sin theta) (overlapnet_b200.augment).  ``images`` [n_images, H, W, C] float32 cuda;
    ``shifts`` int32 [n] / ``rot`` float32 [n, 2] or None (no roll / no rotation); ``out`` [n, H, W, C] or None.
    A row outside the bank raises OVN_ERR_INVALID_ARG at the next check()."""
    dev = self.device
    x = images.contiguous()
    assert tuple(x.shape[1:]) == (self.H, self.W, self.C) and x.dtype == torch.float32
    ri = torch.as_tensor(rows).to(device=dev, dtype=torch.int32).contiguous()
    n = ri.numel()
    sh = None if shifts is None else torch.as_tensor(shifts).to(device=dev, dtype=torch.int32).contiguous()
    ro = None if rot is None else torch.as_tensor(rot).to(device=dev, dtype=torch.float32).contiguous()
    assert (sh is None or sh.numel() == n) and (ro is None or tuple(ro.shape) == (n, 2))
    if out is None:
      out = torch.empty((n, self.H, self.W, self.C), dtype=torch.float32, device=dev)
    assert tuple(out.shape) == (n, self.H, self.W, self.C) and out.dtype == torch.float32 and out.is_contiguous()
    check(self._h, lib().ovn_gather_images(self._h, _ptr(x), int(x.shape[0]), _ptr(ri), _ptr(sh), _ptr(ro), n,
                                          _ptr(out), self._stream()), 'ovn_gather_images')
    return out

  # ---- network -------------------------------------------------------------------------------
  def leg(self, x_nhwc, out=None):
    """[n, H, W, C] float32 cuda -> feature volumes [n, 360, 128] float32 cuda (written into ``out``, a contiguous
    tensor of that shape, when given)."""
    x = x_nhwc.contiguous()
    n = x.shape[0]
    if out is None:
      out = torch.empty((n, self.Wf, FEAT_C), dtype=torch.float32, device=self.device)
    assert tuple(out.shape) == (n, self.Wf, FEAT_C) and out.dtype == torch.float32 and out.is_contiguous()
    check(self._h, lib().ovn_leg_forward(self._h, _ptr(x), n, _ptr(out), self._stream()), 'ovn_leg_forward')
    return out

  def leg_stage(self, x_nhwc, layer):
    """ovn_leg_stage (precision f16_tc): the leg's own launches on [n <= max_batch_scans, H, W, C] scans up to leg
    layer ``layer`` (0 = s_conv1 ... the last but one) -> (hi, lo), float32 cuda [n, h_out, w_out, cout]: the fp16
    halves of that layer's activations as the next layer reads them."""
    x = x_nhwc.contiguous()
    h, w, cout = self.H, self.W, self.C
    s1 = tuple(self.model.get('strides_layer1', (2, 2)))
    table = [r for r in _weights.LEG_TABLE if r[0] in self.leg_layers]
    for name, kh, kw, sh, sw, cout, _ in table[:int(layer) + 1]:
      sh, sw = s1 if sh is None else (sh, sw)
      h, w = (h - kh) // sh + 1, (w - kw) // sw + 1
    hi, lo = (torch.empty((x.shape[0], h, w, cout), dtype=torch.float32, device=self.device) for _ in range(2))
    # the library refuses a layer outside [0, leg layers - 2] and more than max_batch_scans scans before it writes
    check(self._h, lib().ovn_leg_stage(self._h, _ptr(x), int(x.shape[0]), int(layer), _ptr(hi), _ptr(lo), self._stream()),
          'ovn_leg_stage')
    return hi, lo

  def heads(self, bank, left_idx, right_idx, want_corr=False):
    """LEFT = bank[left_idx], RIGHT = bank[right_idx] -> (overlap [n] f32, yaw [n] i32, corr|None)."""
    n = left_idx.numel()
    ov = torch.empty((n,), dtype=torch.float32, device=self.device)
    yaw = torch.empty((n,), dtype=torch.int32, device=self.device)
    corr = torch.empty((n, self.Wf), dtype=torch.float32, device=self.device) if want_corr else None
    li = left_idx.to(device=self.device, dtype=torch.int32).contiguous()
    ri = right_idx.to(device=self.device, dtype=torch.int32).contiguous()
    check(self._h, lib().ovn_heads_forward(self._h, _ptr(bank), int(bank.shape[0]), _ptr(li), _ptr(ri), n, _ptr(ov),
                                          _ptr(yaw), _ptr(corr), self._stream()), 'ovn_heads_forward')
    return ov, yaw, corr

  def heads_stage_pairs(self):
    """ovn_heads_stage_pairs (precision f16_tc): the pairs of the last chunk of the last heads call whose stages are
    stored (0 when there are none)."""
    n = C.c_int64(0)
    check(self._h, lib().ovn_heads_stage_pairs(self._h, C.byref(n)), 'ovn_heads_stage_pairs')
    return int(n.value)

  def heads_stage(self, stage, first=0, count=None):
    """ovn_copy_heads_stage (precision f16_tc): pairs [first, first + count) (default: all of them) of what the last
    chunk of the last heads call stored, as a float32 cuda tensor.  ``stage``: 'o1' [count, 360, 24, 64] (i, jb, o:
    c_conv1 output without its bias, minus the o1 centre), 'x3' [count, 24, 24, 128] (ib, jb, c: ReLU(c_conv2) minus
    the x3 centre), 'dense' [count, 24, 24, 2] (the Dense partial sums of each c_conv3 pixel over output channels
    [0, 128) and [128, 256); 0 where ib or jb >= 22), 'centres' [576] (o1 centre 64, x3 centre 128, b2eff 128, b3eff
    256; first and count ignored)."""
    if count is None:
      count = self.heads_stage_pairs() - first
    nb = self.Wf // 15
    shape = {'o1': (count, self.Wf, nb, 64), 'x3': (count, nb, nb, 128), 'dense': (count, nb, nb, 2),
             'centres': (576,)}[stage]
    out = torch.empty(shape, dtype=torch.float32, device=self.device)
    # the library writes exactly `count` pairs (576 floats for the centres) and refuses a range it does not hold
    check(self._h, lib().ovn_copy_heads_stage(self._h, _cabi.HEADS_STAGES[stage], int(first), int(count), _ptr(out),
                                             self._stream()), 'ovn_copy_heads_stage')
    return out

  def heads_1vsN(self, bank, query, cand_idx=None, n_cand=None, want_corr=False, out=None):
    """RIGHT = query [360,128] for every pair, LEFT = bank[cand_idx] (None = first n_cand rows).
    ``out`` = (overlap f32 [n], yaw i32 [n]) tensors to write into -- they may live in another GPU's
    peer-mapped memory (search.py transport 'symm'): the kernels that finish a pair store there directly."""
    if cand_idx is not None:
      ci = cand_idx.to(device=self.device, dtype=torch.int32).contiguous()
      n = ci.numel()
    else:
      ci = None
      n = int(bank.shape[0] if n_cand is None else n_cand)
    if out is not None:
      ov, yaw = out
      assert ov.numel() == n and yaw.numel() == n and ov.dtype == torch.float32 and yaw.dtype == torch.int32
      assert ov.is_contiguous() and yaw.is_contiguous()
    else:
      ov = torch.empty((n,), dtype=torch.float32, device=self.device)
      yaw = torch.empty((n,), dtype=torch.int32, device=self.device)
    corr = torch.empty((n, self.Wf), dtype=torch.float32, device=self.device) if want_corr else None
    check(self._h, lib().ovn_heads_1vsN(self._h, _ptr(bank), int(bank.shape[0]), _ptr(query), _ptr(ci), n, _ptr(ov),
                                       _ptr(yaw), _ptr(corr), self._stream()), 'ovn_heads_1vsN')
    return ov, yaw, corr

  def heads_rows_vs_bank(self, bank, row_lo, row_hi):
    """Rows [row_lo, row_hi) of the ordered all-pairs matrix of ``bank`` (RIGHT = bank[i], LEFT = every
    row): (overlap [rows, n] f32, yaw [rows, n] i32).  One C-ABI call; the row loop runs in the library."""
    n = int(bank.shape[0])
    rows = int(row_hi) - int(row_lo)
    ov = torch.empty((rows, n), dtype=torch.float32, device=self.device)
    yaw = torch.empty((rows, n), dtype=torch.int32, device=self.device)
    check(self._h, lib().ovn_heads_rows_vs_bank(self._h, _ptr(bank), n, int(row_lo), int(row_hi), _ptr(ov), _ptr(yaw),
                                               self._stream()), 'ovn_heads_rows_vs_bank')
    return ov, yaw

  def _topk_out(self, rows, k):
    dev = self.device
    return (torch.empty((rows, k), dtype=torch.float32, device=dev), torch.empty((rows, k), dtype=torch.int32, device=dev),
            torch.empty((rows, k), dtype=torch.int32, device=dev))

  def rows_topk(self, overlap, yaw, n, k):
    """ovn_rows_topk: the best k (1..32) records of each row of ``overlap`` f32 / ``yaw`` i32 [rows, stride] cuda
    tensors, row r's first n[r] entries (``n``: host integers).  Returns (overlap f32, index i32, yaw i32), each
    [rows, k] cuda; ordered by overlap descending, then index ascending; empty slots index -1, overlap -1, yaw 0."""
    assert overlap.dtype == torch.float32 and yaw.dtype == torch.int32 and overlap.shape == yaw.shape
    assert overlap.dim() == 2 and overlap.is_contiguous() and yaw.is_contiguous()
    rows, stride = int(overlap.shape[0]), int(overlap.shape[1])
    nn = np.ascontiguousarray(n, np.int32).reshape(-1)
    assert nn.size == rows
    out = self._topk_out(rows, int(k))
    check(self._h, lib().ovn_rows_topk(self._h, _ptr(overlap), _ptr(yaw), rows, stride, nn.ctypes.data_as(C.c_void_p),
                                       int(k), *[_ptr(t) for t in out], self._stream()), 'ovn_rows_topk')
    return out

  def heads_prefix_topk(self, bank, row_lo, row_hi, n_cand, k):
    """ovn_heads_prefix_topk: for each row i in [row_lo, row_hi), query bank[i] (RIGHT) against the candidates
    bank[0 : n_cand[i - row_lo]] (LEFT), reduced on the device to its best k (1..32) records.  ``n_cand``: host
    integers.  Returns (overlap f32, index i32, yaw i32), each [row_hi - row_lo, k] cuda, ordered as rows_topk."""
    rows = int(row_hi) - int(row_lo)
    nn = np.ascontiguousarray(n_cand, np.int32).reshape(-1)
    assert nn.size == max(rows, 0)
    out = self._topk_out(max(rows, 0), int(k))
    check(self._h, lib().ovn_heads_prefix_topk(self._h, _ptr(bank), int(bank.shape[0]), int(row_lo), int(row_hi),
                                               nn.ctypes.data_as(C.c_void_p), int(k), *[_ptr(t) for t in out],
                                               self._stream()), 'ovn_heads_prefix_topk')
    return out

  # ---- Monte Carlo localization (ovn_mcl_*, overlapnet_b200.mcl) -----------------------------------------------
  def mcl_set_map(self, keyframes, raster, x0, y0, cell):
    """ovn_mcl_set_map: ``keyframes`` (K, 3) x, y, theta; ``raster`` (rows, cols) keyframe index or -1.  Drops the
    particle set."""
    kf = np.ascontiguousarray(keyframes, np.float64).reshape(-1, 3)
    ras = np.ascontiguousarray(raster, np.int32)
    assert ras.ndim == 2
    check(self._h, lib().ovn_mcl_set_map(self._h, kf.ctypes.data_as(C.c_void_p), kf.shape[0],
                                         ras.ctypes.data_as(C.c_void_p), ras.shape[0], ras.shape[1], float(x0),
                                         float(y0), float(cell)), 'ovn_mcl_set_map')
    self._mcl_k = kf.shape[0]
    self._mcl_n = 0

  def mcl_init(self, mode, n, seed, pose=None, sigma=None, init_radius=0.0):
    """ovn_mcl_init: ``mode`` 'global' (uniform in init_radius around a random keyframe, theta uniform) or 'pose'
    (Gaussian around ``pose`` (x, y, theta) with standard deviations ``sigma``)."""
    pose = np.ascontiguousarray(pose if pose is not None else np.zeros(3), np.float64).reshape(3)
    sigma = np.ascontiguousarray(sigma if sigma is not None else np.zeros(3), np.float64).reshape(3)
    check(self._h, lib().ovn_mcl_init(self._h, _cabi.MCL_INIT_MODES[mode], int(n), int(seed) & (2 ** 64 - 1),
                                      pose.ctypes.data_as(C.c_void_p), sigma.ctypes.data_as(C.c_void_p),
                                      float(init_radius), self._stream()), 'ovn_mcl_init')
    self._mcl_n = int(n)

  def mcl_predict(self, odom, sigma):
    """ovn_mcl_predict: (touched int32 cuda [K], n_touched); the first n_touched entries are the touched keyframes,
    ascending."""
    odom = np.ascontiguousarray(odom, np.float64).reshape(3)
    sigma = np.ascontiguousarray(sigma, np.float64).reshape(3)
    touched = torch.empty((getattr(self, '_mcl_k', 0),), dtype=torch.int32, device=self.device)
    n = C.c_int32(0)
    check(self._h, lib().ovn_mcl_predict(self._h, odom.ctypes.data_as(C.c_void_p), sigma.ctypes.data_as(C.c_void_p),
                                         _ptr(touched), C.byref(n), self._stream()), 'ovn_mcl_predict')
    return touched, int(n.value)

  def mcl_update(self, overlap, yaw, n, sigma_overlap, sigma_yaw, rho=0.5):
    """ovn_mcl_update with the heads' overlap f32 / yaw i32 cuda tensors [n] of the last predict's touched keyframes
    (None when n = 0).  Returns the estimate: dict of x, y, theta, ess, n_touched, resampled, step."""
    for t, dtype in ((overlap, torch.float32), (yaw, torch.int32)):   # the library refuses NULL with n > 0
      if t is not None:
        assert t.dtype == dtype and t.is_contiguous() and t.numel() >= n
    est = _cabi.McEstimate()
    check(self._h, lib().ovn_mcl_update(self._h, _ptr(overlap), _ptr(yaw), int(n), float(sigma_overlap),
                                        float(sigma_yaw), float(rho), C.byref(est), self._stream()), 'ovn_mcl_update')
    return {'x': est.x, 'y': est.y, 'theta': est.theta, 'ess': est.ess, 'n_touched': int(est.n_touched),
            'resampled': bool(est.resampled), 'step': int(est.step)}

  def mcl_particles(self):
    """ovn_mcl_copy_particles: [4, N] float64 cuda tensor x, y, theta, log-weight."""
    out = torch.empty((4, self._mcl_n), dtype=torch.float64, device=self.device)
    check(self._h, lib().ovn_mcl_copy_particles(self._h, _ptr(out), self._stream()), 'ovn_mcl_copy_particles')
    return out

  def mcl_stage(self, stage):
    """ovn_mcl_copy_stage: 'motion' [3, N] f64, 'lookup' [N] i32, 'loglik' / 'weights' / 'prefix' [N] f64,
    'ancestors' [N] i32, 'scalars' [8] f64 (m, S, ess, x, y, theta, resampled, u0 of the last update)."""
    n = self._mcl_n
    shape, dtype = {'motion': ((3, n), torch.float64), 'lookup': ((n,), torch.int32),
                    'ancestors': ((n,), torch.int32), 'scalars': ((8,), torch.float64)}.get(stage, ((n,), torch.float64))
    out = torch.empty(shape, dtype=dtype, device=self.device)
    check(self._h, lib().ovn_mcl_copy_stage(self._h, _cabi.MCL_STAGES[stage], _ptr(out), self._stream()),
          'ovn_mcl_copy_stage')
    return out

  def mcl_philox(self, seed, counters):
    """ovn_mcl_philox: the Philox4x32-10 words [n, 4] (int32 cuda, the uint32 bits) of ``counters`` [n, 4]."""
    ctr = torch.as_tensor(np.ascontiguousarray(counters, np.uint32).view(np.int32)).to(self.device).contiguous()
    out = torch.empty_like(ctr)
    check(self._h, lib().ovn_mcl_philox(self._h, int(seed) & (2 ** 64 - 1), _ptr(ctr), int(ctr.shape[0]), _ptr(out),
                                        self._stream()), 'ovn_mcl_philox')
    return out

  def icp(self, vertex, normal, src, dst, init, params=None, want_stage=False):
    """ovn_icp_pairs: point-to-plane ICP of the pairs (source scan src[i] = RIGHT, target scan dst[i] = LEFT) of the
    images ``vertex`` [n, H, W, 4] and ``normal`` [n, H, W, 3] (Engine.project / Engine.normals), from ``init``
    [np, 4, 4] float64.  ``params``: a dict overriding icp_default_params().  Returns a dict of cuda tensors: pose
    [np, 4, 4] f64, rms [np] f64, inliers / valid / iterations / status [np] i32, and with ``want_stage`` assoc
    [np, H, W] i32 and system [np, 29] f64 of the last iteration run.  Index errors surface at the next check()."""
    prm = _cabi.IcpParams()
    lib().ovn_icp_default_params(C.byref(prm))
    for key, value in (params or {}).items():
      if key not in dict(prm._fields_):
        raise KeyError('unknown ICP parameter %r' % key)
      setattr(prm, key, value)
    dev = self.device
    src = torch.as_tensor(src, dtype=torch.int32).reshape(-1).to(dev).contiguous()
    dst = torch.as_tensor(dst, dtype=torch.int32).reshape(-1).to(dev).contiguous()
    n_pairs = int(src.numel())
    init = torch.as_tensor(init, dtype=torch.float64).reshape(n_pairs, 16).to(dev).contiguous()
    assert dst.numel() == n_pairs
    assert vertex.dtype == torch.float32 and normal.dtype == torch.float32 and vertex.is_contiguous() \
        and normal.is_contiguous()
    n = int(vertex.shape[0])
    assert tuple(vertex.shape) == (n, self.H, self.W, 4) and tuple(normal.shape) == (n, self.H, self.W, 3)
    raw = torch.empty((n_pairs, _cabi.ICP_RESULT_BYTES // 8), dtype=torch.float64, device=dev)
    assoc = torch.empty((n_pairs, self.H, self.W), dtype=torch.int32, device=dev) if want_stage else None
    system = torch.empty((n_pairs, _cabi.ICP_SYSTEM_SIZE), dtype=torch.float64, device=dev) if want_stage else None
    check(self._h, lib().ovn_icp_pairs(self._h, _ptr(vertex), _ptr(normal), n, _ptr(src), _ptr(dst), _ptr(init),
                                       n_pairs, C.byref(prm), _ptr(raw), _ptr(assoc), _ptr(system), self._stream()),
          'ovn_icp_pairs')
    ints = raw[:, 17:].view(torch.int32)
    out = {'pose': raw[:, :16].reshape(n_pairs, 4, 4), 'rms': raw[:, 16], 'inliers': ints[:, 0], 'valid': ints[:, 1],
           'iterations': ints[:, 2], 'status': ints[:, 3]}
    if want_stage:
      out.update(assoc=assoc, system=system)
    return out

  def pose_graph(self, graphs, params=None, want_gradient=False, want_trace=False):
    """ovn_pgo_optimize_host: robust pose-graph optimization of ``graphs`` in one launch (one CTA per graph).  Each
    graph is a dict of poses [n, 4, 4], edges [E, 2] (the chain (k, k + 1) first, then the loops), measurements
    [E, 4, 4] (Z ~ T_a^-1 T_b) and weights [E, 6] ((omega, v) order), as pose_graph.chain_graph builds it; every
    graph is checked by pose_graph.check_graph first.  ``params``: a dict overriding pgo_default_params().  Returns
    one dict of host arrays per graph: poses, chi2 and scale per edge, status (ovn_pgo_status), iterations,
    accepted, cg_iterations, initial_cost, final_cost, lambda, max_gradient, and with ``want_gradient`` gradient
    [n, 6], with ``want_trace`` trace (cost, lambda, accepted, cg_iterations of each trial run)."""
    from .pose_graph import check_graph, default_params
    prm = default_params(params)
    graphs = [check_graph(g) for g in graphs]
    if not 1 <= len(graphs) <= _cabi.PGO_MAX_GRAPHS:
      raise ValueError('pose_graph: 1 .. %d graphs per call, got %d' % (_cabi.PGO_MAX_GRAPHS, len(graphs)))
    node_off = np.concatenate([[0], np.cumsum([g['poses'].shape[0] for g in graphs])]).astype(np.int64)
    edge_off = np.concatenate([[0], np.cumsum([g['edges'].shape[0] for g in graphs])]).astype(np.int64)
    out = self.pose_graph_raw(node_off, edge_off, np.concatenate([g['poses'] for g in graphs]),
                              np.concatenate([g['edges'] for g in graphs]),
                              np.concatenate([g['measurements'] for g in graphs]),
                              np.concatenate([g['weights'] for g in graphs]), prm, want_gradient, want_trace)
    check(self._h, out.pop('rc'), 'ovn_pgo_optimize_host')
    res = []
    for g in range(len(graphs)):
      n0, n1, e0, e1 = node_off[g], node_off[g + 1], edge_off[g], edge_off[g + 1]
      r = out['result'][g]
      d = {'poses': out['poses'][n0:n1], 'chi2': out['chi2'][e0:e1], 'scale': out['scale'][e0:e1],
           'status': int(r['status']), 'iterations': int(r['iterations']), 'accepted': int(r['accepted']),
           'cg_iterations': int(r['cg_iterations']), 'initial_cost': float(r['initial_cost']),
           'final_cost': float(r['final_cost']), 'lambda': float(r['lambda']), 'max_gradient': float(r['max_gradient'])}
      if want_gradient:
        d['gradient'] = out['gradient'][n0:n1]
      if want_trace:
        t = out['trace'][g, :d['iterations']]
        d['trace'] = {k: t[k].copy() for k in ('cost', 'lambda', 'accepted', 'cg_iterations')}
      res.append(d)
    return res

  def pose_graph_raw(self, node_off, edge_off, poses, edges, measurements, weights, params, want_gradient=False,
                     want_trace=False, outputs=None):
    """One ovn_pgo_optimize_host call on packed host arrays, unchecked (the library checks them).  ``params``: a
    PgoParams.  ``outputs``: preallocated output arrays to write into (a dict as returned).  Returns the output
    arrays and the status code ``rc``; nothing raises here."""
    node_off = np.ascontiguousarray(node_off, np.int64)
    edge_off = np.ascontiguousarray(edge_off, np.int64)
    poses = np.ascontiguousarray(poses, np.float64).reshape(-1, 4, 4)
    edges = np.ascontiguousarray(edges, np.int32).reshape(-1, 2)
    measurements = np.ascontiguousarray(measurements, np.float64).reshape(-1, 4, 4)
    weights = np.ascontiguousarray(weights, np.float64).reshape(-1, 6)
    G, N, E = node_off.size - 1, poses.shape[0], edges.shape[0]
    res_dt = np.dtype([('initial_cost', 'f8'), ('final_cost', 'f8'), ('lambda', 'f8'), ('max_gradient', 'f8'),
                       ('status', 'i4'), ('iterations', 'i4'), ('accepted', 'i4'), ('cg_iterations', 'i4')])
    tr_dt = np.dtype([('cost', 'f8'), ('lambda', 'f8'), ('accepted', 'i4'), ('cg_iterations', 'i4')])
    out = outputs if outputs is not None else {
        'poses': np.empty((N, 4, 4)), 'result': np.zeros(max(G, 0), res_dt), 'chi2': np.empty(E),
        'scale': np.empty(E), 'gradient': np.empty((N, 6)) if want_gradient else None,
        'trace': np.empty((max(G, 0), params.max_iterations), tr_dt) if want_trace else None}
    p = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else C.c_void_p(0)  # noqa: E731
    rc = lib().ovn_pgo_optimize_host(self._h, G, p(node_off), p(edge_off), p(poses), p(edges), p(measurements),
                                     p(weights), C.byref(params), p(out['poses']), p(out['result']), p(out['chi2']),
                                     p(out['scale']), p(out['gradient']), p(out['trace']), self._stream())
    self._pgo_sizes = list(zip(np.diff(node_off).tolist(), np.diff(edge_off).tolist())) if rc == 0 else []
    return dict(out, rc=rc)

  def pose_graph_workspace(self, name, graph=0):
    """ovn_pgo_copy_workspace: array ``name`` ('T', 'Tt', 'M', 'q', 'Hd', 'gn', 'Ld', 'Ls', 'Lk', 'x', 'r', 'z', 'p',
    'Ap' or 'y') of graph ``graph`` of the last successful pose_graph call, as a float64 host array: [n, 4, 4] for
    T and Tt, [E, 6, 6] for M, [E, 6] for q, [n, 6, 6] for Hd, Ld, Ls and Lk, [n, 6] for the others.  Which positions
    are defined is in include/ovn_b200.h.  Raises OvnError when there is no such call or graph."""
    code, width, per_edge = _cabi.PGO_ARRAYS[name]
    L = lib()
    if not self._pgo_sizes or not 0 <= graph < len(self._pgo_sizes):
      # the library refuses the copy and says why
      check(self._h, L.ovn_pgo_copy_workspace(self._h, code, int(graph), None), 'ovn_pgo_copy_workspace')
    count = self._pgo_sizes[graph][1 if per_edge else 0]
    shape = {16: (count, 4, 4), 36: (count, 6, 6), 6: (count, 6)}[width]
    out = np.empty(shape, np.float64)
    check(self._h, L.ovn_pgo_copy_workspace(self._h, code, int(graph), out.ctypes.data_as(C.c_void_p)),
          'ovn_pgo_copy_workspace')
    return out

  def bank_prepare(self, bank, first=0, count=None):
    """Keep the tensor-core operand copies of bank rows [first, first+count) resident: later heads
    calls on this same tensor skip the per-call conversion (ovn_bank_prepare)."""
    count = int(bank.shape[0]) - first if count is None else int(count)
    check(self._h, lib().ovn_bank_prepare(self._h, _ptr(bank), int(bank.shape[0]), int(first), count, self._stream()),
          'ovn_bank_prepare')

  def bank_release(self, bank=None):
    check(self._h, lib().ovn_bank_release(self._h, _ptr(bank)), 'ovn_bank_release')

  # ---- training of the overlap head with a frozen leg (fp32 handles) -------------------------------
  def head_gradients(self, bank, left_idx, right_idx, gt_overlap, gt_orientation, min_overlap_for_angle=0.7):
    """ovn_head_gradients: forward of both heads for LEFT = bank[left_idx], RIGHT = bank[right_idx], the
    losses of training.py and the backward of the overlap head.  Synchronous; returns the losses
    (total, overlap, orientation) and keeps the batch gradients in the handle."""
    n = left_idx.numel()
    dev = self.device
    li = left_idx.to(device=dev, dtype=torch.int32).contiguous()
    ri = right_idx.to(device=dev, dtype=torch.int32).contiguous()
    gov = torch.as_tensor(gt_overlap).to(device=dev, dtype=torch.float32).contiguous()
    gor = torch.as_tensor(gt_orientation).to(device=dev, dtype=torch.int32).contiguous()
    assert ri.numel() == n and gov.numel() == n and gor.numel() == n
    loss = np.zeros(3, np.float32)
    check(self._h, lib().ovn_head_gradients(self._h, _ptr(bank), int(bank.shape[0]), _ptr(li), _ptr(ri), n, _ptr(gov),
                                           _ptr(gor), float(min_overlap_for_angle), loss.ctypes.data_as(C.c_void_p),
                                           self._stream()), 'ovn_head_gradients')
    return tuple(float(v) for v in loss)

  def adagrad_step(self, lr):
    """ovn_head_adagrad_step: Adagrad update of the head weights from the last gradients."""
    check(self._h, lib().ovn_head_adagrad_step(self._h, float(lr), self._stream()), 'ovn_head_adagrad_step')

  # ---- training of the whole network (fp32 handles) -------------------------------------------------
  def net_gradients(self, images, left_idx, right_idx, gt_overlap, gt_orientation, min_overlap_for_angle=0.7,
                    fv_grad=False):
    """ovn_net_gradients: forward of leg + both heads for LEFT = images[left_idx], RIGHT = images[right_idx]
    (``images`` [n, H, W, C] float32 cuda), the losses of training.py and the backward of every layer.
    Synchronous; returns the losses (total, overlap, orientation), plus dL/d(volumes) [2, n, Wf, 128] before
    s_conv10's ReLU mask when ``fv_grad``.  The batch gradients stay in the handle."""
    n = left_idx.numel()
    dev = self.device
    x = images.contiguous()
    li = left_idx.to(device=dev, dtype=torch.int32).contiguous()
    ri = right_idx.to(device=dev, dtype=torch.int32).contiguous()
    gov = torch.as_tensor(gt_overlap).to(device=dev, dtype=torch.float32).contiguous()
    gor = torch.as_tensor(gt_orientation).to(device=dev, dtype=torch.int32).contiguous()
    assert ri.numel() == n and gov.numel() == n and gor.numel() == n
    assert tuple(x.shape[1:]) == (self.H, self.W, self.C) and x.dtype == torch.float32
    dfv = torch.empty((2, n, self.Wf, FEAT_C), dtype=torch.float32, device=dev) if fv_grad else None
    loss = np.zeros(3, np.float32)
    check(self._h, lib().ovn_net_gradients(self._h, _ptr(x), int(x.shape[0]), _ptr(li), _ptr(ri), n, _ptr(gov),
                                          _ptr(gor), float(min_overlap_for_angle), loss.ctypes.data_as(C.c_void_p),
                                          _ptr(dfv), self._stream()), 'ovn_net_gradients')
    loss = tuple(float(v) for v in loss)
    self._net_pairs = n
    return (loss, dfv) if fv_grad else loss

  def net_volumes(self):
    """ovn_copy_net_volumes: the feature volumes [2, n, Wf, 128] (LEFT, RIGHT) of the last net_gradients batch, as
    its leg forward computed them at the training precision."""
    out = torch.empty((2, getattr(self, '_net_pairs', 0), self.Wf, FEAT_C), dtype=torch.float32, device=self.device)
    check(self._h, lib().ovn_copy_net_volumes(self._h, _ptr(out), self._stream()), 'ovn_copy_net_volumes')
    return out

  def set_train_stop(self, stage=None, layer=0):
    """ovn_set_train_stop: the next gradient call stops once ``stage`` ('o1', 'x4', 'dfv_corr', or 'leg_dy' of leg
    layer ``layer``) is complete, before the step overwrites it.  None: no stop."""
    code = -1 if stage is None else _cabi.TRAIN_STAGES[stage]
    check(self._h, lib().ovn_set_train_stop(self._h, code, int(layer) if stage is not None else -1),
          'ovn_set_train_stop')

  def train_stage(self, stage, layer=0):
    """ovn_copy_train_stage: a stage of the last gradient call as a flat float32 cuda tensor (layouts in
    include/ovn_b200.h, ovn_train_stage).  ``layer``: the leg layer of 'leg_dy' and 'act'."""
    code = _cabi.TRAIN_STAGES[stage]
    n = C.c_int64(0)
    check(self._h, lib().ovn_train_stage_size(self._h, code, int(layer), C.byref(n)), 'ovn_train_stage_size')
    out = torch.empty((int(n.value),), dtype=torch.float32, device=self.device)
    check(self._h, lib().ovn_copy_train_stage(self._h, code, int(layer), _ptr(out), self._stream()),
          'ovn_copy_train_stage')
    return out

  def net_adagrad_step(self, lr):
    """ovn_net_adagrad_step: Adagrad update of every leg and head layer from the last net_gradients."""
    check(self._h, lib().ovn_net_adagrad_step(self._h, float(lr), self._stream()), 'ovn_net_adagrad_step')

  def set_train_precision(self, precision):
    """ovn_set_train_precision: 'fp32' (the default) or 'tf32x3', the arithmetic of head_gradients and
    net_gradients (3xTF32 tensor-core products with fp32 accumulation).  Every other call stays fp32."""
    if precision not in _cabi.TRAIN_PRECISIONS:
      raise ValueError('training precision %r: use one of %s' % (precision, ', '.join(_cabi.TRAIN_PRECISIONS)))
    check(self._h, lib().ovn_set_train_precision(self._h, _cabi.TRAIN_PRECISIONS[precision]),
          'ovn_set_train_precision')
    self.train_precision = precision

  # ---- data-parallel training (fp32 handles) -------------------------------------------------------
  def gradient_size(self, whole_network=False):
    """ovn_train_gradient_size: floats of the flat gradient vector (the head layers, then the leg layers with
    ``whole_network``)."""
    n = C.c_int64(0)
    check(self._h, lib().ovn_train_gradient_size(self._h, int(bool(whole_network)), C.byref(n)),
          'ovn_train_gradient_size')
    return int(n.value)

  def copy_gradients(self, whole_network=False, out=None):
    """ovn_copy_gradients: the last batch's gradients as one flat float32 cuda tensor [gradient_size]
    (written into ``out`` when given)."""
    n = self.gradient_size(whole_network)
    if out is None:
      out = torch.empty((n,), dtype=torch.float32, device=self.device)
    assert out.numel() == n and out.dtype == torch.float32 and out.is_contiguous() and out.device == self.device
    check(self._h, lib().ovn_copy_gradients(self._h, int(bool(whole_network)), _ptr(out), self._stream()),
          'ovn_copy_gradients')
    return out

  def _gradients_chunks(self, fn, rows, left_idx, right_idx, offsets, gt_overlap, gt_orientation,
                        min_overlap_for_angle, whole_network, out):
    n = left_idx.numel()
    dev = self.device
    li = left_idx.to(device=dev, dtype=torch.int32).contiguous()
    ri = right_idx.to(device=dev, dtype=torch.int32).contiguous()
    gov = torch.as_tensor(gt_overlap).to(device=dev, dtype=torch.float32).contiguous()
    gor = torch.as_tensor(gt_orientation).to(device=dev, dtype=torch.int32).contiguous()
    assert ri.numel() == n and gov.numel() == n and gor.numel() == n
    off = np.ascontiguousarray(offsets, np.int32).reshape(-1)
    k = max(off.size - 1, 0)
    size = self.gradient_size(whole_network)
    if out is None:
      out = torch.empty((max(k, 1), size), dtype=torch.float32, device=dev)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.device == dev and out.numel() >= k * size
    loss = np.zeros((max(k, 1), 3), np.float32)
    check(self._h, getattr(lib(), fn)(self._h, _ptr(rows), int(rows.shape[0]), _ptr(li), _ptr(ri), n,
                                      off.ctypes.data_as(C.c_void_p), k, _ptr(gov), _ptr(gor),
                                      float(min_overlap_for_angle), _ptr(out), loss.ctypes.data_as(C.c_void_p),
                                      self._stream()), fn)
    return [tuple(float(v) for v in row) for row in loss[:k]], out

  def head_gradients_chunks(self, bank, left_idx, right_idx, offsets, gt_overlap, gt_orientation,
                            min_overlap_for_angle=0.7, out=None):
    """ovn_head_gradients_chunks: head_gradients + copy_gradients of each chunk [offsets[c], offsets[c + 1]) of the
    pairs, in one call.  Returns the losses of each chunk and the parts [n_chunks, gradient_size(False)] (written
    into ``out`` when given).  Leaves no gradients in the handle."""
    return self._gradients_chunks('ovn_head_gradients_chunks', bank, left_idx, right_idx, offsets, gt_overlap,
                                  gt_orientation, min_overlap_for_angle, False, out)

  def net_gradients_chunks(self, images, left_idx, right_idx, offsets, gt_overlap, gt_orientation,
                           min_overlap_for_angle=0.7, out=None):
    """ovn_net_gradients_chunks: net_gradients + copy_gradients of each chunk of the pairs, in one call.  Returns
    the losses of each chunk and the parts [n_chunks, gradient_size(True)]."""
    x = images.contiguous()
    assert tuple(x.shape[1:]) == (self.H, self.W, self.C) and x.dtype == torch.float32
    return self._gradients_chunks('ovn_net_gradients_chunks', x, left_idx, right_idx, offsets, gt_overlap,
                                  gt_orientation, min_overlap_for_angle, True, out)

  def adagrad_step_sum(self, parts, weights, lr, whole_network=False):
    """ovn_adagrad_step_sum: one Adagrad step with g = sum_k weights[k] parts[k] (in order, float32, weight-0
    parts skipped).  ``parts`` [n_parts, gradient_size] float32 cuda, ``weights`` n_parts floats."""
    n = self.gradient_size(whole_network)
    p = parts.reshape(-1, n)
    assert p.dtype == torch.float32 and p.is_contiguous() and p.device == self.device
    w = np.ascontiguousarray(weights, np.float32).reshape(-1)
    assert w.size == p.shape[0]
    check(self._h, lib().ovn_adagrad_step_sum(self._h, int(bool(whole_network)), _ptr(p), int(p.shape[0]),
                                             w.ctypes.data_as(C.c_void_p), float(lr), self._stream()),
          'ovn_adagrad_step_sum')

  def train_state(self, whole_network=False, out=None):
    """ovn_copy_train_state: the Adagrad accumulators as one flat float32 cuda tensor [gradient_size] in the
    layout of copy_gradients (written into ``out`` when given); zeros on a handle that never trained."""
    n = self.gradient_size(whole_network)
    if out is None:
      out = torch.empty((n,), dtype=torch.float32, device=self.device)
    assert out.numel() == n and out.dtype == torch.float32 and out.is_contiguous() and out.device == self.device
    check(self._h, lib().ovn_copy_train_state(self._h, int(bool(whole_network)), _ptr(out), self._stream()),
          'ovn_copy_train_state')
    return out

  def set_train_state(self, vec, whole_network=False):
    """ovn_set_train_state: the Adagrad accumulators from ``vec`` [gradient_size] (float32, a NumPy array or a
    tensor); without ``whole_network`` only the head layers' part.  load_weights resets them, so call it after."""
    n = self.gradient_size(whole_network)
    v = torch.as_tensor(vec).to(device=self.device, dtype=torch.float32).contiguous().reshape(-1)
    assert v.numel() == n
    check(self._h, lib().ovn_set_train_state(self._h, int(bool(whole_network)), _ptr(v), self._stream()),
          'ovn_set_train_state')

  # ---- a training image bank in host memory (overlapnet_b200.image_bank) ------------------------------------
  def train_workspace_bytes(self, n_pairs, whole_network=False):
    """ovn_train_workspace_bytes: device bytes of this handle's training buffers for n_pairs-pair batches."""
    n = C.c_int64(0)
    check(self._h, lib().ovn_train_workspace_bytes(self._h, int(bool(whole_network)), int(n_pairs), C.byref(n)),
          'ovn_train_workspace_bytes')
    return int(n.value)

  def host_register(self, array):
    """ovn_host_register: page-lock the memory of a C-contiguous NumPy array.  The handle keeps the array until
    host_unregister or close releases it, so that its memory is never freed while pinned."""
    assert array.flags['C_CONTIGUOUS']
    check(self._h, lib().ovn_host_register(self._h, array.ctypes.data_as(C.c_void_p), int(array.nbytes)),
          'ovn_host_register')
    self._pinned = getattr(self, '_pinned', []) + [array]

  def host_unregister(self, array):
    """ovn_host_unregister of an array host_register pinned."""
    kept = [a for a in getattr(self, '_pinned', []) if a is not array]
    assert len(kept) < len(getattr(self, '_pinned', [])), 'the array is not pinned by this handle'
    check(self._h, lib().ovn_host_unregister(self._h, array.ctypes.data_as(C.c_void_p)), 'ovn_host_unregister')
    self._pinned = kept

  def stage_rows(self, host, rows, out):
    """ovn_stage_rows: out[i] = host[rows[i]], one asynchronous copy per row on the current stream.  ``host`` a
    C-contiguous page-locked NumPy array, ``rows`` host integers, ``out`` a contiguous cuda tensor of at least
    len(rows) rows of host's row size."""
    r = np.ascontiguousarray(rows, np.int64).reshape(-1)
    row_bytes = host[0].nbytes if host.shape[0] else 0
    assert host.flags['C_CONTIGUOUS'] and out.is_contiguous() and out.device == self.device
    assert out.shape[0] >= r.size and out[0].numel() * out.element_size() == row_bytes
    check(self._h, lib().ovn_stage_rows(self._h, host.ctypes.data_as(C.c_void_p), int(host.shape[0]), row_bytes,
                                        r.ctypes.data_as(C.c_void_p), int(r.size), _ptr(out), self._stream()),
          'ovn_stage_rows')

  # ---- a training image bank sharded over the GPUs of a node (overlapnet_b200.image_bank) -------------------
  def shard_create(self, n_rows):
    """ovn_shard_create: a shard of ``n_rows`` images [n_rows, H, W, C] float32 in this handle's device memory (at
    least one image's bytes, so that every shard has an address).  Returns (a torch view of it, zero-copy; its
    device address; its 64-byte IPC handle as bytes).  The view is valid until shard_close or close."""
    n_rows = int(n_rows)
    row = self.H * self.W * self.C * 4
    ptr, ipc = C.c_void_p(0), (C.c_uint8 * _cabi.IPC_HANDLE_BYTES)()
    check(self._h, lib().ovn_shard_create(self._h, max(n_rows, 1) * row, C.byref(ptr), ipc), 'ovn_shard_create')
    self._shards = getattr(self, '_shards', {})
    self._shards[ptr.value] = 'own'
    view = torch.as_tensor(_DeviceBlock(ptr.value, (max(n_rows, 1), self.H, self.W, self.C)), device=self.device)
    return view[:n_rows], int(ptr.value), bytes(ipc)

  def shard_open(self, ipc):
    """ovn_shard_open: the device address of another process's shard, from its IPC handle (bytes)."""
    ipc = bytes(ipc)
    assert len(ipc) == _cabi.IPC_HANDLE_BYTES, len(ipc)
    buf = (C.c_uint8 * _cabi.IPC_HANDLE_BYTES).from_buffer_copy(ipc)
    ptr = C.c_void_p(0)
    check(self._h, lib().ovn_shard_open(self._h, buf, C.byref(ptr)), 'ovn_shard_open')
    self._shards = getattr(self, '_shards', {})
    self._shards[ptr.value] = 'open'
    return int(ptr.value)

  def shard_close(self, ptr):
    """ovn_shard_close: synchronises the device, then unmaps a shard shard_open mapped or frees one shard_create
    made (its view must not be used afterwards)."""
    check(self._h, lib().ovn_shard_close(self._h, C.c_void_p(int(ptr))), 'ovn_shard_close')
    self._shards.pop(int(ptr), None)

  def open_shard_count(self):
    """The other processes' shards this handle has mapped and not closed."""
    return sum(1 for kind in getattr(self, '_shards', {}).values() if kind == 'open')

  def gather_rows(self, shards, first, rows, out):
    """ovn_gather_rows: out[i] = row rows[i] of the bank of which shards[s] (device addresses) holds rows
    [first[s], first[s + 1]), one launch on the current stream.  ``rows`` host integers, ``out`` a contiguous cuda
    tensor of at least len(rows) images."""
    r = np.ascontiguousarray(rows, np.int64).reshape(-1)
    f = np.ascontiguousarray(first, np.int64).reshape(-1)
    s = (C.c_void_p * max(len(shards), 1))(*[int(p) for p in shards])
    assert f.size == len(shards) + 1 and out.is_contiguous() and out.device == self.device
    assert out.shape[0] >= r.size and out.dtype == torch.float32
    row_bytes = out[0].numel() * 4 if out.shape[0] else self.H * self.W * self.C * 4
    check(self._h, lib().ovn_gather_rows(self._h, s, f.ctypes.data_as(C.c_void_p), len(shards), row_bytes,
                                         r.ctypes.data_as(C.c_void_p), int(r.size), _ptr(out), self._stream()),
          'ovn_gather_rows')

  @property
  def leg_layers(self):
    """Names of the leg layers of this handle's config, input to output."""
    return leg_layers(self.model)

  @property
  def layers(self):
    """Every layer of this handle's config: the leg layers, then HEAD_LAYERS."""
    return self.leg_layers + HEAD_LAYERS

  def _layer_shapes(self):
    return _weights.layer_shapes(self.C, self.model, self.H, self.W)

  def _read_layers(self, fn, names, what):
    shapes = self._layer_shapes()
    out = {}
    for name in names:
      ks, bs = shapes[name]
      k = np.empty(ks, np.float32)
      b = np.empty(bs, np.float32)
      check(self._h, fn(self._h, name.encode(), k.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p)),
            '%s(%s)' % (what, name))
      out[name] = (k, b)
    return out

  def get_weights(self, names=None):
    """Current weights {layer name: (kernel, bias)} in Keras layouts (every layer when names is None)."""
    names = list(self._layer_shapes()) if names is None else list(names)
    return self._read_layers(lib().ovn_get_weights, names, 'ovn_get_weights')

  def get_gradients(self, names=HEAD_LAYERS):
    """Gradients of the last head_gradients call {layer name: (kernel, bias)} (head layers), or of the last
    net_gradients call (any layer, e.g. ``names=eng.layers``)."""
    return self._read_layers(lib().ovn_get_gradients, names, 'ovn_get_gradients')

  # ---- host-buffer entry points (synchronous) ------------------------------------------------
  def encode_clouds_host(self, clouds, probs=None):
    """list of (N_i, 4) float32 host clouds -> host feature volumes [n, Wf, 128].  ``probs``: a list of (N_i, n_prob)
    per-point class probabilities, one per cloud; given, the call is ovn_encode_clouds_probs_host."""
    if probs is not None:
      if len(probs) != len(clouds):
        raise ValueError('encode_clouds_host: %d probability arrays for %d clouds' % (len(probs), len(clouds)))
      probs = [check_probs(p, c.shape[0], self.n_prob, 'encode_clouds_host') for c, p in zip(clouds, probs)]
    offs = np.zeros(len(clouds) + 1, np.int64)
    for i, c in enumerate(clouds):
      offs[i + 1] = offs[i] + c.shape[0]
    flat = np.ascontiguousarray(np.concatenate([np.asarray(c, np.float32).reshape(-1, 4) for c in clouds]))
    out = np.empty((len(clouds), self.Wf, FEAT_C), np.float32)
    if probs is None:
      check(self._h, lib().ovn_encode_clouds_host(self._h, flat.ctypes.data_as(C.c_void_p),
                                                 offs.ctypes.data_as(C.c_void_p), len(clouds),
                                                 out.ctypes.data_as(C.c_void_p)), 'ovn_encode_clouds_host')
      return out
    flat_probs = np.ascontiguousarray(np.concatenate([np.asarray(p, np.float32) for p in probs]))
    check(self._h, lib().ovn_encode_clouds_probs_host(self._h, flat.ctypes.data_as(C.c_void_p),
                                                     offs.ctypes.data_as(C.c_void_p), len(clouds),
                                                     flat_probs.ctypes.data_as(C.c_void_p),
                                                     out.ctypes.data_as(C.c_void_p)), 'ovn_encode_clouds_probs_host')
    return out

  def query_cloud_vs_bank_host(self, points_host, bank, cand_idx_host=None, n_cand=None, out_overlap=None,
                               out_yaw=None, out_query_fv=None, probs=None):
    """points_host: (N,4) float32 numpy or pinned CPU tensor; bank: cuda [n,360,128]; probs: the points' (N, n_prob)
    class probabilities (float32 numpy or CPU tensor), given: the call is ovn_query_cloud_probs_vs_bank_host.
    Returns (overlap float32 [n_cand], yaw int32 [n_cand]) host arrays."""
    if isinstance(points_host, torch.Tensor):
      p_ptr, npts = C.c_void_p(points_host.data_ptr()), int(points_host.shape[0])
    else:
      points_host = np.ascontiguousarray(points_host, np.float32)
      p_ptr, npts = points_host.ctypes.data_as(C.c_void_p), int(points_host.shape[0])
    probs = check_probs(probs, npts, self.n_prob, 'query_cloud_vs_bank_host')
    if isinstance(probs, torch.Tensor):
      assert probs.device.type == 'cpu' and probs.dtype == torch.float32 and probs.is_contiguous()
      pr_ptr = C.c_void_p(probs.data_ptr())
    elif probs is not None:
      probs = np.ascontiguousarray(probs, np.float32)
      pr_ptr = probs.ctypes.data_as(C.c_void_p)
    if cand_idx_host is not None:
      cand_idx_host = np.ascontiguousarray(cand_idx_host, np.int32)
      n = cand_idx_host.size
      c_ptr = cand_idx_host.ctypes.data_as(C.c_void_p)
    else:
      n = int(bank.shape[0] if n_cand is None else n_cand)
      c_ptr = C.c_void_p(0)
    ov = out_overlap if out_overlap is not None else np.empty((n,), np.float32)
    yw = out_yaw if out_yaw is not None else np.empty((n,), np.int32)
    def hp(a):
      if a is None: return C.c_void_p(0)
      return C.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else a.ctypes.data_as(C.c_void_p)
    if probs is None:
      check(self._h, lib().ovn_query_cloud_vs_bank_host(self._h, p_ptr, npts, _ptr(bank), int(bank.shape[0]), c_ptr,
                                                       n, hp(ov), hp(yw), hp(out_query_fv)),
            'ovn_query_cloud_vs_bank_host')
    else:
      check(self._h, lib().ovn_query_cloud_probs_vs_bank_host(self._h, p_ptr, npts, pr_ptr, _ptr(bank),
                                                             int(bank.shape[0]), c_ptr, n, hp(ov), hp(yw),
                                                             hp(out_query_fv)),
            'ovn_query_cloud_probs_vs_bank_host')
    return ov, yw
