"""GPU drop-in for the reference's ground-truth generator ``com_overlap_yaw``
(``src/utils/com_overlap_yaw.py:10-68``, used by ``demo/demo4_gen_gt_files.py:77``): same name,
arguments and return value.  The O(N) pose-transformed float64 range projections and the pixel
comparisons run in csrc/gt_overlap.cu through the C ABI (``ovn_gt_range_batch``,
``ovn_gt_overlap_count``); the yaw bin is 4x4 host arithmetic exactly as the reference writes it.

``overlap_yaw_all_pairs`` computes the same ground truth for every (frame, reference) pair of a
sequence at once (``ovn_gt_pairs_count``): the clouds are uploaded once and stay on the device, and
pairs that provably cannot overlap are skipped.  There is no CPU fallback."""
import collections
import math

import numpy as np
import torch

from .engine import CloudBatch
from .preprocess import _engine, _read_scan


def load_poses(pose_path):
  """``load_poses`` (utils.py:10-36): KITTI ``.txt`` (12 numbers per line) or ``.npz['arr_0']`` -> (n,4,4)."""
  poses = []
  try:
    if '.txt' in pose_path:
      with open(pose_path, 'r') as f:
        for line in f.readlines():
          T = np.array(line.split(), dtype=float).reshape(3, 4)
          poses.append(np.vstack((T, [0, 0, 0, 1])))
    else:
      poses = np.load(pose_path)['arr_0']
  except FileNotFoundError:
    print('Ground truth poses are not avaialble.')
  return np.array(poses)


def load_calib(calib_path):
  """``load_calib`` (utils.py:39-56): the ``Tr:`` line of a KITTI calib file -> T_cam_velo (4,4)."""
  T_cam_velo = []
  try:
    with open(calib_path, 'r') as f:
      for line in f.readlines():
        if 'Tr:' in line:
          T = np.array(line.replace('Tr:', '').split(), dtype=float).reshape(3, 4)
          T_cam_velo = np.vstack((T, [0, 0, 0, 1]))
  except FileNotFoundError:
    print('Calibrations are not avaialble.')
  return np.array(T_cam_velo)


def euler_angles_from_rotation_matrix(R):
  """(psi, theta, phi) = roll, pitch, yaw after Slabaugh, as ``utils.py:178-216``."""
  def isclose(x, y, rtol=1.e-5, atol=1.e-8):
    return abs(x - y) <= atol + rtol * abs(y)
  phi = 0.0
  if isclose(R[2, 0], -1.0):
    theta = math.pi / 2.0
    psi = math.atan2(R[0, 1], R[0, 2])
  elif isclose(R[2, 0], 1.0):
    theta = -math.pi / 2.0
    psi = math.atan2(-R[0, 1], -R[0, 2])
  else:
    theta = -math.asin(R[2, 0])
    cos_theta = math.cos(theta)
    psi = math.atan2(R[2, 1] / cos_theta, R[2, 2] / cos_theta)
    phi = math.atan2(R[1, 0] / cos_theta, R[0, 0] / cos_theta)
  return psi, theta, phi


def overlap_yaw_from_clouds(clouds, poses, frame_idx, leg_output_width=360, scans_per_launch=16):
  """The body of ``com_overlap_yaw``: rows [frame_idx, reference_idx, overlap, yaw bin] as float64.
  ``clouds``: list of (N,4) float32 arrays, or of zero-argument callables returning one (read lazily,
  ``scans_per_launch`` at a time, so a whole KITTI sequence never sits in host memory)."""
  poses = np.asarray(poses, dtype=np.float64)
  n = len(clouds)
  eng = _engine(3.0, -25.0, 64, 900, 50)

  def get(i):
    c = clouds[i]
    return np.ascontiguousarray(c() if callable(c) else c, np.float32)

  cur = eng.gt_range(eng.upload_clouds([get(frame_idx)]))[0]
  current_pose = poses[frame_idx]
  cur_inv = np.linalg.inv(current_pose)
  counts = np.zeros(n, np.int64)
  valid_num = 0
  for s0 in range(0, n, scans_per_launch):
    s1 = min(n, s0 + scans_per_launch)
    batch = eng.upload_clouds([get(i) for i in range(s0, s1)])
    ref = eng.gt_range(batch, pose_ref=poses[s0:s1], pose_cur_inv=cur_inv)
    c = eng.gt_overlap_count(ref, cur).cpu().numpy()
    counts[s0:s1] = c[:-1]
    valid_num = int(c[-1])
  mapping = np.zeros((n, 4))
  mapping[:, 0] = np.ones(n) * frame_idx
  mapping[:, 1] = np.arange(n)
  for r in range(n):
    mapping[r, 2] = int(counts[r]) / valid_num                                   # com_overlap_yaw.py:44-46
    mapping[r, 3] = yaw_bin(cur_inv, poses[r], leg_output_width)
  return mapping


def yaw_bin(cur_inv, reference_pose, yaw_resolution=360):
  """Discretised relative yaw of a reference pose seen from the current frame (com_overlap_yaw.py:49-54)."""
  relative_transform = cur_inv.dot(reference_pose)                               # :49
  _, _, yaw = euler_angles_from_rotation_matrix(relative_transform[:3, :3])      # :50-51
  return int(- (yaw / np.pi) * yaw_resolution//2 + yaw_resolution//2)            # :54, same expression


def com_overlap_yaw(scan_paths, poses, frame_idx, leg_output_width=360):
  """Drop-in for ``com_overlap_yaw`` (com_overlap_yaw.py:10-68): ground-truth overlap and yaw bin of
  every scan in ``scan_paths`` against scan ``frame_idx``, from the ground-truth ``poses`` (n,4,4).
  Returns the (n, 4) float64 array [current_frame_idx, reference_frame_idx, overlap, yaw]."""
  print('Start to compute ground truth overlap and yaw ...')
  clouds = [(lambda p=p: _read_scan(p)) for p in scan_paths]      # streamed like the reference (one scan at a time there)
  mapping = overlap_yaw_from_clouds(clouds, poses, frame_idx, leg_output_width)
  print('Finish generating ground_truth_mapping!')
  return mapping


# ---- every frame pair of a sequence --------------------------------------------------------------------

PRUNE_EPS = 1e-3        # metres; the absolute margin of the pruning bound (kGtPruneEps in csrc/gt_overlap.cu)

AllPairs = collections.namedtuple('AllPairs', 'frames counts valid_num yaw_bin n_pruned')
AllPairs.__doc__ = """Ground truth of frames x every scan: ``frames`` int64 [F], ``counts`` int32 [F, N] (pixels
with |dr| < 1), ``valid_num`` int64 [F] (valid pixels of each frame's own image), ``yaw_bin`` int64
[F, N] and ``n_pruned``, the number of pairs skipped because no point can be in range."""


def depth_lower_bound(relative_transform, radius):
  """The bound ovn_gt_pairs_count prunes with, in NumPy: for T = cur_inv . pose_ref (4, 4) and a scan
  whose points satisfy ||p|| <= radius, every transformed point has depth >= the returned value.
  ||M p + t|| >= ||t|| - ||M||_2 ||p||, and ||M||_2^2 <= max row sum of |M^T M|."""
  T = np.asarray(relative_transform, np.float64)
  M, t = T[:3, :3], T[:3, 3]
  s = math.sqrt(np.max(np.sum(np.abs(M.T.dot(M)), axis=1))) * (1.0 + 1e-12)
  return float(np.linalg.norm(t) - s * radius - PRUNE_EPS)


def _cloud_reader(clouds):
  def get(i):
    c = clouds[i]
    a = np.ascontiguousarray(c() if callable(c) else c, np.float32)
    if a.ndim != 2 or a.shape[1] != 4:
      raise ValueError('cloud %d has shape %s, expected (N, 4)' % (i, a.shape))
    if a.shape[0] == 0:
      raise ValueError('cloud %d is empty' % i)
    return a
  return get


def _runs(frames, positions):
  """Split ``positions`` (indices into ``frames``) into runs where both the position and the frame
  index go up by one: [(first position, first frame, length)]."""
  out, j = [], 0
  while j < len(positions):
    k = j + 1
    while (k < len(positions) and positions[k] == positions[k - 1] + 1
           and frames[positions[k]] == frames[positions[k - 1]] + 1):
      k += 1
    out.append((int(positions[j]), int(frames[positions[j]]), k - j))
    j = k
  return out


def _all_pairs_local(clouds, poses, frames, leg_output_width, device_budget_bytes, tile_cur, tile_ref):
  try:
    return _all_pairs_blocks(clouds, poses, frames, leg_output_width, device_budget_bytes, tile_cur, tile_ref)
  finally:
    # the scan staging buffer is half the free device memory by default: hand it back to the driver rather than
    # leave it in torch's cache, where the library's own allocations (a new handle, its workspaces) cannot reach it
    torch.cuda.empty_cache()


def _all_pairs_blocks(clouds, poses, frames, leg_output_width, device_budget_bytes, tile_cur, tile_ref):
  eng = _engine(3.0, -25.0, 64, 900, 50)
  dev = eng.device
  n, F = len(clouds), len(frames)
  get = _cloud_reader(clouds)
  if device_budget_bytes is None:
    device_budget_bytes = torch.cuda.mem_get_info(dev)[0] // 2
  cap_points = int(device_budget_bytes) // 16
  cur_inv = np.stack([np.linalg.inv(poses[f]) for f in frames]) if F else np.zeros((0, 4, 4))   # :30,40
  d_pose = torch.from_numpy(np.ascontiguousarray(poses.reshape(n, 16))).to(dev)
  d_inv = torch.from_numpy(np.ascontiguousarray(cur_inv.reshape(F, 16))).to(dev)
  counts = torch.zeros((F, n), dtype=torch.int32, device=dev)
  cur = torch.empty((F, eng.H, eng.W), dtype=torch.float32, device=dev)
  valid = torch.zeros((F,), dtype=torch.int32, device=dev)
  pruned = []
  yaw = np.zeros((F, n), np.int64)
  buf = torch.empty((max(cap_points, 1), 4), dtype=torch.float32, device=dev)
  no_ref = torch.empty((0, eng.H, eng.W), dtype=torch.float32, device=dev)

  def frame_images(batch, first, positions):
    # the untransformed images of the frames (com_overlap_yaw.py:29-32); `batch` holds scans first..
    for j, f0, m in _runs(frames, positions):
      a, b = f0 - first, f0 - first + m
      p0 = int(batch.offsets_host[a])
      sub = CloudBatch(batch.points[p0:int(batch.offsets_host[b])], batch.offsets[a:b + 1] - p0,
                       batch.offsets_host[a:b + 1] - p0)
      cur[j:j + m] = eng.gt_range(sub)
    for j in positions:
      valid[j:j + 1] = eng.gt_overlap_count(no_ref, cur[j])

  start, carry = 0, None
  while start < n:
    offs, i = [0], start
    while i < n:                                   # fill the device buffer with whole scans
      a = carry if carry is not None else get(i)
      carry = None
      if offs[-1] + a.shape[0] > cap_points:
        if i == start:
          raise ValueError('cloud %d (%d points) does not fit device_budget_bytes=%d' % (i, a.shape[0],
                                                                                      device_budget_bytes))
        carry = a
        break
      buf[offs[-1]:offs[-1] + a.shape[0]].copy_(torch.from_numpy(a))
      offs.append(offs[-1] + a.shape[0])
      i += 1
    end = i
    offs = np.asarray(offs, np.int64)
    block = CloudBatch(buf[:offs[-1]], torch.from_numpy(offs).to(dev), offs)
    if start == 0:
      inside = np.flatnonzero(frames < end)
      frame_images(block, 0, inside)
      for j in np.flatnonzero(frames >= end):      # frames beyond the first block: uploaded once more, alone
        one = eng.upload_clouds([get(int(frames[j]))])
        frame_images(one, int(frames[j]), np.array([j]))
    radius = eng.gt_scan_radius(block)
    pruned.append(torch.zeros((), dtype=torch.int64, device=dev))
    eng.gt_pairs_count(block, d_pose[start:end], radius, cur, d_inv, counts=counts[:, start:end],
                       n_pruned=pruned[-1], tile_cur=tile_cur, tile_ref=tile_ref)
    for j in range(F):                             # host pose arithmetic while the device counts
      for r in range(start, end):
        yaw[j, r] = yaw_bin(cur_inv[j], poses[r], leg_output_width)
    start = end
  return AllPairs(frames.copy(), counts.cpu().numpy(), valid.cpu().numpy().astype(np.int64), yaw,
                  int(sum(int(p) for p in pruned)))


def overlap_yaw_all_pairs(clouds, poses, frames=None, leg_output_width=360, device_budget_bytes=None,
                          tile_cur=0, tile_ref=0):
  """Ground truth of every pair (frame f, reference scan r) for f in ``frames`` (default: all) and every
  scan r, equal pair by pair to ``overlap_yaw_from_clouds(clouds, poses, f)``.  Returns ``AllPairs``;
  ``all_pairs_rows`` turns it into the reference's rows.

  ``clouds``: (N, 4) float32 arrays or zero-argument callables returning one.  The scans are uploaded in
  blocks of at most ``device_budget_bytes`` (default: half the free device memory), each block once; the
  first block also gives the frames' own images, and a frame outside it is read and uploaded once more.
  ``tile_cur`` x ``tile_ref``: the pair tile of the kernel (0 = default); results do not depend on it.
  With torch.distributed initialised, the frames are split into contiguous blocks over the ranks (each rank
  uses its current CUDA device and reads the whole sequence); rank 0 returns the gathered result, the
  other ranks None."""
  poses = np.asarray(poses, dtype=np.float64)
  n = len(clouds)
  if poses.shape != (n, 4, 4):
    raise ValueError('poses has shape %s, expected (%d, 4, 4)' % (poses.shape, n))
  frames = np.arange(n, dtype=np.int64) if frames is None else np.asarray(frames, np.int64).reshape(-1)
  if frames.size and (frames.min() < 0 or frames.max() >= n):
    raise IndexError('frame index outside [0, %d)' % n)
  dist = torch.distributed
  if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
    rank, world = dist.get_rank(), dist.get_world_size()
    mine = frames[rank * len(frames) // world:(rank + 1) * len(frames) // world]
    part = _all_pairs_local(clouds, poses, mine, leg_output_width, device_budget_bytes, tile_cur, tile_ref)
    parts = [None] * world if rank == 0 else None
    dist.gather_object(part, parts, dst=0)
    if rank != 0:
      return None
    return AllPairs(np.concatenate([p.frames for p in parts]), np.concatenate([p.counts for p in parts]),
                    np.concatenate([p.valid_num for p in parts]), np.concatenate([p.yaw_bin for p in parts]),
                    sum(p.n_pruned for p in parts))
  return _all_pairs_local(clouds, poses, frames, leg_output_width, device_budget_bytes, tile_cur, tile_ref)


def all_pairs_rows(result):
  """The reference's rows [frame, reference, overlap, yaw] (float64), frame-major: the rows of
  ``overlap_yaw_from_clouds`` for each frame, concatenated.  overlap = int(count) / valid_num."""
  F, n = result.counts.shape
  if np.any(result.valid_num[:F] == 0):
    raise ZeroDivisionError('a frame has no valid pixel (valid_num = 0)')
  rows = np.zeros((F * n, 4))
  rows[:, 0] = np.repeat(np.asarray(result.frames, np.float64), n)
  rows[:, 1] = np.tile(np.arange(n), F)
  # int64 / int64 -> float64 is the correctly rounded quotient, as int / int is in Python
  rows[:, 2] = (result.counts.astype(np.int64) / result.valid_num.astype(np.int64)[:, None]).ravel()
  rows[:, 3] = result.yaw_bin.ravel()
  return rows
