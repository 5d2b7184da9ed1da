"""Registration cases shared by the ICP tests: known transforms of kitti_000000 and street-scene pairs."""
import math

import numpy as np

from conftest import load_golden

# (yaw in degrees, translation in metres) of T*, the pose of RIGHT in LEFT's frame
KITTI_TRANSFORMS = [(0.0, (0.5, 0.3, 0.0)), (30.0, (1.5, -1.0, 0.1)), (-30.0, (-1.2, 1.0, 0.0)),
                    (90.0, (0.0, 2.0, 0.0)), (179.0, (1.0, 1.0, 0.0))]
# street-scene pairs: (x, y, yaw in degrees) of RIGHT's sensor in the world; LEFT sits at (2, 3, 0 deg)
STREET_LEFT = (2.0, 3.0, 0.0)
STREET_RIGHT = [(3.0, 3.5, 10.0), (4.5, 1.5, -20.0), (2.0, 3.0, 45.0), (-0.5, 4.0, 170.0)]
SENSOR_HEIGHT = 1.73
# measured on the oracle (tests/test_oracle_icp.py): at most 3.8 mm and 0.022 deg over KITTI_TRANSFORMS from the
# yaw seed; the gates leave about twice that
GATE_TRANSLATION = 0.01
GATE_ROTATION_DEG = 0.05


def rz(yaw, t=(0.0, 0.0, 0.0)):
  T = np.eye(4)
  c, s = math.cos(yaw), math.sin(yaw)
  T[:2, :2] = [[c, -s], [s, c]]
  T[:3, 3] = t
  return T


def moved(points, T):
  """points (N, 4) float32 with xyz mapped by T (float64), intensity kept."""
  out = points.copy()
  out[:, :3] = (np.c_[points[:, :3].astype(np.float64), np.ones(len(points))] @ T.T)[:, :3]
  return out


def kitti_pair(yaw_deg, t):
  """(LEFT cloud, RIGHT cloud, T*): LEFT = kitti_000000's even points, RIGHT = its odd points moved by T*^-1."""
  pts = load_golden('kitti_000000')['points']
  T = rz(math.radians(yaw_deg), t)
  return pts[0::2].copy(), moved(pts[1::2], np.linalg.inv(T)), T


def street_pose(x, y, yaw_deg):
  return rz(math.radians(yaw_deg), (x, y, SENSOR_HEIGHT))


def street_pair(k, seed=7, noise=0.0):
  """(LEFT cloud, RIGHT cloud, T* = T_LEFT^-1 T_RIGHT) of street-scene pair k."""
  from overlapnet_b200.synth import street_scene_cloud
  TL, TR = street_pose(*STREET_LEFT), street_pose(*STREET_RIGHT[k])
  return (street_scene_cloud(TL, seed, noise), street_scene_cloud(TR, seed, noise), np.linalg.solve(TL, TR))


def pixel_centre_image(g, depth=10.0, nz=True, seed=3):
  """(vertex [H, W, 4], normal [H, W, 3]) float32: every vertex on its own pixel's centre ray, a random unit normal
  (with n_z = 0 when not ``nz``: no point constrains z, so H has rank 5)."""
  H, W = g['H'], g['W']
  down = abs(g['fov_down'] / 180.0 * np.pi)
  fov = down + abs(g['fov_up'] / 180.0 * np.pi)
  r, c = np.meshgrid(np.arange(H) + 0.5, np.arange(W) + 0.5, indexing='ij')
  yaw = np.pi * (2.0 * c / W - 1.0)
  pitch = (1.0 - r / H) * fov - down
  v = np.ones((H, W, 4), np.float32)
  v[..., 0] = depth * np.cos(pitch) * np.cos(-yaw)
  v[..., 1] = depth * np.cos(pitch) * np.sin(-yaw)
  v[..., 2] = depth * np.sin(pitch)
  rng = np.random.default_rng(seed)
  n = rng.normal(size=(H, W, 3))
  if not nz:
    n[..., 2] = 0.0
  n /= np.linalg.norm(n, axis=-1, keepdims=True)
  return v, n.astype(np.float32)
