// range_bin.cuh -- the float64 pixel of a point under range_projection (utils.py:75-104), shared by the ground-truth
// generator (gt_overlap.cu) and the projective association of ICP (icp.cu), so both bin a point the same way.
#pragma once
#include "common.cuh"

namespace ovn {

struct GtParams {
  int H, W;
  double pi, abs_fov_down, fov, max_range;
};

// depth, -atan2, asin, floor and clamp in float64, every product and sum rounded separately; false when the depth is
// outside (0, max_range), which drops the point
__device__ __forceinline__ bool range_bin(double x, double y, double z, const GtParams& P, double& depth, int& bx,
                                          int& by) {
  depth = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));   // utils.py:75
  if (!(depth > 0.0 && depth < P.max_range)) return false;                                 // :76-77
  const double yaw = -atan2(y, x);                                                         // :86
  const double pitch = asin(__ddiv_rn(z, depth));                                          // :87
  double px = __dmul_rn(0.5, __dadd_rn(__ddiv_rn(yaw, P.pi), 1.0));                        // :90
  double py = __dsub_rn(1.0, __ddiv_rn(__dadd_rn(pitch, P.abs_fov_down), P.fov));          // :91
  px = floor(__dmul_rn(px, (double)P.W));                                                  // :94,98
  py = floor(__dmul_rn(py, (double)P.H));
  bx = (int)fmax(0.0, fmin((double)(P.W - 1), px));                                        // :99-104
  by = (int)fmax(0.0, fmin((double)(P.H - 1), py));
  return true;
}

// the handle's projection geometry in float64 (utils.py:70-72); max_range < 0 takes the handle's
inline GtParams gt_params(const ovn_handle* h, float max_range) {
  GtParams P;
  P.H = h->cfg.proj_H; P.W = h->cfg.proj_W;
  P.pi = 3.14159265358979323846;
  const double fu = (double)h->cfg.fov_up_deg / 180.0 * P.pi, fd = (double)h->cfg.fov_down_deg / 180.0 * P.pi;
  P.abs_fov_down = fabs(fd);
  P.fov = fabs(fd) + fabs(fu);
  P.max_range = max_range < 0 ? (double)h->cfg.max_range : (double)max_range;
  return P;
}

}  // namespace ovn
