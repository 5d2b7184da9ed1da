// se3.cuh -- the pose update shared by ICP (icp.cu) and the pose-graph optimizer (pose_graph.cu), DESIGN.md section 7,
// and the float64 point transform shared by the ground-truth generator (gt_overlap.cu) and the render (projection.cu).
// A pose is the first three rows of a row-major 4x4; an update xi = (omega, v) moves it on the left,
// T <- [R(omega) | v] T, with R by Rodrigues.
#pragma once
#include <math.h>

namespace ovn {

// row-major 4x4 times (x, y, z, w): left-to-right sums of separately rounded products, which is
// what a reference BLAS without FMA contraction produces; FMA vs non-FMA differences (<= 1 ulp of a
// coordinate) move a point across a bin edge or the |dr| < 1 threshold with probability ~1e-12.
__device__ __forceinline__ void mat4_apply(const double* __restrict__ M, double& x, double& y, double& z, double& w) {
  double r[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    r[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(M[4 * i + 0], x), __dmul_rn(M[4 * i + 1], y)),
                               __dmul_rn(M[4 * i + 2], z)), __dmul_rn(M[4 * i + 3], w));
  x = r[0]; y = r[1]; z = r[2]; w = r[3];
}

// R(omega) = I + sin(th) K + (1 - cos(th)) K^2, K the cross-product matrix of the unit axis (row-major 3x3)
__device__ __forceinline__ void rodrigues(const double* d, double R[9]) {
  const double th = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
  if (th > 0.0) {
    const double kx = d[0] / th, ky = d[1] / th, kz = d[2] / th, s = sin(th), c1 = 1.0 - cos(th);
    const double K[9] = {0, -kz, ky, kz, 0, -kx, -ky, kx, 0};
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const double kk = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
        R[3 * i + j] += s * K[3 * i + j] + c1 * kk;
      }
  }
}

// T[0..11] <- [R(d[0..2]) | d[3..5]] T
__device__ __forceinline__ void left_update(const double* d, double* T) {
  double R[9];
  rodrigues(d, R);
  double N[12];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j)
      N[4 * i + j] = R[3 * i] * T[j] + R[3 * i + 1] * T[4 + j] + R[3 * i + 2] * T[8 + j] + (j == 3 ? d[3 + i] : 0.0);
  for (int i = 0; i < 12; ++i) T[i] = N[i];
}

}  // namespace ovn
