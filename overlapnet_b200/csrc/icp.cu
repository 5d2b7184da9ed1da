// icp.cu -- point-to-plane ICP of loop-closure pairs on range images (ovn_icp_pairs, DESIGN.md sections 4 and 7).
//
// One CTA registers one pair and runs every iteration of it: the pose lives in shared memory, each thread walks the
// source pixels tid, tid + 384, ... and keeps the 29 float64 sums of its pixels, a warp xor tree and then the warps
// in order reduce them, and thread 0 solves the 6x6 system and updates the pose.  Nothing depends on the batch, the
// pair's position in it or the launch, so a pair's result has the same bits in any call.  The association uses the
// ground-truth generator's float64 bin (range_bin.cuh), so a point lands in the pixel the float64 oracle gives it.
#include "range_bin.cuh"
#include "se3.cuh"
#include <math.h>
#include <math_constants.h>

namespace ovn {

constexpr int kIcpThreads = 384;            // 12 warps: the 154 registers of a thread allow one CTA per SM
constexpr int kIcpWarps = kIcpThreads / 32;
constexpr int kIcpSums = OVN_ICP_SYSTEM_SIZE;     // H's upper triangle row by row (21), g (6), inliers, sum e^2
constexpr double kIcpPivot = 1e-12;               // a Cholesky pivot <= kIcpPivot trace(H) is degenerate

// the projection's fill: the vertex map has w = 1 where a point landed, -1 elsewhere; the normal map is (-1, -1, -1)
// where no normal exists, and a unit normal never equals it
__device__ __forceinline__ bool normal_is_fill(float x, float y, float z) { return x == -1.f && y == -1.f && z == -1.f; }

// r = M v for the 3x3 block of a row-major 4x4 (+ its translation when `point`), every operation rounded separately
__device__ __forceinline__ void apply3(const double* T, double x, double y, double z, bool point, double r[3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double s = __dadd_rn(__dadd_rn(__dmul_rn(T[4 * i], x), __dmul_rn(T[4 * i + 1], y)), __dmul_rn(T[4 * i + 2], z));
    r[i] = point ? __dadd_rn(s, T[4 * i + 3]) : s;
  }
}

__device__ __forceinline__ double dot3(double ax, double ay, double az, double bx, double by, double bz) {
  return __dadd_rn(__dadd_rn(__dmul_rn(ax, bx), __dmul_rn(ay, by)), __dmul_rn(az, bz));
}

// Thread 0: Cholesky solve of H delta = -g from the sums S, Rodrigues, T <- [R(omega) | v] T.  Returns the status
// that ends the pair, or -1 to go on.
__device__ int icp_solve_update(const double* S, double* T, double dk, const ovn_icp_params& prm) {
  if (S[27] < (double)prm.min_inliers) return OVN_ICP_TOO_FEW_INLIERS;
  double A[6][6], L[6][6] = {};
  for (int r = 0, k = 0; r < 6; ++r)
    for (int c = r; c < 6; ++c, ++k) A[r][c] = A[c][r] = S[k];
  double tr = 0.0;
  for (int i = 0; i < 6; ++i) tr += A[i][i];
  for (int j = 0; j < 6; ++j) {
    double s = A[j][j];
    for (int k = 0; k < j; ++k) s -= L[j][k] * L[j][k];
    if (!(s > kIcpPivot * tr)) return OVN_ICP_DEGENERATE;
    L[j][j] = sqrt(s);
    for (int i = j + 1; i < 6; ++i) {
      double t = A[i][j];
      for (int k = 0; k < j; ++k) t -= L[i][k] * L[j][k];
      L[i][j] = t / L[j][j];
    }
  }
  double y[6], d[6];
  for (int i = 0; i < 6; ++i) {
    double t = -S[21 + i];
    for (int k = 0; k < i; ++k) t -= L[i][k] * y[k];
    y[i] = t / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double t = y[i];
    for (int k = i + 1; k < 6; ++k) t -= L[k][i] * d[k];
    d[i] = t / L[i][i];
  }
  left_update(d, T);                                   // Rodrigues and T <- [R(omega) | v] T (se3.cuh)
  const double th = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  const double tn = sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5]);
  if (dk == prm.d_end && th < prm.eps_rot && tn < prm.eps_trans) return OVN_ICP_CONVERGED;
  return -1;
}

__global__ void __launch_bounds__(kIcpThreads)
k_icp_pairs(const float4* __restrict__ vertex, const float* __restrict__ normal, int n_scans,
            const int32_t* __restrict__ src, const int32_t* __restrict__ dst, const double* __restrict__ init,
            ovn_icp_params prm, GtParams P, ovn_icp_result* __restrict__ out, int32_t* __restrict__ assoc,
            double* __restrict__ system, int* __restrict__ err) {
  __shared__ double s_T[16];
  __shared__ double s_part[kIcpWarps][kIcpSums];
  __shared__ int s_valid[kIcpWarps];
  __shared__ int s_end;
  const int pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int HW = P.H * P.W;
  int32_t* my_assoc = assoc ? assoc + (size_t)pair * HW : nullptr;
  double* my_system = system ? system + (size_t)pair * kIcpSums : nullptr;
  const int a = src[pair], b = dst[pair];
  if (a < 0 || a >= n_scans || b < 0 || b >= n_scans) {
    // nothing is read for this pair: its outputs are poisoned and the handle's flag is raised
    if (tid == 0) {
      atomicCAS(err, 0, kErrIcpBadIndex);
      for (int i = 0; i < 16; ++i) out[pair].pose[i] = CUDART_NAN;
      out[pair].rms = CUDART_NAN;
      out[pair].inliers = out[pair].valid = out[pair].iterations = 0;
      out[pair].status = OVN_ICP_BAD_INDEX;
    }
    if (my_system && tid < kIcpSums) my_system[tid] = CUDART_NAN;
    if (my_assoc)
      for (int i = tid; i < HW; i += kIcpThreads) my_assoc[i] = -1;
    return;
  }
  const float4* vs = vertex + (size_t)a * HW;
  const float* ns = normal + (size_t)a * HW * 3;
  const float4* vt = vertex + (size_t)b * HW;
  const float* nt = normal + (size_t)b * HW * 3;
  if (tid < 16) s_T[tid] = init[(size_t)pair * 16 + tid];
  int nv = 0;
  for (int i = tid; i < HW; i += kIcpThreads)
    nv += vs[i].w > 0.f && !normal_is_fill(ns[3 * i], ns[3 * i + 1], ns[3 * i + 2]);
  nv = __reduce_add_sync(0xffffffffu, nv);
  if (lane == 0) s_valid[warp] = nv;
  __syncthreads();

  double dk_raw = prm.d_start;
  int status = OVN_ICP_MAX_ITERATIONS, it = 0;
  double S[kIcpSums];                                  // thread 0: the last iteration's sums
  for (; it < prm.iterations; ++it) {
    const double dk = fmax(prm.d_end, dk_raw);
    const double d2max = __dmul_rn(dk, dk);
    double T[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) T[i] = s_T[i];
    double acc[kIcpSums];
#pragma unroll
    for (int k = 0; k < kIcpSums; ++k) acc[k] = 0.0;
    for (int i = tid; i < HW; i += kIcpThreads) {
      int q = -1;
      const float4 v = vs[i];
      const float nx = ns[3 * i], ny = ns[3 * i + 1], nz = ns[3 * i + 2];
      double p[3], m[3], depth;
      int bx, by;
      if (v.w > 0.f && !normal_is_fill(nx, ny, nz)) {
        apply3(T, v.x, v.y, v.z, true, p);
        if (range_bin(p[0], p[1], p[2], P, depth, bx, by)) {
          const int j = by * P.W + bx;
          const float4 w = vt[j];
          const float tx = nt[3 * j], ty = nt[3 * j + 1], tz = nt[3 * j + 2];
          if (w.w > 0.f && !normal_is_fill(tx, ty, tz)) {
            apply3(T, nx, ny, nz, false, m);
            const double dx = __dsub_rn(p[0], (double)w.x), dy = __dsub_rn(p[1], (double)w.y),
                         dz = __dsub_rn(p[2], (double)w.z);
            const double d2 = dot3(dx, dy, dz, dx, dy, dz);
            const double cn = dot3(tx, ty, tz, m[0], m[1], m[2]);
            if (d2 <= d2max && cn >= prm.cos_normal) {
              q = j;
              const double e = dot3(tx, ty, tz, dx, dy, dz);
              const double J[6] = {__dsub_rn(__dmul_rn(p[1], tz), __dmul_rn(p[2], ty)),
                                   __dsub_rn(__dmul_rn(p[2], tx), __dmul_rn(p[0], tz)),
                                   __dsub_rn(__dmul_rn(p[0], ty), __dmul_rn(p[1], tx)), tx, ty, tz};
              int k = 0;
#pragma unroll
              for (int r = 0; r < 6; ++r)
#pragma unroll
                for (int c = r; c < 6; ++c) acc[k++] += J[r] * J[c];
#pragma unroll
              for (int r = 0; r < 6; ++r) acc[21 + r] += J[r] * e;
              acc[27] += 1.0;
              acc[28] += e * e;
            }
          }
        }
      }
      if (my_assoc) my_assoc[i] = q;                   // every iteration: the last one run is what stays
    }
    // fixed order: the xor tree within each warp, then the warps in order
#pragma unroll
    for (int k = 0; k < kIcpSums; ++k) {
      double x = acc[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
      if (lane == 0) s_part[warp][k] = x;
    }
    __syncthreads();
    if (tid == 0) {
      for (int k = 0; k < kIcpSums; ++k) {
        double x = s_part[0][k];
        for (int w = 1; w < kIcpWarps; ++w) x += s_part[w][k];
        S[k] = x;
        if (my_system) my_system[k] = x;
      }
      s_end = icp_solve_update(S, s_T, dk, prm);
    }
    __syncthreads();
    const int end = s_end;
    if (end >= 0) {
      status = end;
      ++it;
      break;
    }
    dk_raw = __dmul_rn(dk_raw, prm.gamma);
  }
  if (tid == 0) {
    ovn_icp_result& r = out[pair];
    for (int i = 0; i < 12; ++i) r.pose[i] = s_T[i];
    r.pose[12] = 0.0; r.pose[13] = 0.0; r.pose[14] = 0.0; r.pose[15] = 1.0;
    r.rms = S[27] > 0.0 ? sqrt(S[28] / S[27]) : 0.0;
    r.inliers = (int32_t)S[27];
    int valid = 0;
    for (int w = 0; w < kIcpWarps; ++w) valid += s_valid[w];
    r.valid = valid;
    r.iterations = it;
    r.status = status;
  }
}

int icp_pairs(ovn_handle* h, const float* d_vertex, const float* d_normal, int n_scans, const int32_t* d_src,
              const int32_t* d_dst, const double* d_init, int np, const ovn_icp_params& prm, ovn_icp_result* d_out,
              int32_t* d_assoc, double* d_system, cudaStream_t s) {
  if (np == 0) return OVN_OK;
  const GtParams P = gt_params(h, -1.0f);
  k_icp_pairs<<<np, kIcpThreads, 0, s>>>(reinterpret_cast<const float4*>(d_vertex), d_normal, n_scans, d_src, d_dst,
                                         d_init, prm, P, d_out, d_assoc, d_system, h->d_err);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

}  // namespace ovn
