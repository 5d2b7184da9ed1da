// pose_graph.cu -- robust pose-graph optimization of a batch of graphs (ovn_pgo_optimize_host, DESIGN.md sections 4
// and 7, "Pose-graph optimization").
//
// One CTA optimizes one graph and runs every Levenberg-Marquardt trial and every conjugate-gradient iteration of it.
// Threads walk the edges and the nodes in a fixed stride; each edge writes its own Hessian block and gradient part,
// and each node gathers its incident edges in a fixed order (chain (i-1, i), chain (i, i+1), then its loop edges in
// edge order), so there are no atomics.  Sums go through a warp xor tree and then the warps in order.  The
// preconditioner -- the damped diagonal blocks plus the chain's off-diagonal blocks, block tridiagonal -- is factored
// exactly by block Cholesky in nested-dissection order: a separator every ceil((n-1)/W) nodes, each warp eliminates
// its segment's interior and forms its part of the separators' Schur complement, warp 0 factors the separator chain,
// and every warp back-substitutes its segment.  Nothing depends on the batch or the graph's position in it, so a
// graph's outputs have the same bits in any call.
#include "common.cuh"
#include "se3.cuh"
#include <math.h>
#include <math_constants.h>
#include <algorithm>

namespace ovn {

constexpr int kPgoThreads = 256;            // 8 warps, 8 segments of the chain: 254 registers, no spills (DESIGN section 4)
constexpr int kPgoWarps = kPgoThreads / 32;
constexpr int kPgoBlocks = 5;               // 6x6 scratch blocks per warp
constexpr int kPgoSeg = 3 * 36 + 12;        // per segment: dLL, dRR, fill(sL, sR), cL, cR
// Log of a rotation at an angle above pi - kPgoPiBranch takes its axis from the symmetric part of R (the oracle's
// PI_BRANCH is the same number)
constexpr double kPgoPiBranch = 1e-2;
// J_l^-1's coefficient of K^2 takes its series below this angle (the oracle's SERIES_BELOW)
constexpr double kPgoSeriesBelow = 1e-2;

struct PgoArgs {
  const int64_t* node_off;
  const int64_t* edge_off;
  const int32_t* enodes;      // [E][2] local node indices
  const int64_t* loop_off;    // [N + 1] node -> loop edges (local edge indices, in edge order)
  const int32_t* loop_list;
  const double* Z;            // [E][16]
  const double* wgt;          // [E][6]
  double *T, *Tt;             // [N][16] current and trial poses
  double *M, *q, *chi2, *scale;   // per edge: rho' A^T W A [36], rho' A^T W e [6], chi2, s
  double *Hd, *gn;            // per node: diagonal block [36], gradient [6]
  double *Ld, *Ls, *Lk;       // per node: Cholesky blocks (diagonal, sub-diagonal, spike / separator chain)
  double *x, *r, *z, *p, *Ap, *y;   // [N][6] CG vectors and the forward solve
  double* seg;                // [G][kPgoWarps][kPgoSeg]
  ovn_pgo_result* res;
  ovn_pgo_trial* trace;       // [G][max_iterations] or NULL
  ovn_pgo_params prm;
};

// ---- SO(3) and the edge residual ----------------------------------------------------------------------------
// phi = Log(R): angle atan2(|axis| / 2, (tr R - 1) / 2) as registration.pose_error computes it
__device__ __forceinline__ void log_so3(const double* R, double phi[3]) {
  const double ax = R[7] - R[5], ay = R[2] - R[6], az = R[3] - R[1];
  const double sn = sqrt(ax * ax + ay * ay + az * az), cs = 0.5 * (R[0] + R[4] + R[8] - 1.0);
  const double th = atan2(0.5 * sn, cs);
  if (th > CUDART_PI - kPgoPiBranch) {
    // R + R^T = 2 cos(th) I + 2 (1 - cos(th)) k k^T: the largest diagonal gives the best-conditioned column
    int i = 0;
    if (R[4] > R[0]) i = 1;
    if (R[8] > R[4 * i]) i = 2;
    const double oc = 1.0 - cs;
    double k[3];
    k[i] = sqrt(fmax((R[4 * i] - cs) / oc, 0.0));
    for (int j = 0; j < 3; ++j)
      if (j != i) k[j] = (R[3 * i + j] + R[3 * j + i]) / (2.0 * oc * k[i]);
    const double sg = (k[0] * ax + k[1] * ay + k[2] * az) < 0.0 ? -1.0 : 1.0;
    for (int j = 0; j < 3; ++j) phi[j] = sg * th * k[j];
  } else if (sn > 0.0) {
    const double f = th / sn;
    phi[0] = f * ax; phi[1] = f * ay; phi[2] = f * az;
  } else {
    phi[0] = phi[1] = phi[2] = 0.0;
  }
}

// J_l^-1(phi) = I - K / 2 + c K^2, c = 1 / th^2 - (1 + cos th) / (2 th sin th)
__device__ __forceinline__ void jl_inv(const double* phi, double J[9]) {
  const double t2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2], th = sqrt(t2);
  const double c = th < kPgoSeriesBelow ? 1.0 / 12.0 + t2 / 720.0 + t2 * t2 / 30240.0
                                        : 1.0 / t2 - (1.0 + cos(th)) / (2.0 * th * sin(th));
  const double K[9] = {0, -phi[2], phi[1], phi[2], 0, -phi[0], -phi[1], phi[0], 0};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double kk = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
      J[3 * i + j] = (i == j ? 1.0 : 0.0) - 0.5 * K[3 * i + j] + c * kk;
    }
}

// E = Z^-1 T_a^-1 T_b: C = Z^-1 T_a^-1 = [RC | tC], e = (Log(R_E), t_E), returns chi2 = e^T diag(w) e
__device__ __forceinline__ double edge_residual(const double* Ta, const double* Tb, const double* Z, const double* w,
                                                double RC[9], double tC[3], double e[6]) {
  double u[3];
  for (int i = 0; i < 3; ++i) u[i] = Ta[i] * Ta[3] + Ta[4 + i] * Ta[7] + Ta[8 + i] * Ta[11] + Z[4 * i + 3];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) RC[3 * i + j] = Z[i] * Ta[4 * j] + Z[4 + i] * Ta[4 * j + 1] + Z[8 + i] * Ta[4 * j + 2];
    tC[i] = -(Z[i] * u[0] + Z[4 + i] * u[1] + Z[8 + i] * u[2]);
  }
  double RE[9];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) RE[3 * i + j] = RC[3 * i] * Tb[j] + RC[3 * i + 1] * Tb[4 + j] + RC[3 * i + 2] * Tb[8 + j];
    e[3 + i] = RC[3 * i] * Tb[3] + RC[3 * i + 1] * Tb[7] + RC[3 * i + 2] * Tb[11] + tC[i];
  }
  log_so3(RE, e);
  double x = 0.0;
  for (int k = 0; k < 6; ++k) x += w[k] * e[k] * e[k];
  return x;
}

// rho(chi2) of an edge and s = rho' ^ (1/2): the chain and phi = inf are least squares, loops Geman-McClure
__device__ __forceinline__ double edge_rho(double x, bool loop, double phi, double& s) {
  if (!loop || isinf(phi)) {
    s = 1.0;
    return x;
  }
  s = phi / (phi + x);
  return s * x;
}

// ---- CTA reductions: the xor tree within each warp, then the warps in order ------------------------------------
__device__ __forceinline__ double block_sum(double v, double* s_red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  double t = s_red[0];
  for (int w = 1; w < kPgoWarps; ++w) t += s_red[w];
  __syncthreads();
  return t;
}

__device__ __forceinline__ double block_max(double v, double* s_red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  double t = s_red[0];
  for (int w = 1; w < kPgoWarps; ++w) t = fmax(t, s_red[w]);
  __syncthreads();
  return t;
}

// ---- 6x6 block operations of one warp, row-major blocks ------------------------------------------------------
// dst = src + lam diag(src) (lam = 0: a copy), or -src with neg
__device__ __forceinline__ void w_load(double* dst, const double* src, double lam, bool neg, int lane) {
  for (int e = lane; e < 36; e += 32) {
    const double v = src[e];
    dst[e] = neg ? -v : (e % 7 == 0 ? v + lam * v : v);
  }
  __syncwarp();
}

__device__ __forceinline__ void w_fill(double* dst, double v, int lane) {
  for (int e = lane; e < 36; e += 32) dst[e] = v;
  __syncwarp();
}

__device__ __forceinline__ void w_copy_t(double* dst, const double* src, int lane) {
  for (int e = lane; e < 36; e += 32) dst[e] = src[6 * (e % 6) + e / 6];
  __syncwarp();
}

// C += beta A B^T
__device__ __forceinline__ void w_abt(double* C, const double* A, const double* B, double beta, int lane) {
  for (int e = lane; e < 36; e += 32) {
    const int r = e / 6, c = e % 6;
    double s = 0.0;
    for (int k = 0; k < 6; ++k) s += A[6 * r + k] * B[6 * c + k];
    C[e] += beta * s;
  }
  __syncwarp();
}

// A <- its lower Cholesky factor (upper part zeroed); false at a pivot that is not positive
__device__ __forceinline__ bool w_chol(double* A, int lane) {
  for (int j = 0; j < 6; ++j) {
    const double d = A[7 * j];
    if (!(d > 0.0)) return false;
    const double l = sqrt(d);
    __syncwarp();
    if (lane == j) A[7 * j] = l;
    else if (lane > j && lane < 6) A[6 * lane + j] /= l;
    __syncwarp();
    for (int e = lane; e < 36; e += 32) {
      const int r = e / 6, c = e % 6;
      if (c > j && c <= r) A[e] -= A[6 * r + j] * A[6 * c + j];
    }
    __syncwarp();
  }
  for (int e = lane; e < 36; e += 32)
    if (e % 6 > e / 6) A[e] = 0.0;
  __syncwarp();
  return true;
}

// B <- B L^-T, one row per lane
__device__ __forceinline__ void w_trsm(const double* L, double* B, int lane) {
  if (lane < 6)
    for (int c = 0; c < 6; ++c) {
      double s = B[6 * lane + c];
      for (int k = 0; k < c; ++k) s -= B[6 * lane + k] * L[6 * c + k];
      B[6 * lane + c] = s / L[7 * c];
    }
  __syncwarp();
}

__device__ __forceinline__ void w_store(double* dst, const double* src, int lane) {
  for (int e = lane; e < 36; e += 32) dst[e] = src[e];
}

// 6-vectors live in lanes 0..5 of a warp.  B v (or B^T v)
__device__ __forceinline__ double w_mv(const double* B, double v, bool trans, int lane) {
  const int r = lane < 6 ? lane : 0;
  double s = 0.0;
  for (int c = 0; c < 6; ++c) {
    const double vc = __shfl_sync(0xffffffffu, v, c);
    s += (trans ? B[6 * c + r] : B[6 * r + c]) * vc;
  }
  return s;
}

// L^-1 v
__device__ __forceinline__ double w_fwd(const double* L, double v, int lane) {
  const int r = lane < 6 ? lane : 0;
  double acc = v, x = 0.0;
  for (int c = 0; c < 6; ++c) {
    if (r == c) x = acc / L[7 * c];
    const double xc = __shfl_sync(0xffffffffu, x, c);
    if (r > c) acc -= L[6 * r + c] * xc;
  }
  return x;
}

// L^-T v
__device__ __forceinline__ double w_bwd(const double* L, double v, int lane) {
  const int r = lane < 6 ? lane : 0;
  double acc = v, x = 0.0;
  for (int c = 5; c >= 0; --c) {
    if (r == c) x = acc / L[7 * c];
    const double xc = __shfl_sync(0xffffffffu, x, c);
    if (r < c) acc -= L[6 * c + r] * xc;
  }
  return x;
}

__device__ __forceinline__ double vload(const double* v, int64_t i, int lane) { return lane < 6 ? v[6 * i + lane] : 0.0; }

// ---- the kernel ------------------------------------------------------------------------------------------------
struct PgoGraph {
  int n, ne;
  int64_t n0, e0;
  const int32_t* en;
  const int64_t* loff;
  const int32_t* ll;
  const double *Z, *w;
  double *T, *Tt, *M, *q, *chi2, *scale, *Hd, *gn, *Ld, *Ls, *Lk, *x, *r, *z, *p, *Ap, *y, *seg;
  int P[kPgoWarps + 2];       // P[0] = 0, separators P[1 .. Q], P[Q + 1] = n
  int Q;
};

// F, the per-edge chi2, s, M and q at G.T, then every node's diagonal block and gradient; returns F and max |g|
// over nodes 1 .. n-1 in gmax
__device__ double linearize(const PgoGraph& G, double phi, double* s_red, double& gmax) {
  double part = 0.0;
  for (int k = threadIdx.x; k < G.ne; k += kPgoThreads) {
    const int a = G.en[2 * k], b = G.en[2 * k + 1];
    const double* w = G.w + 6 * k;
    double RC[9], tC[3], e[6];
    const double x = edge_residual(G.T + 16 * a, G.T + 16 * b, G.Z + 16 * k, w, RC, tC, e);
    double s;
    part += edge_rho(x, k >= G.n - 1, phi, s);
    G.chi2[k] = x;
    G.scale[k] = s;
    const double d = s * s;
    // A = J_E Ad_C = [[J_l^-1 RC, 0], [(tC - tE)^ RC, RC]]
    double Jl[9], A[36];
    jl_inv(e, Jl);
    const double dx = tC[0] - e[3], dy = tC[1] - e[4], dz = tC[2] - e[5];
    const double S[9] = {0, -dz, dy, dz, 0, -dx, -dy, dx, 0};
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        A[6 * i + j] = Jl[3 * i] * RC[j] + Jl[3 * i + 1] * RC[3 + j] + Jl[3 * i + 2] * RC[6 + j];
        A[6 * i + 3 + j] = 0.0;
        A[6 * (3 + i) + j] = S[3 * i] * RC[j] + S[3 * i + 1] * RC[3 + j] + S[3 * i + 2] * RC[6 + j];
        A[6 * (3 + i) + 3 + j] = RC[3 * i + j];
      }
    double* Mk = G.M + 36 * k;
    for (int i = 0; i < 6; ++i) {
      for (int j = i; j < 6; ++j) {
        double t = 0.0;
        for (int r = 0; r < 6; ++r) t += A[6 * r + i] * w[r] * A[6 * r + j];
        Mk[6 * i + j] = Mk[6 * j + i] = d * t;
      }
      double t = 0.0;
      for (int r = 0; r < 6; ++r) t += A[6 * r + i] * w[r] * e[r];
      G.q[6 * k + i] = d * t;
    }
  }
  const double F = 0.5 * block_sum(part, s_red);
  double gm = 0.0;
  for (int i = threadIdx.x; i < G.n; i += kPgoThreads) {
    double H[36], g[6];
    for (int t = 0; t < 36; ++t) H[t] = 0.0;
    for (int t = 0; t < 6; ++t) g[t] = 0.0;
    if (i >= 1) {
      for (int t = 0; t < 36; ++t) H[t] += G.M[36 * (i - 1) + t];
      for (int t = 0; t < 6; ++t) g[t] += G.q[6 * (i - 1) + t];
    }
    if (i <= G.n - 2) {
      for (int t = 0; t < 36; ++t) H[t] += G.M[36 * i + t];
      for (int t = 0; t < 6; ++t) g[t] -= G.q[6 * i + t];
    }
    for (int64_t l = G.loff[i]; l < G.loff[i + 1]; ++l) {
      const int k = G.ll[l];
      for (int t = 0; t < 36; ++t) H[t] += G.M[36 * k + t];
      const double sg = G.en[2 * k + 1] == i ? 1.0 : -1.0;
      for (int t = 0; t < 6; ++t) g[t] += sg * G.q[6 * k + t];
    }
    for (int t = 0; t < 36; ++t) G.Hd[36 * i + t] = H[t];
    for (int t = 0; t < 6; ++t) {
      G.gn[6 * i + t] = g[t];
      if (i >= 1) gm = fmax(gm, fabs(g[t]));
    }
  }
  gmax = block_max(gm, s_red);
  return F;
}

// F at the trial poses G.Tt
__device__ double trial_cost(const PgoGraph& G, double phi, double* s_red) {
  double part = 0.0;
  for (int k = threadIdx.x; k < G.ne; k += kPgoThreads) {
    const int a = G.en[2 * k], b = G.en[2 * k + 1];
    double RC[9], tC[3], e[6], s;
    const double x = edge_residual(G.Tt + 16 * a, G.Tt + 16 * b, G.Z + 16 * k, G.w + 6 * k, RC, tC, e);
    part += edge_rho(x, k >= G.n - 1, phi, s);
  }
  return 0.5 * block_sum(part, s_red);
}

// out = (H + lam diag(H)) v over nodes 1 .. n-1 (v_0 = 0); returns v . out
__device__ double matvec(const PgoGraph& G, double lam, const double* v, double* out, double* s_red) {
  double part = 0.0;
  for (int i = 1 + threadIdx.x; i < G.n; i += kPgoThreads) {
    double vi[6], o[6];
    for (int t = 0; t < 6; ++t) vi[t] = v[6 * i + t];
    const double* H = G.Hd + 36 * i;
    for (int r = 0; r < 6; ++r) {
      double s = lam * H[7 * r] * vi[r];
      for (int c = 0; c < 6; ++c) s += H[6 * r + c] * vi[c];
      o[r] = s;
    }
    auto sub = [&](int k, int j) {            // o -= M_k v_j
      const double* Mk = G.M + 36 * k;
      for (int r = 0; r < 6; ++r) {
        double s = 0.0;
        for (int c = 0; c < 6; ++c) s += Mk[6 * r + c] * v[6 * j + c];
        o[r] -= s;
      }
    };
    if (i - 1 >= 1) sub(i - 1, i - 1);
    if (i + 1 <= G.n - 1) sub(i, i + 1);
    for (int64_t l = G.loff[i]; l < G.loff[i + 1]; ++l) {
      const int k = G.ll[l];
      const int j = G.en[2 * k] == i ? G.en[2 * k + 1] : G.en[2 * k];
      if (j != 0) sub(k, j);
    }
    for (int t = 0; t < 6; ++t) {
      out[6 * i + t] = o[t];
      part += vi[t] * o[t];
    }
  }
  return block_sum(part, s_red);
}

// The block Cholesky factor of the preconditioner at damping lam, in nested-dissection order.  Returns false (on
// every thread) at a pivot that is not positive.  s_fail[0] flags the segments, s_fail[1] the separator chain: each
// is read only after the barrier that follows its last write.
__device__ bool factor(const PgoGraph& G, double lam, double (*blk)[kPgoBlocks][36], int* s_fail) {
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_fail[0] = s_fail[1] = 0;
  __syncthreads();
  if (wp <= G.Q) {
    const int a = G.P[wp] + 1, b = G.P[wp + 1], sL = wp >= 1 ? G.P[wp] : -1, sR = wp + 1 <= G.Q ? G.P[wp + 1] : -1;
    double* sg = G.seg + kPgoSeg * wp;
    int iD = 0, iLp = 1, iF = 2, iT = 3;
    double* dL = blk[wp][4];
    w_fill(dL, 0.0, lane);
    if (sL >= 0 && a < b) w_load(blk[wp][iF], G.M + 36 * sL, 0.0, true, lane);    // A(sL, a) = -M_sL
    bool ok = true;
    for (int j = a; j < b; ++j) {
      double* D = blk[wp][iD];
      w_load(D, G.Hd + 36 * j, lam, false, lane);
      if (j > a) w_abt(D, blk[wp][iLp], blk[wp][iLp], -1.0, lane);
      if (!w_chol(D, lane)) { ok = false; break; }
      w_store(G.Ld + 36 * j, D, lane);
      double* F = blk[wp][iF];
      if (sL >= 0) {
        w_trsm(D, F, lane);                               // L(sL, j)
        w_store(G.Lk + 36 * j, F, lane);
        w_abt(dL, F, F, 1.0, lane);
      }
      if (j + 1 < G.n) {
        double* Tm = blk[wp][iT];
        w_load(Tm, G.M + 36 * j, 0.0, true, lane);       // A(j + 1, j) = -M_j
        w_trsm(D, Tm, lane);                              // L(j + 1, j)
        w_store(G.Ls + 36 * j, Tm, lane);
        if (sL >= 0) {
          w_fill(blk[wp][iLp], 0.0, lane);
          w_abt(blk[wp][iLp], F, Tm, -1.0, lane);         // the fill of (sL, j + 1)
          const int t = iF; iF = iLp; iLp = iT; iT = t;
        } else {
          const int t = iLp; iLp = iT; iT = t;
        }
      }
    }
    if (ok) {
      w_store(sg, dL, lane);
      if (a < b && sR >= 0) {
        w_fill(blk[wp][iT], 0.0, lane);
        w_abt(blk[wp][iT], blk[wp][iLp], blk[wp][iLp], 1.0, lane);
        w_store(sg + 36, blk[wp][iT], lane);
        if (sL >= 0) w_store(sg + 72, blk[wp][iF], lane);
      } else if (sL >= 0 && sR >= 0) {
        for (int e = lane; e < 36; e += 32) sg[72 + e] = -G.M[36 * sL + e];
      }
    } else if (lane == 0) {
      s_fail[0] = 1;
    }
  }
  __syncthreads();
  if (s_fail[0]) return false;
  if (wp == 0) {
    // the separator chain: S_qq = B_s - dRR(segment q - 1) - dLL(segment q), S(q, q-1) = fill(q - 1)^T
    double* D = blk[0][0];
    double* Lp = blk[0][1];
    double* Tm = blk[0][2];
    bool ok = true;
    for (int qq = 1; qq <= G.Q; ++qq) {
      const int s = G.P[qq];
      const bool left_live = G.P[qq - 1] + 1 < s, right_live = s + 1 < G.P[qq + 1];
      w_load(D, G.Hd + 36 * s, lam, false, lane);
      for (int e = lane; e < 36; e += 32) {
        double v = D[e];
        if (left_live) v -= G.seg[kPgoSeg * (qq - 1) + 36 + e];
        if (right_live) v -= G.seg[kPgoSeg * qq + e];
        D[e] = v;
      }
      __syncwarp();
      if (qq >= 2) {
        w_copy_t(Tm, G.seg + kPgoSeg * (qq - 1) + 72, lane);
        w_trsm(Lp, Tm, lane);
        w_store(G.Lk + 36 * s, Tm, lane);
        w_abt(D, Tm, Tm, -1.0, lane);
      }
      if (!w_chol(D, lane)) { ok = false; break; }
      w_store(G.Ld + 36 * s, D, lane);
      double* t = Lp; Lp = D; D = t;
    }
    if (!ok && lane == 0) s_fail[1] = 1;
  }
  __syncthreads();
  return s_fail[1] == 0;
}

// out = M^-1 v with the factor of `factor`
__device__ void apply(const PgoGraph& G, const double* v, double* out) {
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const bool writer = lane < 6;
  if (wp <= G.Q) {
    const int a = G.P[wp] + 1, b = G.P[wp + 1], sL = wp >= 1 ? G.P[wp] : -1, sR = wp + 1 <= G.Q ? G.P[wp + 1] : -1;
    double yp = 0.0, cL = 0.0, cR = 0.0;
    for (int j = a; j < b; ++j) {
      double t = vload(v, j, lane);
      if (j > a) t -= w_mv(G.Ls + 36 * (j - 1), yp, false, lane);
      yp = w_fwd(G.Ld + 36 * j, t, lane);
      if (writer) G.y[6 * j + lane] = yp;
      if (sL >= 0) cL += w_mv(G.Lk + 36 * j, yp, false, lane);
    }
    if (a < b && sR >= 0) cR = w_mv(G.Ls + 36 * (b - 1), yp, false, lane);
    if (writer) {
      G.seg[kPgoSeg * wp + 108 + lane] = cL;
      G.seg[kPgoSeg * wp + 114 + lane] = cR;
    }
  }
  __syncthreads();
  if (wp == 0) {
    double yp = 0.0;
    for (int qq = 1; qq <= G.Q; ++qq) {
      const int s = G.P[qq];
      double t = vload(v, s, lane);
      if (writer) t -= G.seg[kPgoSeg * (qq - 1) + 114 + lane] + G.seg[kPgoSeg * qq + 108 + lane];
      if (qq >= 2) t -= w_mv(G.Lk + 36 * s, yp, false, lane);
      yp = w_fwd(G.Ld + 36 * s, t, lane);
      if (writer) G.y[6 * s + lane] = yp;
    }
    double zn = 0.0;
    for (int qq = G.Q; qq >= 1; --qq) {
      const int s = G.P[qq];
      double t = vload(G.y, s, lane);
      if (qq < G.Q) t -= w_mv(G.Lk + 36 * G.P[qq + 1], zn, true, lane);
      zn = w_bwd(G.Ld + 36 * s, t, lane);
      if (writer) out[6 * s + lane] = zn;
    }
  }
  __syncthreads();
  if (wp <= G.Q) {
    const int a = G.P[wp] + 1, b = G.P[wp + 1], sL = wp >= 1 ? G.P[wp] : -1, sR = wp + 1 <= G.Q ? G.P[wp + 1] : -1;
    double zn = sR >= 0 ? vload(out, sR, lane) : 0.0;
    const double zl = sL >= 0 ? vload(out, sL, lane) : 0.0;
    for (int j = b - 1; j >= a; --j) {
      double t = vload(G.y, j, lane);
      if (j < b - 1 || sR >= 0) t -= w_mv(G.Ls + 36 * j, zn, true, lane);
      if (sL >= 0) t -= w_mv(G.Lk + 36 * j, zl, true, lane);
      zn = w_bwd(G.Ld + 36 * j, t, lane);
      if (writer) out[6 * j + lane] = zn;
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kPgoThreads) k_pgo_graphs(PgoArgs A) {
  __shared__ double s_red[kPgoWarps];
  __shared__ double s_blk[kPgoWarps][kPgoBlocks][36];
  __shared__ int s_fail[2];
  const int gi = blockIdx.x, tid = threadIdx.x;
  const ovn_pgo_params& prm = A.prm;
  PgoGraph G;
  G.n0 = A.node_off[gi];
  G.e0 = A.edge_off[gi];
  G.n = (int)(A.node_off[gi + 1] - G.n0);
  G.ne = (int)(A.edge_off[gi + 1] - G.e0);
  G.en = A.enodes + 2 * G.e0;
  G.loff = A.loop_off + G.n0;
  G.ll = A.loop_list;
  G.Z = A.Z + 16 * G.e0; G.w = A.wgt + 6 * G.e0;
  G.T = A.T + 16 * G.n0; G.Tt = A.Tt + 16 * G.n0;
  G.M = A.M + 36 * G.e0; G.q = A.q + 6 * G.e0; G.chi2 = A.chi2 + G.e0; G.scale = A.scale + G.e0;
  G.Hd = A.Hd + 36 * G.n0; G.gn = A.gn + 6 * G.n0;
  G.Ld = A.Ld + 36 * G.n0; G.Ls = A.Ls + 36 * G.n0; G.Lk = A.Lk + 36 * G.n0;
  G.x = A.x + 6 * G.n0; G.r = A.r + 6 * G.n0; G.z = A.z + 6 * G.n0; G.p = A.p + 6 * G.n0; G.Ap = A.Ap + 6 * G.n0;
  G.y = A.y + 6 * G.n0;
  G.seg = A.seg + (int64_t)kPgoSeg * kPgoWarps * gi;
  // separators every ceil((n - 1) / W) free nodes, never the last node
  const int m = G.n - 1, len = (m + kPgoWarps - 1) / kPgoWarps;
  G.Q = 0;
  G.P[0] = 0;
  for (int qq = 1; qq <= kPgoWarps && qq * len < G.n - 1; ++qq) G.P[++G.Q] = qq * len;
  G.P[G.Q + 1] = G.n;
  ovn_pgo_trial* trace = A.trace ? A.trace + (int64_t)gi * prm.max_iterations : nullptr;
  if (trace)
    for (int t = tid; t < prm.max_iterations; t += kPgoThreads)
      trace[t] = ovn_pgo_trial{CUDART_NAN, CUDART_NAN, -1, -1};

  double gmax;
  double F = linearize(G, prm.phi, s_red, gmax);
  const double F0 = F;
  double lam = prm.lambda0;
  int status = OVN_PGO_MAX_ITERATIONS, it = 0, accepted = 0, cg_total = 0;
  while (it < prm.max_iterations) {
    // ---- PCG on (H + lam D) x = -g over nodes 1 .. n-1 ----
    double part = 0.0;
    for (int i = 1 + tid; i < G.n; i += kPgoThreads)
      for (int t = 0; t < 6; ++t) {
        const double g = G.gn[6 * i + t];
        G.x[6 * i + t] = 0.0;
        G.r[6 * i + t] = -g;
        part += g * g;
      }
    const double gnorm = sqrt(block_sum(part, s_red));
    double rnorm = gnorm;
    int cg = 0;
    bool failed = false;
    if (!(rnorm <= prm.cg_tol * gnorm)) {
      failed = !factor(G, lam, s_blk, s_fail);
      if (!failed) {
        apply(G, G.r, G.z);
        part = 0.0;
        for (int i = 1 + tid; i < G.n; i += kPgoThreads)
          for (int t = 0; t < 6; ++t) {
            G.p[6 * i + t] = G.z[6 * i + t];
            part += G.r[6 * i + t] * G.z[6 * i + t];
          }
        double rz = block_sum(part, s_red);
        for (;;) {
          const double pAp = matvec(G, lam, G.p, G.Ap, s_red);
          if (!(pAp > 0.0)) { failed = true; break; }
          const double alpha = rz / pAp;
          part = 0.0;
          for (int i = 1 + tid; i < G.n; i += kPgoThreads)
            for (int t = 0; t < 6; ++t) {
              G.x[6 * i + t] += alpha * G.p[6 * i + t];
              const double rr = G.r[6 * i + t] - alpha * G.Ap[6 * i + t];
              G.r[6 * i + t] = rr;
              part += rr * rr;
            }
          rnorm = sqrt(block_sum(part, s_red));
          ++cg;
          if (rnorm <= prm.cg_tol * gnorm || cg >= prm.max_cg_iterations) break;
          apply(G, G.r, G.z);
          part = 0.0;
          for (int i = 1 + tid; i < G.n; i += kPgoThreads)
            for (int t = 0; t < 6; ++t) part += G.r[6 * i + t] * G.z[6 * i + t];
          const double rz_new = block_sum(part, s_red);
          const double beta = rz_new / rz;
          rz = rz_new;
          for (int i = 1 + tid; i < G.n; i += kPgoThreads)
            for (int t = 0; t < 6; ++t) G.p[6 * i + t] = G.z[6 * i + t] + beta * G.p[6 * i + t];
          __syncthreads();
        }
      }
    }
    ++it;
    cg_total += cg;
    if (failed) {
      if (tid == 0 && trace) trace[it - 1] = ovn_pgo_trial{CUDART_NAN, lam, 0, cg};
      status = OVN_PGO_FAILED;
      break;
    }
    // ---- the trial: T_i <- [R(omega) | v] T_i for nodes 1 .. n-1 ----
    double dmax = 0.0;
    for (int i = tid; i < G.n; i += kPgoThreads) {
      double Tn[16];
      for (int t = 0; t < 16; ++t) Tn[t] = G.T[16 * i + t];
      if (i >= 1) {
        double d[6];
        for (int t = 0; t < 6; ++t) {
          d[t] = G.x[6 * i + t];
          dmax = fmax(dmax, fabs(d[t]));
        }
        left_update(d, Tn);
      }
      for (int t = 0; t < 16; ++t) G.Tt[16 * i + t] = Tn[t];
    }
    dmax = block_max(dmax, s_red);
    const double Ft = trial_cost(G, prm.phi, s_red);
    const bool ok = Ft < F;
    if (tid == 0 && trace) trace[it - 1] = ovn_pgo_trial{Ft, lam, ok ? 1 : 0, cg};
    if (ok) {
      for (int i = tid; i < G.n; i += kPgoThreads)
        for (int t = 0; t < 16; ++t) G.T[16 * i + t] = G.Tt[16 * i + t];
      __syncthreads();
      const double Fold = F;
      lam = fmax(lam / 10.0, prm.lambda_min);
      ++accepted;
      F = linearize(G, prm.phi, s_red, gmax);
      if (Fold - F <= prm.rel_cost_tol * Fold || dmax <= prm.step_tol) {
        status = OVN_PGO_CONVERGED;
        break;
      }
    } else {
      lam = lam * 10.0;
      if (dmax <= prm.step_tol) {
        status = OVN_PGO_CONVERGED;
        break;
      }
      if (lam > prm.lambda_max) {
        status = OVN_PGO_STALLED;
        break;
      }
    }
  }
  if (tid == 0) {
    ovn_pgo_result& r = A.res[gi];
    r.initial_cost = F0;
    r.final_cost = F;
    r.lambda = lam;
    r.max_gradient = gmax;
    r.status = status;
    r.iterations = it;
    r.accepted = accepted;
    r.cg_iterations = cg_total;
  }
}

// ---- host side: the node -> loop-edge CSR, the workspace, one launch and the copies --------------------------
static size_t align16(size_t b) { return (b + 15) & ~size_t(15); }

int pgo_graphs(ovn_handle* h, int n_graphs, const int64_t* node_off, const int64_t* edge_off, const double* poses,
               const int32_t* edge_nodes, const double* edge_pose, const double* edge_weight,
               const ovn_pgo_params& prm, double* out_poses, ovn_pgo_result* out_result, double* out_chi2,
               double* out_scale, double* out_gradient, ovn_pgo_trial* out_trace, cudaStream_t s) {
  const int64_t N = node_off[n_graphs], E = edge_off[n_graphs];
  // node -> loop edges in edge order (counting sort), global node offsets, local edge indices
  std::vector<int64_t> loop_off(N + 1, 0);
  for (int g = 0; g < n_graphs; ++g) {
    const int64_t n = node_off[g + 1] - node_off[g];
    for (int64_t k = edge_off[g] + n - 1; k < edge_off[g + 1]; ++k) {
      ++loop_off[node_off[g] + edge_nodes[2 * k] + 1];
      ++loop_off[node_off[g] + edge_nodes[2 * k + 1] + 1];
    }
  }
  for (int64_t i = 0; i < N; ++i) loop_off[i + 1] += loop_off[i];
  std::vector<int32_t> loop_list(std::max<int64_t>(loop_off[N], 1));
  {
    std::vector<int64_t> fill(loop_off.begin(), loop_off.end() - 1);
    for (int g = 0; g < n_graphs; ++g) {
      const int64_t n = node_off[g + 1] - node_off[g];
      for (int64_t k = edge_off[g] + n - 1; k < edge_off[g + 1]; ++k)
        for (int t = 0; t < 2; ++t) loop_list[fill[node_off[g] + edge_nodes[2 * k + t]]++] = (int32_t)(k - edge_off[g]);
    }
  }
  // one block: inputs, then the workspace
  struct Part { size_t off, bytes; };
  size_t total = 0;
  auto part = [&](size_t bytes) { Part p{total, bytes}; total += align16(bytes); return p; };
  const size_t D = sizeof(double);
  const Part p_noff = part((n_graphs + 1) * sizeof(int64_t)), p_eoff = part((n_graphs + 1) * sizeof(int64_t));
  const Part p_en = part(E * 2 * sizeof(int32_t)), p_loff = part((N + 1) * sizeof(int64_t));
  const Part p_ll = part(loop_list.size() * sizeof(int32_t));
  const Part p_Z = part(E * 16 * D), p_w = part(E * 6 * D), p_T = part(N * 16 * D), p_Tt = part(N * 16 * D);
  const Part p_M = part(E * 36 * D), p_q = part(E * 6 * D), p_chi2 = part(E * D), p_scale = part(E * D);
  const Part p_Hd = part(N * 36 * D), p_gn = part(N * 6 * D);
  const Part p_Ld = part(N * 36 * D), p_Ls = part(N * 36 * D), p_Lk = part(N * 36 * D);
  Part p_vec[6];
  for (int v = 0; v < 6; ++v) p_vec[v] = part(N * 6 * D);
  const Part p_seg = part((size_t)n_graphs * kPgoWarps * kPgoSeg * D);
  const Part p_res = part(n_graphs * sizeof(ovn_pgo_result));
  const Part p_tr = part((size_t)n_graphs * std::max(prm.max_iterations, 1) * sizeof(ovn_pgo_trial));
  const int rc = h->d_pgo.ensure(h, total);
  if (rc != OVN_OK) return rc;
  uint8_t* base = h->d_pgo;
  auto at = [&](const Part& p) { return (void*)(base + p.off); };
  auto up = [&](const Part& p, const void* src) {
    return cudaMemcpyAsync(at(p), src, p.bytes, cudaMemcpyHostToDevice, s);
  };
  OVN_CUDA(h, up(p_noff, node_off));
  OVN_CUDA(h, up(p_eoff, edge_off));
  OVN_CUDA(h, up(p_en, edge_nodes));
  OVN_CUDA(h, up(p_loff, loop_off.data()));
  OVN_CUDA(h, up(p_ll, loop_list.data()));
  OVN_CUDA(h, up(p_Z, edge_pose));
  OVN_CUDA(h, up(p_w, edge_weight));
  OVN_CUDA(h, up(p_T, poses));
  PgoArgs a;
  a.node_off = (const int64_t*)at(p_noff); a.edge_off = (const int64_t*)at(p_eoff);
  a.enodes = (const int32_t*)at(p_en); a.loop_off = (const int64_t*)at(p_loff); a.loop_list = (const int32_t*)at(p_ll);
  a.Z = (const double*)at(p_Z); a.wgt = (const double*)at(p_w);
  a.T = (double*)at(p_T); a.Tt = (double*)at(p_Tt);
  a.M = (double*)at(p_M); a.q = (double*)at(p_q); a.chi2 = (double*)at(p_chi2); a.scale = (double*)at(p_scale);
  a.Hd = (double*)at(p_Hd); a.gn = (double*)at(p_gn);
  a.Ld = (double*)at(p_Ld); a.Ls = (double*)at(p_Ls); a.Lk = (double*)at(p_Lk);
  double** vecs[6] = {&a.x, &a.r, &a.z, &a.p, &a.Ap, &a.y};
  for (int v = 0; v < 6; ++v) *vecs[v] = (double*)at(p_vec[v]);
  a.seg = (double*)at(p_seg);
  a.res = (ovn_pgo_result*)at(p_res);
  a.trace = out_trace && prm.max_iterations > 0 ? (ovn_pgo_trial*)at(p_tr) : nullptr;
  a.prm = prm;
  prof_mark(h, PROF_PGO, s);
  k_pgo_graphs<<<n_graphs, kPgoThreads, 0, s>>>(a);
  OVN_LAUNCH_CHECK(h);
  prof_mark(h, PROF_PGO, s);
  auto down = [&](void* dst, const Part& p) { return cudaMemcpyAsync(dst, at(p), p.bytes, cudaMemcpyDeviceToHost, s); };
  OVN_CUDA(h, down(out_poses, p_T));
  OVN_CUDA(h, down(out_result, p_res));
  OVN_CUDA(h, down(out_chi2, p_chi2));
  OVN_CUDA(h, down(out_scale, p_scale));
  if (out_gradient) OVN_CUDA(h, down(out_gradient, p_gn));
  if (a.trace) OVN_CUDA(h, down(out_trace, p_tr));
  OVN_CUDA(h, cudaStreamSynchronize(s));
  const Part* arrays[15] = {&p_T, &p_Tt, &p_M, &p_q, &p_Hd, &p_gn, &p_Ld, &p_Ls, &p_Lk,
                            &p_vec[0], &p_vec[1], &p_vec[2], &p_vec[3], &p_vec[4], &p_vec[5]};
  for (int v = 0; v < 15; ++v) h->pgo_array_off[v] = arrays[v]->off;
  h->pgo_node_off.assign(node_off, node_off + n_graphs + 1);
  h->pgo_edge_off.assign(edge_off, edge_off + n_graphs + 1);
  return OVN_OK;
}

int pgo_copy_workspace(ovn_handle* h, int array, int graph, double* h_out) {
  // doubles per node or per edge of each ovn_pgo_array, and whether it is per edge
  static const int width[15] = {16, 16, 36, 6, 36, 6, 36, 36, 36, 6, 6, 6, 6, 6, 6};
  const bool per_edge = array == OVN_PGO_M || array == OVN_PGO_Q;
  const std::vector<int64_t>& off = per_edge ? h->pgo_edge_off : h->pgo_node_off;
  const size_t first = (size_t)off[graph] * width[array], count = (size_t)(off[graph + 1] - off[graph]) * width[array];
  const double* src = reinterpret_cast<const double*>(h->d_pgo.get() + h->pgo_array_off[array]) + first;
  OVN_CUDA(h, cudaMemcpy(h_out, src, count * sizeof(double), cudaMemcpyDeviceToHost));
  return OVN_OK;
}

}  // namespace ovn
