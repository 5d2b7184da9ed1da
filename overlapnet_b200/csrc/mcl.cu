// mcl.cu -- the particle filter of overlap-based Monte Carlo localization (ovn_mcl_*, DESIGN.md sections 4 and 7).
//
// Particles are structure-of-arrays float64 (x, y, theta, log-weight) in one of two buffers; systematic resampling
// writes the other one.  Every random number comes from Philox4x32-10 keyed by the 64-bit seed with the counter
// (particle, step, stream, block), so a particle's draws do not depend on the launch geometry.  Every reduction
// (max, log-sum-exp, ESS, the estimate, the prefix sum) runs in an order fixed by N alone: the same seed, map,
// observations and N give bit-identical particles on every run and handle.  All kernels are memory-bound.
#include "common.cuh"
#include <algorithm>
#include <math.h>

namespace ovn {

constexpr int kMclThreads = 256;
constexpr int kMclRedBlocks = 1024;             // the most per-block partials of one reduction
constexpr int kMclScanPer = 8;                  // prefix sum: consecutive weights per thread
constexpr int kMclScanTile = kMclThreads * kMclScanPer;
constexpr int kMclCompactThreads = 1024;
constexpr double kPi = 3.141592653589793;
constexpr double kTwoPi = 6.283185307179586;
enum McStream : uint32_t { kStreamMotion = 0, kStreamInit = 1, kStreamResample = 2 };

// ---- Philox4x32-10 and the conversions (restated bit for bit by oracle/mcl.py) ------------------------------
static __device__ __forceinline__ uint4 philox(uint64_t seed, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c0, hi0 = __umulhi(0xD2511F53u, c0);
    const uint32_t lo1 = 0xCD9E8D57u * c2, hi1 = __umulhi(0xCD9E8D57u, c2);
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

// 53 bits of two words, k = (a >> 5) 2^26 + (b >> 6); u = k 2^-53, with k = 0 read as 1/2: u in (0, 1), exact
static __device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
  const uint64_t k = ((uint64_t)(a >> 5) << 26) | (uint64_t)(b >> 6);
  return (k == 0 ? 0.5 : (double)k) * 0x1p-53;
}

// Box-Muller on the four words of one block: n0 = r cos(2 pi u_b), n1 = r sin(2 pi u_b), r = sqrt(-2 ln u_a)
static __device__ __forceinline__ void box_muller(uint4 w, double& n0, double& n1) {
  const double r = sqrt(-2.0 * log(u53(w.x, w.y)));
  const double a = kTwoPi * u53(w.z, w.w);
  n0 = r * cos(a);
  n1 = r * sin(a);
}

// an angle into (-pi, pi]; IEEE additions and fmod only, so the oracle reproduces it exactly
static __device__ __forceinline__ double wrap_pi(double a) {
  double r = fmod(__dadd_rn(a, kPi), kTwoPi);
  if (r <= 0.0) r = __dadd_rn(r, kTwoPi);
  return __dadd_rn(r, -kPi);
}

// the keyframe under (x, y), -1 outside the raster (NaN included); float64, no contraction
static __device__ __forceinline__ int raster_lookup(double x, double y, const McMap& m, const int32_t* raster) {
  const double fy = floor(__ddiv_rn(__dadd_rn(y, -m.y0), m.cell));
  const double fx = floor(__ddiv_rn(__dadd_rn(x, -m.x0), m.cell));
  if (!(fy >= 0.0 && fy < (double)m.rows && fx >= 0.0 && fx < (double)m.cols)) return -1;
  return raster[(int64_t)fy * m.cols + (int64_t)fx];
}

static int red_blocks(int n) { return std::max(1, std::min((n + kMclThreads - 1) / kMclThreads, kMclRedBlocks)); }

// ---- initialisation ---------------------------------------------------------------------------------------
static __global__ void __launch_bounds__(kMclThreads)
k_mcl_init(McParticles p, int n, int mode, uint64_t seed, const double* __restrict__ kf, int K, double radius,
           double px, double py, double pt, double sx, double sy, double st) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint4 b0 = philox(seed, (uint32_t)i, 0u, kStreamInit, 0u);
  const uint4 b1 = philox(seed, (uint32_t)i, 0u, kStreamInit, 1u);
  double x, y, th;
  if (mode == OVN_MCL_INIT_GLOBAL) {
    // keyframe floor(u K), a point uniform in the disk of `radius` around it, theta uniform
    const int k = min((int)(u53(b0.x, b0.y) * (double)K), K - 1);
    const double r = radius * sqrt(u53(b0.z, b0.w));
    const double phi = kTwoPi * u53(b1.x, b1.y);
    x = kf[3 * k] + r * cos(phi);
    y = kf[3 * k + 1] + r * sin(phi);
    th = kPi - kTwoPi * u53(b1.z, b1.w);
  } else {
    double n0, n1, n2, unused;
    box_muller(b0, n0, n1);
    box_muller(b1, n2, unused);
    x = px + sx * n0;
    y = py + sy * n1;
    th = wrap_pi(pt + st * n2);
  }
  p.x[i] = x;
  p.y[i] = y;
  p.th[i] = th;
  p.lw[i] = -log((double)n);
}

// ---- motion, lookup and the touched flags -------------------------------------------------------------------
static __global__ void __launch_bounds__(kMclThreads)
k_mcl_motion(McParticles p, int n, uint64_t seed, uint32_t step, double dx, double dy, double dth, double sx,
             double sy, double st, McMap m, const int32_t* __restrict__ raster, int32_t* __restrict__ kidx,
             int32_t* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double n0, n1, n2, unused;
  box_muller(philox(seed, (uint32_t)i, step, kStreamMotion, 0u), n0, n1);
  box_muller(philox(seed, (uint32_t)i, step, kStreamMotion, 1u), n2, unused);
  const double x = p.x[i], y = p.y[i], th = p.th[i];
  const double c = cos(th), s = sin(th);
  const double ex = dx + sx * n0, ey = dy + sy * n1;
  const double x2 = x + c * ex - s * ey;
  const double y2 = y + s * ex + c * ey;
  p.x[i] = x2;
  p.y[i] = y2;
  p.th[i] = wrap_pi(th + dth + st * n2);
  const int k = raster_lookup(x2, y2, m, raster);
  kidx[i] = k;
  if (k >= 0) flags[k] = 1;                       // every writer stores the same value
}

// One block lists the flagged keyframes in ascending order: touched[j] = the j-th, slot[k] = its position or -1,
// *count = their number.
static __global__ void __launch_bounds__(kMclCompactThreads)
k_mcl_compact(const int32_t* __restrict__ flags, int K, int32_t* __restrict__ touched, int32_t* __restrict__ slot,
              int32_t* __restrict__ count) {
  __shared__ int warp_sum[kMclCompactThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int base = 0;
  for (int k0 = 0; k0 < K; k0 += kMclCompactThreads) {
    const int k = k0 + threadIdx.x;
    const int f = (k < K && flags[k]) ? 1 : 0;
    const unsigned ballot = __ballot_sync(0xffffffffu, f);
    const int in_warp = __popc(ballot & ((1u << lane) - 1u));
    if (lane == 0) warp_sum[warp] = __popc(ballot);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < kMclCompactThreads / 32; ++w) {
      before += w < warp ? warp_sum[w] : 0;
      total += warp_sum[w];
    }
    if (k < K) {
      const int pos = base + before + in_warp;
      slot[k] = f ? pos : -1;
      if (f) touched[pos] = k;
    }
    base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = base;
}

// ---- fixed-order reductions ---------------------------------------------------------------------------------
// Each block reduces its grid-stride share (the grid depends on n alone) to one partial per value; k_mcl_final
// reduces the partials with one fixed tree.  V values per element.
template <int V, bool Max>
static __device__ __forceinline__ void block_reduce(double (&v)[V], double* __restrict__ partial) {
  __shared__ double sm[V][kMclThreads];
#pragma unroll
  for (int j = 0; j < V; ++j) sm[j][threadIdx.x] = v[j];
  __syncthreads();
  for (int s = kMclThreads / 2; s >= 1; s >>= 1) {
    if (threadIdx.x < s) {
#pragma unroll
      for (int j = 0; j < V; ++j)
        sm[j][threadIdx.x] = Max ? fmax(sm[j][threadIdx.x], sm[j][threadIdx.x + s]) : sm[j][threadIdx.x] + sm[j][threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int j = 0; j < V; ++j) partial[blockIdx.x * kMcPartialStride + j] = sm[j][0];
  }
}

// log l_i = -1/2 ((1 - O) / s_o)^2 - 1/2 (D / s_psi)^2 into ll_out; per-block max of the updated log-weights
// lw + log l, and whether a touched overlap is not finite.  The log-weights themselves are left as they are: the
// update writes them in k_mcl_normalize, once k_mcl_final has accepted the observations.
static __global__ void __launch_bounds__(kMclThreads)
k_mcl_loglik(McParticles p, int n, const int32_t* __restrict__ kidx, const int32_t* __restrict__ slot,
             const double* __restrict__ kf, const float* __restrict__ ov, const int32_t* __restrict__ yaw, int Wf,
             double s_o, double s_psi, double* __restrict__ ll_out, double* __restrict__ partial) {
  double v[2] = {-INFINITY, 0.0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int k = kidx[i];
    double O = 0.0, D = kPi;
    if (k >= 0) {
      const int j = slot[k];
      O = (double)ov[j];
      const int64_t a = 180 - (int64_t)yaw[j];                              // the heads return 180 - argmax
      const double psi = wrap_pi(__dadd_rn(p.th[i], -kf[3 * k + 2]));
      // gt.yaw_bin: int(-(psi / pi) * Wf // 2 + Wf // 2), then mod Wf
      const double e = floor(__dmul_rn(__dmul_rn(-__ddiv_rn(psi, kPi), (double)Wf), 0.5)) + (double)(Wf / 2);
      int64_t d = ((a - (int64_t)e) % Wf + Wf) % Wf;
      d = min(d, (int64_t)Wf - d);
      D = __dmul_rn((double)d, kTwoPi / (double)Wf);
      if (!isfinite(O)) v[1] = 1.0;
    }
    const double t1 = (1.0 - O) / s_o, t2 = D / s_psi;
    const double ll = -0.5 * (t1 * t1) - 0.5 * (t2 * t2);
    ll_out[i] = ll;
    v[0] = fmax(v[0], p.lw[i] + ll);
  }
  block_reduce<2, true>(v, partial);
}

// per-block sums of exp(lw + ll - m), m = scal[kScMax]
static __global__ void __launch_bounds__(kMclThreads)
k_mcl_expsum(const double* __restrict__ lw, const double* __restrict__ ll, int n, const double* __restrict__ scal,
             double* __restrict__ partial) {
  if (scal[kScRefused] != 0.0) return;
  const double m = scal[kScMax];
  double v[1] = {0.0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    v[0] += exp(lw[i] + ll[i] - m);
  block_reduce<1, false>(v, partial);
}

// lw = lw + ll - (m + log s); w = exp(lw); per-block sums of w, w^2, w x, w y, w sin theta, w cos theta
static __global__ void __launch_bounds__(kMclThreads)
k_mcl_normalize(McParticles p, const double* __restrict__ ll, int n, const double* __restrict__ scal,
                double* __restrict__ w_out, double* __restrict__ partial) {
  if (scal[kScRefused] != 0.0) return;
  const double L = scal[kScMax] + log(scal[kScExpSum]);
  double v[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double lw = (p.lw[i] + ll[i]) - L;
    const double w = exp(lw);
    const double th = p.th[i];
    p.lw[i] = lw;
    w_out[i] = w;
    v[0] += w;
    v[1] += w * w;
    v[2] += w * p.x[i];
    v[3] += w * p.y[i];
    v[4] += w * sin(th);
    v[5] += w * cos(th);
  }
  block_reduce<6, false>(v, partial);
}

// One block of kMclRedBlocks threads reduces the partials with a fixed tree, then finishes the stage:
// mode 0: scal[kScMax] = max, scal[kScRefused] = 1 when a touched overlap is not finite, else 2 when no updated
// log-weight is finite (the max is -inf), else 0, and no resampling until mode 2 decides; mode 1: scal[kScExpSum] =
// sum; mode 2: the six sums, the ESS, the estimate, the resampling decision and its offset u0.  Modes 1 and 2 do
// nothing once mode 0 has refused the update.
static __global__ void __launch_bounds__(kMclRedBlocks)
k_mcl_final(const double* __restrict__ partial, int n_parts, int mode, int n, double rho, uint64_t seed,
            uint32_t step, double* __restrict__ scal) {
  constexpr int V = 6;
  __shared__ double sm[V][kMclRedBlocks];
  if (mode != 0 && scal[kScRefused] != 0.0) return;
  const int nv = mode == 2 ? V : mode == 0 ? 2 : 1;
  const bool is_max = mode == 0;
  for (int j = 0; j < nv; ++j)
    sm[j][threadIdx.x] = threadIdx.x < n_parts ? partial[threadIdx.x * kMcPartialStride + j] : (is_max ? -INFINITY : 0.0);
  __syncthreads();
  for (int s = kMclRedBlocks / 2; s >= 1; s >>= 1) {
    if (threadIdx.x < s)
      for (int j = 0; j < nv; ++j)
        sm[j][threadIdx.x] = is_max ? fmax(sm[j][threadIdx.x], sm[j][threadIdx.x + s]) : sm[j][threadIdx.x] + sm[j][threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  if (mode == 0) {
    scal[kScMax] = sm[0][0];
    scal[kScRefused] = sm[1][0] != 0.0 ? 1.0 : sm[0][0] == -INFINITY ? 2.0 : 0.0;
    scal[kScResample] = 0.0;
  } else if (mode == 1) {
    scal[kScExpSum] = sm[0][0];
  } else {
    const double sw = sm[0][0];
    const double ess = 1.0 / sm[1][0];
    scal[kScEss] = ess;
    scal[kScX] = sm[2][0] / sw;
    scal[kScY] = sm[3][0] / sw;
    scal[kScTheta] = atan2(sm[4][0], sm[5][0]);
    scal[kScResample] = ess < rho * (double)n ? 1.0 : 0.0;
    const uint4 w = philox(seed, 0u, step, kStreamResample, 0u);
    scal[kScU0] = u53(w.x, w.y);
  }
}

// ---- systematic resampling ----------------------------------------------------------------------------------
// The inclusive prefix sum C of the weights in tiles of kMclScanTile: thread t of tile b sums its kMclScanPer
// consecutive weights in order; a Hillis-Steele scan over the threads; tile totals scanned in order by one thread.
static __device__ __forceinline__ double thread_prefix(const double* __restrict__ w, int n, double (&own)[kMclScanPer],
                                                       double& excl) {
  __shared__ double sm[2][kMclThreads];
  const int64_t first = (int64_t)blockIdx.x * kMclScanTile + (int64_t)threadIdx.x * kMclScanPer;
  double t = 0.0;
#pragma unroll
  for (int j = 0; j < kMclScanPer; ++j) {
    own[j] = first + j < n ? w[first + j] : 0.0;
    t += own[j];
  }
  int buf = 0;
  sm[0][threadIdx.x] = t;
  __syncthreads();
  for (int s = 1; s < kMclThreads; s <<= 1) {
    const double v = sm[buf][threadIdx.x] + (threadIdx.x >= s ? sm[buf][threadIdx.x - s] : 0.0);
    sm[buf ^ 1][threadIdx.x] = threadIdx.x >= s ? v : sm[buf][threadIdx.x];
    buf ^= 1;
    __syncthreads();
  }
  excl = threadIdx.x ? sm[buf][threadIdx.x - 1] : 0.0;
  return sm[buf][kMclThreads - 1];                 // the tile total
}

static __global__ void __launch_bounds__(kMclThreads)
k_mcl_tile_sums(const double* __restrict__ w, int n, const double* __restrict__ scal, double* __restrict__ tiles) {
  if (scal[kScResample] == 0.0) return;
  double own[kMclScanPer], excl;
  const double total = thread_prefix(w, n, own, excl);
  if (threadIdx.x == 0) tiles[blockIdx.x] = total;
}

static __global__ void k_mcl_tile_offsets(double* __restrict__ tiles, int n_tiles, const double* __restrict__ scal) {
  if (scal[kScResample] == 0.0 || threadIdx.x != 0) return;
  double run = 0.0;
  for (int b = 0; b < n_tiles; ++b) {                // exclusive, in tile order
    const double t = tiles[b];
    tiles[b] = run;
    run += t;
  }
}

static __global__ void __launch_bounds__(kMclThreads)
k_mcl_prefix(const double* __restrict__ w, int n, const double* __restrict__ scal, const double* __restrict__ tiles,
             double* __restrict__ cdf) {
  if (scal[kScResample] == 0.0) return;
  double own[kMclScanPer], excl;
  thread_prefix(w, n, own, excl);
  double run = tiles[blockIdx.x] + excl;
  const int64_t first = (int64_t)blockIdx.x * kMclScanTile + (int64_t)threadIdx.x * kMclScanPer;
#pragma unroll
  for (int j = 0; j < kMclScanPer; ++j) {
    run += own[j];
    if (first + j < n) cdf[first + j] = run;
  }
}

// ancestor of j: the least i with C_i > t_j = (j + u0) / n, clamped to n - 1; the new set has log-weights -log n
static __global__ void __launch_bounds__(kMclThreads)
k_mcl_resample(const double* __restrict__ cdf, int n, const double* __restrict__ scal, McParticles src,
               McParticles dst, int32_t* __restrict__ anc) {
  if (scal[kScResample] == 0.0) return;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const double t = ((double)j + scal[kScU0]) / (double)n;
  int lo = 0, hi = n - 1;                          // C_hi > t or hi = n - 1
  while (lo < hi) {
    const int mid = lo + (hi - lo) / 2;
    if (cdf[mid] > t) hi = mid;
    else lo = mid + 1;
  }
  anc[j] = lo;
  dst.x[j] = src.x[lo];
  dst.y[j] = src.y[lo];
  dst.th[j] = src.th[lo];
  dst.lw[j] = -log((double)n);
}

// ---- host side ----------------------------------------------------------------------------------------------
static McParticles particles(ovn_handle* h, int b) {
  double* base = h->mcl.part[b].get();
  const int64_t c = h->mcl.cap;
  return McParticles{base, base + c, base + 2 * c, base + 3 * c};
}

int mcl_alloc(ovn_handle* h, int n) {
  McState& m = h->mcl;
  if (n > m.cap) {
    for (auto& b : m.part) {
      b = {};
      int rc = b.ensure(h, (size_t)n * 4 * sizeof(double));
      if (rc != OVN_OK) { m.cap = 0; return rc; }
    }
    m.kidx = {}; m.ll = {}; m.w = {}; m.cdf = {}; m.anc = {}; m.tiles = {};
    int rc;
    if ((rc = m.kidx.ensure(h, (size_t)n * sizeof(int32_t))) != OVN_OK ||
        (rc = m.ll.ensure(h, (size_t)n * sizeof(double))) != OVN_OK ||
        (rc = m.w.ensure(h, (size_t)n * sizeof(double))) != OVN_OK ||
        (rc = m.cdf.ensure(h, (size_t)n * sizeof(double))) != OVN_OK ||
        (rc = m.anc.ensure(h, (size_t)n * sizeof(int32_t))) != OVN_OK ||
        (rc = m.tiles.ensure(h, (size_t)((n + kMclScanTile - 1) / kMclScanTile) * sizeof(double))) != OVN_OK) {
      m.cap = 0;
      return rc;
    }
    m.cap = n;
  }
  int rc;
  if ((rc = m.partial.ensure(h, (size_t)kMclRedBlocks * kMcPartialStride * sizeof(double))) != OVN_OK) return rc;
  if ((rc = m.scal.ensure(h, kScCount * sizeof(double))) != OVN_OK) return rc;
  if ((rc = m.host.ensure(h, kScCount * sizeof(double))) != OVN_OK) return rc;
  return OVN_OK;
}

int mcl_init(ovn_handle* h, int mode, int n, uint64_t seed, const double* pose, const double* sigma, double radius,
             cudaStream_t s) {
  McState& m = h->mcl;
  int rc = mcl_alloc(h, n);
  if (rc != OVN_OK) return rc;
  const double z[3] = {0.0, 0.0, 0.0};
  if (!pose) pose = z;
  if (!sigma) sigma = z;
  k_mcl_init<<<(n + kMclThreads - 1) / kMclThreads, kMclThreads, 0, s>>>(
      particles(h, 0), n, mode, seed, m.kf, m.map.K, radius, pose[0], pose[1], pose[2], sigma[0], sigma[1], sigma[2]);
  OVN_LAUNCH_CHECK(h);
  m.n = n;
  m.cur = 0;
  m.seed = seed;
  m.step = 0;
  m.pending = -1;
  m.stages = 0;
  return OVN_OK;
}

int mcl_predict(ovn_handle* h, const double* odom, const double* sigma, int32_t* d_touched, int32_t* n_touched,
                cudaStream_t s) {
  McState& m = h->mcl;
  const int K = m.map.K;
  m.step += 1;
  OVN_CUDA(h, cudaMemsetAsync(m.flags, 0, (size_t)K * sizeof(int32_t), s));
  k_mcl_motion<<<(m.n + kMclThreads - 1) / kMclThreads, kMclThreads, 0, s>>>(
      particles(h, m.cur), m.n, m.seed, (uint32_t)m.step, odom[0], odom[1], odom[2], sigma[0], sigma[1], sigma[2],
      m.map, m.raster, m.kidx, m.flags);
  OVN_LAUNCH_CHECK(h);
  int32_t* d_count = reinterpret_cast<int32_t*>(m.scal.get() + kScTouched);
  k_mcl_compact<<<1, kMclCompactThreads, 0, s>>>(m.flags, K, d_touched, m.slot, d_count);
  OVN_LAUNCH_CHECK(h);
  int32_t* h_count = reinterpret_cast<int32_t*>(m.host.get() + kScTouched);
  OVN_CUDA(h, cudaMemcpyAsync(h_count, d_count, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  OVN_CUDA(h, cudaStreamSynchronize(s));
  *n_touched = *h_count;
  m.pending = *h_count;
  m.pred_buf = m.cur;
  m.stages = kMcHeldPredict;
  return OVN_OK;
}

int mcl_update(ovn_handle* h, const float* d_ov, const int32_t* d_yaw, double s_o, double s_psi, double rho,
               ovn_mcl_estimate* est, cudaStream_t s) {
  McState& m = h->mcl;
  const int n = m.n, G = red_blocks(n), n_tiles = (n + kMclScanTile - 1) / kMclScanTile;
  const McParticles p = particles(h, m.cur);
  double* scal = m.scal;
  k_mcl_loglik<<<G, kMclThreads, 0, s>>>(p, n, m.kidx, m.slot, m.kf, d_ov, d_yaw, h->cfg.leg_output_width, s_o, s_psi,
                                         m.ll, m.partial);
  OVN_LAUNCH_CHECK(h);
  k_mcl_final<<<1, kMclRedBlocks, 0, s>>>(m.partial, G, 0, n, rho, m.seed, (uint32_t)m.step, scal);
  OVN_LAUNCH_CHECK(h);
  k_mcl_expsum<<<G, kMclThreads, 0, s>>>(p.lw, m.ll, n, scal, m.partial);
  OVN_LAUNCH_CHECK(h);
  k_mcl_final<<<1, kMclRedBlocks, 0, s>>>(m.partial, G, 1, n, rho, m.seed, (uint32_t)m.step, scal);
  OVN_LAUNCH_CHECK(h);
  k_mcl_normalize<<<G, kMclThreads, 0, s>>>(p, m.ll, n, scal, m.w, m.partial);
  OVN_LAUNCH_CHECK(h);
  k_mcl_final<<<1, kMclRedBlocks, 0, s>>>(m.partial, G, 2, n, rho, m.seed, (uint32_t)m.step, scal);
  OVN_LAUNCH_CHECK(h);
  // the resampling kernels read the decision on the device and return at once when there is none (k_mcl_final
  // clears it when it refuses the update)
  k_mcl_tile_sums<<<n_tiles, kMclThreads, 0, s>>>(m.w, n, scal, m.tiles);
  OVN_LAUNCH_CHECK(h);
  k_mcl_tile_offsets<<<1, 32, 0, s>>>(m.tiles, n_tiles, scal);
  OVN_LAUNCH_CHECK(h);
  k_mcl_prefix<<<n_tiles, kMclThreads, 0, s>>>(m.w, n, scal, m.tiles, m.cdf);
  OVN_LAUNCH_CHECK(h);
  k_mcl_resample<<<(n + kMclThreads - 1) / kMclThreads, kMclThreads, 0, s>>>(m.cdf, n, scal, p, particles(h, m.cur ^ 1),
                                                                             m.anc);
  OVN_LAUNCH_CHECK(h);
  double* hs = m.host.get();
  OVN_CUDA(h, cudaMemcpyAsync(hs, scal, kScTouched * sizeof(double), cudaMemcpyDeviceToHost, s));
  OVN_CUDA(h, cudaStreamSynchronize(s));
  // a refused update has written nothing to the particle set: the predict still awaits its update
  if (hs[kScRefused] == 1.0)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_mcl_update: an observed overlap is not finite; the particles are unchanged");
  if (hs[kScRefused] != 0.0)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG,
                "ovn_mcl_update: no particle has a finite log-weight after the update; the particles are unchanged");
  est->x = hs[kScX];
  est->y = hs[kScY];
  est->theta = hs[kScTheta];
  est->ess = hs[kScEss];
  est->n_touched = m.pending;
  est->resampled = hs[kScResample] != 0.0;
  est->step = m.step;
  m.pending = -1;
  m.stages |= kMcHeldUpdate;
  if (est->resampled) {
    m.cur ^= 1;
    m.stages |= kMcHeldResample;
  }
  return OVN_OK;
}

int mcl_copy_particles(ovn_handle* h, double* d_out, cudaStream_t s) {
  McState& m = h->mcl;
  const McParticles p = particles(h, m.cur);
  const double* src[4] = {p.x, p.y, p.th, p.lw};
  for (int j = 0; j < 4; ++j)
    OVN_CUDA(h, cudaMemcpyAsync(d_out + (size_t)j * m.n, src[j], (size_t)m.n * sizeof(double), cudaMemcpyDeviceToDevice, s));
  return OVN_OK;
}

int mcl_copy_stage(ovn_handle* h, int stage, void* d_out, cudaStream_t s) {
  McState& m = h->mcl;
  const size_t n = (size_t)m.n;
  if (stage == OVN_MCL_STAGE_MOTION) {
    const McParticles p = particles(h, m.pred_buf);
    const double* src[3] = {p.x, p.y, p.th};
    for (int j = 0; j < 3; ++j)
      OVN_CUDA(h, cudaMemcpyAsync(static_cast<double*>(d_out) + j * n, src[j], n * sizeof(double),
                                  cudaMemcpyDeviceToDevice, s));
    return OVN_OK;
  }
  if (stage == OVN_MCL_STAGE_SCALARS) {
    OVN_CUDA(h, cudaMemcpyAsync(d_out, m.scal.get() + kScMax, (kScU0 + 1 - kScMax) * sizeof(double),
                                cudaMemcpyDeviceToDevice, s));
    return OVN_OK;
  }
  const void* src = stage == OVN_MCL_STAGE_LOOKUP ? (const void*)m.kidx.get()
                    : stage == OVN_MCL_STAGE_LOGLIK ? (const void*)m.ll.get()
                    : stage == OVN_MCL_STAGE_WEIGHTS ? (const void*)m.w.get()
                    : stage == OVN_MCL_STAGE_PREFIX ? (const void*)m.cdf.get() : (const void*)m.anc.get();
  const size_t bytes = (stage == OVN_MCL_STAGE_LOOKUP || stage == OVN_MCL_STAGE_ANCESTORS) ? 4 : 8;
  OVN_CUDA(h, cudaMemcpyAsync(d_out, src, n * bytes, cudaMemcpyDeviceToDevice, s));
  return OVN_OK;
}

static __global__ void k_mcl_philox(uint64_t seed, const uint32_t* __restrict__ ctr, int n, uint32_t* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint4 w = philox(seed, ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]);
  out[4 * i] = w.x;
  out[4 * i + 1] = w.y;
  out[4 * i + 2] = w.z;
  out[4 * i + 3] = w.w;
}

int mcl_philox(ovn_handle* h, uint64_t seed, const uint32_t* d_ctr, int n, uint32_t* d_out, cudaStream_t s) {
  if (n == 0) return OVN_OK;
  k_mcl_philox<<<(n + kMclThreads - 1) / kMclThreads, kMclThreads, 0, s>>>(seed, d_ctr, n, d_out);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

}  // namespace ovn
