// gt_overlap.cu -- ground-truth overlap generator (com_overlap_yaw.py:10-68) on the GPU.
//
// The reference projects every reference scan, moved into the current frame by two float64 matrix
// products (com_overlap_yaw.py:39-40), with range_projection running in FLOAT64 (load_vertex builds
// a float64 array, utils.py:218-231) and compares float32 range images pixel by pixel (:44-45).
// Here: one thread per point does the two 4x4 products, the float64 depth / angle / bin pipeline
// of utils.py:75-104 and a 64-bit atomicMin of the depth's bit pattern (positive doubles order
// like integers; only the range image is needed, so no point index travels with the key); a second
// kernel rounds the winners to float32 (the image dtype, utils.py:120) and a third counts pixels.
// HBM-bound byte work: 16 B read per point, 8 B atomic per valid point into an L2-resident key image.
#include "range_bin.cuh"
#include "se3.cuh"

namespace ovn {

constexpr unsigned long long kGtEmpty = 0xFFFFFFFFFFFFFFFFull;

// range_projection of one transformed point in float64 (utils.py:75-104, range_bin) and the atomic-min of its
// depth into the key image `keys` [H][W]; points outside (0, max_range) are dropped
__device__ __forceinline__ void gt_scatter_point(double x, double y, double z, const GtParams& P,
                                                 unsigned long long* __restrict__ keys) {
  double depth;
  int bx, by;
  if (!range_bin(x, y, z, P, depth, bx, by)) return;
  atomicMin(keys + (size_t)by * P.W + bx, (unsigned long long)__double_as_longlong(depth));
}

__global__ void __launch_bounds__(256)
k_gt_scatter_f64(const float4* __restrict__ pts, const int64_t* __restrict__ offsets, int n_scans, int64_t n_total,
                 const double* __restrict__ pose_ref, const double* __restrict__ pose_cur_inv, GtParams P,
                 unsigned long long* __restrict__ keys) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_total || g < offsets[0] || g >= offsets[n_scans]) return;
  int lo = 0, hi = n_scans;                      // largest b with offsets[b] <= g
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (offsets[mid] <= g) lo = mid; else hi = mid;
  }
  const int b = lo;
  const float4 p = __ldg(pts + g);
  double x = (double)p.x, y = (double)p.y, z = (double)p.z, w = 1.0;   // load_vertex: (x, y, z, 1) float64
  if (pose_ref != nullptr) mat4_apply(pose_ref + (size_t)b * 16, x, y, z, w);      // com_overlap_yaw.py:39
  if (pose_cur_inv != nullptr) mat4_apply(pose_cur_inv, x, y, z, w);               // :40
  gt_scatter_point(x, y, z, P, keys + (size_t)b * P.H * P.W);
}

__global__ void __launch_bounds__(256)
k_gt_keys_to_range(const unsigned long long* __restrict__ keys, int64_t n, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  out[i] = (k == kGtEmpty) ? -1.0f : __double2float_rn(__longlong_as_double((long long)k));   // float32 image, utils.py:120,129
}

// counts[b] = #{ref_b > 0 and |ref_b - cur| < 1} (float32 arithmetic, com_overlap_yaw.py:44-45);
// row b == n_scans counts the current image's valid pixels (:31-32)
__global__ void __launch_bounds__(256)
k_gt_overlap_count(const float* __restrict__ ref, const float* __restrict__ cur, int n_scans, int HW,
                   int32_t* __restrict__ counts) {
  const int b = blockIdx.y;
  int c = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    if (b == n_scans) {
      c += cur[i] > 0.0f;
    } else {
      const float r = ref[(size_t)b * HW + i];
      c += (r > 0.0f) && (fabsf(__fsub_rn(r, cur[i])) < 1.0f);
    }
  }
  c = __reduce_add_sync(0xffffffffu, c);
  __shared__ int s[8];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int k = 0; k < 8; ++k) t += s[k];
    if (t) atomicAdd(counts + b, t);
  }
}

int gt_range_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans, int64_t n_total,
                   const double* d_pose_ref, const double* d_pose_cur_inv, float max_range, float* d_range,
                   cudaStream_t s) {
  if (n_scans <= 0) return OVN_OK;
  if (n_scans > h->cfg.max_batch_scans)
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "n_scans=%d exceeds max_batch_scans=%d", n_scans, h->cfg.max_batch_scans);
  const GtParams P = gt_params(h, max_range);
  const int64_t n_pix = (int64_t)n_scans * P.H * P.W;
  OVN_CUDA(h, cudaMemsetAsync(h->d_keys, 0xFF, (size_t)n_pix * sizeof(unsigned long long), s));
  if (n_total > 0) {
    k_gt_scatter_f64<<<(unsigned)((n_total + 255) / 256), 256, 0, s>>>(reinterpret_cast<const float4*>(d_points), d_offsets,
                                                                      n_scans, n_total, d_pose_ref, d_pose_cur_inv, P,
                                                                      h->d_keys);
    OVN_LAUNCH_CHECK(h);
  }
  k_gt_keys_to_range<<<(unsigned)((n_pix + 255) / 256), 256, 0, s>>>(h->d_keys, n_pix, d_range);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

int gt_overlap_count(ovn_handle* h, const float* d_ref, const float* d_cur, int n_scans, int32_t* d_counts, cudaStream_t s) {
  if (n_scans < 0) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "n_scans < 0");
  const int HW = h->cfg.proj_H * h->cfg.proj_W;
  OVN_CUDA(h, cudaMemsetAsync(d_counts, 0, (size_t)(n_scans + 1) * sizeof(int32_t), s));
  k_gt_overlap_count<<<dim3(8, (unsigned)(n_scans + 1)), 256, 0, s>>>(d_ref, d_cur, n_scans, HW, d_counts);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

// ---- all pairs: counts[f][r] for every current frame f x reference scan r -----------------------------
// The per-frame path above projects every reference scan into one current frame and writes a float32
// image per pair.  Here the clouds stay resident and a tile of tc current frames x tr reference scans is
// done in one pass: a thread loads one reference point, applies pose_ref once (keeping all four float64
// components, since w multiplies cur_inv's translation column) and then, for each frame of the tile,
// applies cur_inv and scatters into that pair's key image; the count then reads each key image once,
// compares it with the resident float32 image of the frame and resets it to empty for the next tile.
// Per point and pair the arithmetic is the per-frame path's: mat4_apply(pose_ref), mat4_apply(cur_inv)
// and gt_scatter_point, so every count is bit-for-bit the one ovn_gt_range_batch + ovn_gt_overlap_count give.
//
// Exact pruning: with T = cur_inv * pose_ref (exact), M its 3x3 block and t its translation, a point p
// lands at depth ||M p + t|| >= ||t|| - ||M||_2 ||p|| >= ||t|| - s rho, rho = max ||p|| of the scan and
// s^2 = max row sum of |M^T M| >= lambda_max(M^T M) = ||M||_2^2 (an induced norm bounds the spectral
// radius; s = 1 for an orthonormal block).  When ||t|| - s rho - eps >= max_range, no point of the scan
// is in range, every pixel of its image is -1 and the count is 0: the pair is skipped.  eps absorbs the
// rounding of T, of rho and of the device's own pose products (~1e-16 relative to the coordinates).
constexpr int kGtTileCurMax = 32;              // cur_inv of a frame tile lives in shared memory
constexpr int kGtTileRefMax = 64;              // reference offsets of a tile travel as a kernel argument
constexpr size_t kGtKeyBudget = 32u << 20;     // default tiles keep their key images within 32 MB of L2
constexpr double kGtPruneEps = 1e-3;           // metres

struct GtRefTile { int64_t off[kGtTileRefMax + 1]; };

// rho[b] = max ||p|| over the points of scan b, float64 (0 for an empty scan; max is order-free, so exact)
__global__ void __launch_bounds__(256)
k_gt_scan_radius(const float4* __restrict__ pts, const int64_t* __restrict__ offsets, double* __restrict__ radius) {
  const int b = blockIdx.x;
  const int64_t p1 = offsets[b + 1];
  double m = 0.0;
  for (int64_t i = offsets[b] + threadIdx.x; i < p1; i += blockDim.x) {
    const float4 p = __ldg(pts + i);
    const double x = p.x, y = p.y, z = p.z;
    m = fmax(m, __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ double s[8];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) m = fmax(m, s[k]);
    radius[b] = sqrt(m);
  }
}

// prune[f][r] = 1 when the bound above proves that pair (f, r) has count 0; *n_pruned += their number
__global__ void __launch_bounds__(256)
k_gt_pairs_prune(const double* __restrict__ pose_ref, const double* __restrict__ radius, int n_ref,
                 const double* __restrict__ cur_inv, int n_cur, double max_range, uint8_t* __restrict__ prune,
                 unsigned long long* __restrict__ n_pruned) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool pruned = false;
  if (i < (int64_t)n_cur * n_ref) {
    const double* A = cur_inv + (i / n_ref) * 16;
    const double* B = pose_ref + (i % n_ref) * 16;
    double T[3][4];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 4; ++c)
        T[r][c] = A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c] + A[4 * r + 2] * B[8 + c] + A[4 * r + 3] * B[12 + c];
    double g = 0.0;                                                   // max row sum of |M^T M|
    for (int r = 0; r < 3; ++r) {
      double row = 0.0;
      for (int c = 0; c < 3; ++c) row += fabs(T[0][r] * T[0][c] + T[1][r] * T[1][c] + T[2][r] * T[2][c]);
      g = fmax(g, row);
    }
    const double s = sqrt(g) * (1.0 + 1e-12);
    const double tn = sqrt(T[0][3] * T[0][3] + T[1][3] * T[1][3] + T[2][3] * T[2][3]);
    pruned = tn - s * radius[i % n_ref] - kGtPruneEps >= max_range;
    prune[i] = pruned;
  }
  const unsigned ballot = __ballot_sync(0xffffffffu, pruned);
  if ((threadIdx.x & 31) == 0 && ballot) atomicAdd(n_pruned, (unsigned long long)__popc(ballot));
}

// blockIdx.y = reference scan r0 + y of the tile; keys [nf][nr][H*W]
__global__ void __launch_bounds__(256)
k_gt_pairs_scatter(const float4* __restrict__ pts, GtRefTile T, int r0, int nr, const double* __restrict__ pose_ref,
                   const double* __restrict__ cur_inv, int f0, int nf, const uint8_t* __restrict__ prune, int n_ref,
                   GtParams P, unsigned long long* __restrict__ keys) {
  __shared__ double s_inv[kGtTileCurMax * 16];
  __shared__ uint8_t s_on[kGtTileCurMax];
  const int rl = blockIdx.y;
  for (int i = threadIdx.x; i < nf * 16; i += blockDim.x) s_inv[i] = cur_inv[(size_t)f0 * 16 + i];
  const bool on = threadIdx.x < nf && !prune[(size_t)(f0 + threadIdx.x) * n_ref + r0 + rl];
  if (threadIdx.x < nf) s_on[threadIdx.x] = on;
  if (!__syncthreads_or(on)) return;                                // every frame of the tile pruned
  const int64_t g = T.off[rl] + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= T.off[rl + 1]) return;
  const float4 p = __ldg(pts + g);
  double x = (double)p.x, y = (double)p.y, z = (double)p.z, w = 1.0;    // load_vertex: (x, y, z, 1) float64
  mat4_apply(pose_ref + (size_t)(r0 + rl) * 16, x, y, z, w);            // com_overlap_yaw.py:39, once per tile
  const size_t HW = (size_t)P.H * P.W;
  for (int f = 0; f < nf; ++f) {
    if (!s_on[f]) continue;
    double a = x, b = y, c = z, d = w;
    mat4_apply(s_inv + f * 16, a, b, c, d);                             // :40
    gt_scatter_point(a, b, c, P, keys + ((size_t)f * nr + rl) * HW);
  }
}

// blockIdx.y = pair f * nr + rl of the tile: the count of k_gt_overlap_count on the key image, which is
// left empty again
__global__ void __launch_bounds__(256)
k_gt_pairs_count(unsigned long long* __restrict__ keys, const float* __restrict__ cur, int f0, int r0, int nr,
                 const uint8_t* __restrict__ prune, int n_ref, int HW, int32_t* __restrict__ counts, int64_t ld) {
  const int f = blockIdx.y / nr, rl = blockIdx.y % nr;
  if (prune[(size_t)(f0 + f) * n_ref + r0 + rl]) return;           // an image of -1 only: count 0
  unsigned long long* k = keys + (size_t)blockIdx.y * HW;
  const float* c = cur + (size_t)(f0 + f) * HW;
  int n = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    const unsigned long long key = k[i];
    if (key == kGtEmpty) continue;                                  // -1: never counted
    k[i] = kGtEmpty;
    const float r = __double2float_rn(__longlong_as_double((long long)key));
    n += (r > 0.0f) && (fabsf(__fsub_rn(r, c[i])) < 1.0f);
  }
  n = __reduce_add_sync(0xffffffffu, n);
  __shared__ int s[8];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int j = 0; j < 8; ++j) t += s[j];
    if (t) atomicAdd(counts + (size_t)(f0 + f) * ld + r0 + rl, t);
  }
}

int gt_scan_radius(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans, double* d_radius,
                   cudaStream_t s) {
  if (n_scans <= 0) return OVN_OK;
  k_gt_scan_radius<<<n_scans, 256, 0, s>>>(reinterpret_cast<const float4*>(d_points), d_offsets, d_radius);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

int gt_pairs_count(ovn_handle* h, const float* d_points, const int64_t* h_offsets, int n_ref, const double* d_pose_ref,
                   const double* d_radius, const float* d_cur_range, const double* d_pose_cur_inv, int n_cur,
                   float max_range, int tile_cur, int tile_ref, int32_t* d_counts, int64_t ld_counts,
                   int64_t* d_n_pruned, cudaStream_t s) {
  const GtParams P = gt_params(h, max_range);
  const int HW = P.H * P.W;
  if (tile_cur <= 0) tile_cur = 8;
  if (tile_ref <= 0) {
    const size_t fit = kGtKeyBudget / ((size_t)tile_cur * HW * sizeof(unsigned long long));
    tile_ref = fit < 1 ? 1 : (fit > (size_t)kGtTileRefMax ? kGtTileRefMax : (int)fit);
  }
  if (tile_cur > kGtTileCurMax || tile_ref > kGtTileRefMax)
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "ovn_gt_pairs_count: tile %d x %d exceeds %d x %d", tile_cur, tile_ref,
                kGtTileCurMax, kGtTileRefMax);
  const int tc = n_cur < tile_cur ? n_cur : tile_cur, tr = n_ref < tile_ref ? n_ref : tile_ref;
  if (n_cur > 0 && n_ref > 0)          // only the n_ref columns of each row: the others may belong to another call
    OVN_CUDA(h, cudaMemset2DAsync(d_counts, (size_t)ld_counts * sizeof(int32_t), 0, (size_t)n_ref * sizeof(int32_t),
                                  (size_t)n_cur, s));
  if (d_n_pruned) OVN_CUDA(h, cudaMemsetAsync(d_n_pruned, 0, sizeof(int64_t), s));
  if (n_cur == 0 || n_ref == 0) return OVN_OK;
  // workspaces, allocated by the first call that needs them
  const size_t key_bytes = (size_t)tc * tr * HW * sizeof(unsigned long long);
  int rc = h->d_pair_keys.ensure(h, key_bytes);
  if (rc != OVN_OK) return rc;
  rc = h->d_pair_prune.ensure(h, (size_t)n_cur * n_ref + sizeof(unsigned long long));
  if (rc != OVN_OK) return rc;
  // [8-byte pruned counter][n_cur][n_ref] flags
  unsigned long long* cnt = reinterpret_cast<unsigned long long*>(h->d_pair_prune.get());
  uint8_t* prune = h->d_pair_prune + sizeof(unsigned long long);
  OVN_CUDA(h, cudaMemsetAsync(h->d_pair_keys, 0xFF, key_bytes, s));
  OVN_CUDA(h, cudaMemsetAsync(cnt, 0, sizeof(unsigned long long), s));
  const int64_t n_pairs = (int64_t)n_cur * n_ref;
  k_gt_pairs_prune<<<(unsigned)((n_pairs + 255) / 256), 256, 0, s>>>(d_pose_ref, d_radius, n_ref, d_pose_cur_inv, n_cur,
                                                                    P.max_range, prune, cnt);
  OVN_LAUNCH_CHECK(h);
  if (d_n_pruned)
    OVN_CUDA(h, cudaMemcpyAsync(d_n_pruned, cnt, sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
  const float4* pts = reinterpret_cast<const float4*>(d_points);
  const unsigned count_blocks = (unsigned)((HW + 256 * 8 - 1) / (256 * 8));
  for (int f0 = 0; f0 < n_cur; f0 += tc) {
    const int nf = n_cur - f0 < tc ? n_cur - f0 : tc;
    for (int r0 = 0; r0 < n_ref; r0 += tr) {
      const int nr = n_ref - r0 < tr ? n_ref - r0 : tr;
      GtRefTile T;
      int64_t most = 0;
      for (int i = 0; i <= nr; ++i) {
        T.off[i] = h_offsets[r0 + i];
        if (i > 0 && T.off[i] - T.off[i - 1] > most) most = T.off[i] - T.off[i - 1];
      }
      if (most > 0) {
        k_gt_pairs_scatter<<<dim3((unsigned)((most + 255) / 256), nr), 256, 0, s>>>(
            pts, T, r0, nr, d_pose_ref, d_pose_cur_inv, f0, nf, prune, n_ref, P, h->d_pair_keys);
        OVN_LAUNCH_CHECK(h);
      }
      k_gt_pairs_count<<<dim3(count_blocks, nf * nr), 256, 0, s>>>(h->d_pair_keys, d_cur_range, f0, r0, nr, prune,
                                                                   n_ref, HW, d_counts, ld_counts);
      OVN_LAUNCH_CHECK(h);
    }
  }
  return OVN_OK;
}

}  // namespace ovn
