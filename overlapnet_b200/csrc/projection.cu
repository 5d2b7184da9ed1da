// projection.cu -- stage 1 of the hot path: raw Velodyne clouds -> 64x900 range / vertex /
// intensity / index / normal / semantic images and the packed NHWC network input.
//
// Replaces (reference file:line):
//   range_projection        src/utils/utils.py:59-134
//   gen_normal_map + wrap   src/utils/utils.py:137-186
//   gen_semantic_data body  src/utils/gen_semantic_data.py:36-46
//   prepareOneInput packing src/two_heads/ImagePairOverlapOrientationSequence.py:130-207
//
// Design (HBM-bound integer/byte work, no tensor cores):
//   K1 scatter : one thread per point, one coalesced 16-byte load per point, float32 arithmetic in
//                exactly the reference's operation order (no FMA contraction), 64-bit atomicMin of
//                (depth_bits << 32 | point_index) into a per-scan key image that stays in L2.
//                "nearest point wins, lowest index on exact ties" == the reference's
//                depth-descending argsort + last-write-wins scatter.
//   K2 gather  : one thread per pixel; an 8x32 pixel tile stages its 9x33 winners (with the wrapped
//                right halo and the lower halo) in shared memory, then writes every requested
//                image with coalesced stores; normals are computed in the reference's rounding
//                order (float32 products, double accumulate, one rounding -- NumPy's sdot).
//   Bit-exact bins: atan2/asin are defined as the correctly rounded float32 values (oracle
//                docstring).  The fast path estimates the pre-floor bin from atan2f/asinf and keeps
//                its floor when it is further from a bin edge than a margin derived from H, W and the
//                fov (make_params); otherwise the float64 function is evaluated (see K1).
#include "common.cuh"
#include "se3.cuh"

#include <cmath>
#include <cstring>

namespace ovn {

struct ProjParams {
  int H, W;
  float pi32;            // float32(np.pi)
  float abs_fov_down32;  // float32(abs(fov_down/180*pi))
  float fov32;           // float32(abs(fov_down_r)+abs(fov_up_r))
  float W32, H32;
  float max_range;
  float kx, cx;          // fast estimate of the pre-floor x bin: yaw * W / (2 pi) + W / 2
  float ky, cy;          // ... and of the y bin: -pitch * H / fov + (1 - |fov_down| / fov) * H
  float mx, my;          // the estimate decides a bin when it lies further than this from a bin edge
};

// float32 ulp in the binade of a > 0
static double ulp32(double a) {
  int e;
  frexp(a, &e);
  return ldexp(1.0, e - 24);
}

// Worst-case distance, in bins, between the fast estimate t and the exact pre-floor value P(fl32(angle))
// (DESIGN.md section 4).  Three sources: atan2f / asinf against the correctly rounded angle (3 / 2 ulp in the
// CUDA Programming Guide's table, + 1/2 ulp for the rounding of the exact angle), the roundings of the
// reference's float32 pipeline (pi32 and fov32 included), and the estimate's own (kx / ky / cy and the fma).
// x: |yaw| <= pi.  y: the estimate only decides points inside the fov, so |pitch| <= max(|fov_up|, |fov_down|).
static double bound_x(int W) {
  const double pi = 3.14159265358979323846, e24 = ldexp(1.0, -24);
  const double kx = W / (2.0 * pi);
  return kx * 3.5 * ulp32(pi) + 0.5 * W * 3.5 * e24 + ulp32(W);
}
static double bound_y(int H, double fu, double fd) {
  const double e24 = ldexp(1.0, -24);
  const double fov = fabs(fd) + fabs(fu), ky = H / fov;
  const double pmax = fmax(fabs(fu), fabs(fd)) * (1.0 + 1e-6);
  return ky * (2.5 * ulp32(pmax) + pmax * e24 + 0.5 * ulp32(fabs(fd)) + 0.5 * ulp32(pmax + fabs(fd))) +
         H * 4.0 * e24 + ulp32(H);
}

static ProjParams make_params(const ovn_handle* h, float max_range) {
  ProjParams p;
  p.H = h->cfg.proj_H;
  p.W = h->cfg.proj_W;
  const double pi = 3.14159265358979323846;
  double fu = (double)h->cfg.fov_up_deg / 180.0 * pi;     // utils.py:70
  double fd = (double)h->cfg.fov_down_deg / 180.0 * pi;   // utils.py:71
  double fov = fabs(fd) + fabs(fu);                       // utils.py:72
  p.pi32 = (float)pi;
  p.abs_fov_down32 = (float)fabs(fd);
  p.fov32 = (float)fov;
  p.W32 = (float)p.W;
  p.H32 = (float)p.H;
  p.max_range = max_range;
  p.kx = (float)(p.W / (2.0 * pi));
  p.cx = (float)(p.W / 2.0);
  p.ky = (float)(-(double)p.H / fov);
  p.cy = (float)((1.0 - fabs(fd) / fov) * p.H);
  // twice the worst case, and never below the margins of the 64 x 900, 28-degree default (1e-3 / 1e-4, where
  // the bounds are 2.8e-4 / 4.2e-5): the default geometry keeps its fast-path decisions
  p.mx = (float)fmax(1e-3, 2.0 * bound_x(p.W));
  p.my = (float)fmax(1e-4, 2.0 * bound_y(p.H, fu, fd));
  return p;
}

constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;

__device__ __forceinline__ int bin_x(float yaw, const ProjParams& P) {
  // utils.py:90,94,98-100 in float32, one rounding per operation
  float t = __fdiv_rn(yaw, P.pi32);
  t = __fadd_rn(t, 1.0f);
  t = __fmul_rn(0.5f, t);
  t = __fmul_rn(t, P.W32);
  t = floorf(t);
  t = fminf((float)(P.W - 1), t);
  t = fmaxf(0.0f, t);
  return (int)t;
}

__device__ __forceinline__ int bin_y(float pitch, const ProjParams& P) {
  // utils.py:91,95,102-104
  float t = __fadd_rn(pitch, P.abs_fov_down32);
  t = __fdiv_rn(t, P.fov32);
  t = __fsub_rn(1.0f, t);
  t = __fmul_rn(t, P.H32);
  t = floorf(t);
  t = fminf((float)(P.H - 1), t);
  t = fmaxf(0.0f, t);
  return (int)t;
}

__device__ __forceinline__ int find_scan(const int64_t* __restrict__ offsets, int n_scans, int64_t g) {
  // largest b with offsets[b] <= g  (offsets has n_scans+1 entries, non-decreasing)
  int lo = 0, hi = n_scans;
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (offsets[mid] <= g) lo = mid; else hi = mid;
  }
  return lo;
}

// ------------------------------------------------------------------------------------------
// Point sources of the scatter and the gather.  The scatter runs one thread per g in [seg[0], seg[n_seg]) and
// finds the segment s with seg[s] <= g < seg[s + 1]; the source gives the point of g, the image it lands in and
// the index its key carries (from g and seg[s]).  Image b's points are g = base(b) + key index, from which the gather recomputes a
// winner's point.
// ------------------------------------------------------------------------------------------
// Raw clouds (ovn_project_batch and the preprocess calls): segment b is scan b and image b, seg the caller's
// point offsets; the key carries the point's index in its scan.
struct RawPoints {
  static constexpr bool kRanked = true;      // d_idx is the winner's index in the FILTERED cloud
  const float4* __restrict__ pts;
  const int64_t* __restrict__ offsets;
  __device__ __forceinline__ float4 point(int b, int64_t g) const { return __ldg(pts + g); }
  __device__ __forceinline__ int image(int b) const { return b; }
  __device__ __forceinline__ uint32_t key_index(int b, int64_t g, int64_t seg_start) const {
    return (uint32_t)(g - seg_start);
  }
  __device__ __forceinline__ int64_t base(int b) const { return __ldg(offsets + b); }
  __device__ __forceinline__ float4 winner(int b, int64_t base, uint32_t k, int, int) const {
    return __ldg(pts + base + k);
  }
};

// One render entry (ovn_render_batch): a resident cloud moved by a float64 pose into a virtual frame.
struct RenderEntry {
  double M[16];          // row-major 4x4, bottom row 0 0 0 1
  int64_t cloud_start;   // the cloud's first point in d_points
  int64_t image_base;    // seg[] of the image's first entry: the key carries g - image_base, the concatenated index
  int32_t image;
  int32_t pad;
};
static_assert(sizeof(RenderEntry) == 152, "RenderEntry layout");

// Posed entries: segment e is entry e, seg the prefix of the entries' point counts over the call, so an image's
// entries are consecutive segments and g - image_base is the point's index in the image's concatenated cloud.
struct PosedPoints {
  static constexpr bool kRanked = false;     // d_idx (d_winner) is the concatenated index itself
  const float4* __restrict__ pts;
  const RenderEntry* __restrict__ ent;       // [n_entries]
  const int64_t* __restrict__ seg;           // [n_entries + 1]
  const int64_t* __restrict__ first;         // [n_images + 1] first entry of each image
  // q = fl32(M (x, y, z, 1)) in float64 without contraction (mat4_apply), intensity kept
  __device__ __forceinline__ float4 load(int e, int64_t local) const {
    const float4 p = __ldg(pts + ent[e].cloud_start + local);
    double x = (double)p.x, y = (double)p.y, z = (double)p.z, w = 1.0;
    mat4_apply(ent[e].M, x, y, z, w);
    return make_float4(__double2float_rn(x), __double2float_rn(y), __double2float_rn(z), p.w);
  }
  __device__ __forceinline__ float4 point(int e, int64_t g) const { return load(e, g - seg[e]); }
  __device__ __forceinline__ int image(int e) const { return ent[e].image; }
  __device__ __forceinline__ uint32_t key_index(int e, int64_t g, int64_t seg_start) const {
    return (uint32_t)(g - ent[e].image_base);
  }
  __device__ __forceinline__ int64_t base(int b) const { return seg[first[b]]; }
  __device__ __forceinline__ float4 winner(int b, int64_t base, uint32_t k, int, int) const {
    const int64_t e0 = first[b], g = base + k;
    const int e = (int)e0 + find_scan(seg + e0, (int)(first[b + 1] - e0), g);
    return point(e, g);
  }
};

// utils.py:75  np.linalg.norm(xyz, 2, axis=1): sqrt((x*x + y*y) + z*z), float32, no FMA
__device__ __forceinline__ float point_depth(const float4 p) {
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(p.x, p.x), __fmul_rn(p.y, p.y)), __fmul_rn(p.z, p.z)));
}

// utils.py:86-104: the pixel of a point of float32 depth `depth` > 0
__device__ __forceinline__ void point_bins(const float4 p, const float depth, const ProjParams& P, int& bx, int& by) {
  // Bins: the exact answer is floor(P(fl32(angle))) with P the reference's float32 pipeline (bin_x /
  // bin_y, monotone) and fl32 the correctly rounded float32 angle.  Fast path: ONE fused estimate
  // t = angle * scale + offset of the pre-floor value; all error sources together (atan2f <= 3 ulp,
  // asinf <= 2 ulp, the pipeline's roundings, the estimate's own) stay below bound_x / bound_y bins
  // (2.8e-4 / 4.2e-5 at 64 x 900 and the default fov), so whenever t is further than P.mx (P.my, at
  // least twice the bound) from an integer -- and inside the image -- floor(t) IS the reference's bin.
  // Otherwise (0.2 % of the points at 64 x 900) the float64 function is rounded once and pushed through
  // the exact pipeline.  The first version ran the exact pipeline on
  // both ends of an error bracket for every point: 4 correctly rounded divisions, 295 instructions per
  // point, issue-bound.
  // ---- yaw bin (utils.py:86,90,94,98-100)
  {
    const float yaw_f = -atan2f(p.y, p.x);
    const float t = fmaf(yaw_f, P.kx, P.cx);
    const float fl = floorf(t);
    const float fr = t - fl;
    if (fr > P.mx && fr < 1.0f - P.mx && t > P.mx && t < P.W32 - P.mx) {
      bx = (int)fl;
    } else {
      const float yaw_cr = __double2float_rn(-atan2((double)p.y, (double)p.x));
      bx = bin_x(yaw_cr, P);
    }
  }
  // ---- pitch bin (utils.py:87,91,95,102-104); q must be the reference's correctly rounded z / depth
  {
    const float q = __fdiv_rn(p.z, depth);
    const float pit_f = asinf(q);
    const float t = fmaf(pit_f, P.ky, P.cy);
    const float fl = floorf(t);
    const float fr = t - fl;
    if (fr > P.my && fr < 1.0f - P.my && t > P.my && t < P.H32 - P.my) {
      by = (int)fl;
    } else {
      const float pit_cr = __double2float_rn(asin((double)q));
      by = bin_y(pit_cr, P);
    }
  }
}

// ------------------------------------------------------------------------------------------
// K1: scatter.  grid = ceil(n_total / 256), block = 256; one thread per g of the source's segments.
// kCues (ovn_preprocess_cues_batch, raw points only): two key images per call, keys = A [n_scans][H*W] then
// B [n_scans][H*W].  A takes the points of the configured filter (0 < depth < max_range, utils.py:76-77), B those
// of the semantic cue's (0 < depth < inf, gen_semantic_data.py:39; NaN fails both).  The bins are computed once per
// point, and the validity bits (the ranks) follow B's filter: the probability gather indexes with B's filtered
// index.
// ------------------------------------------------------------------------------------------
template <bool kCues, class Src>
__global__ void __launch_bounds__(256)
k_project_scatter(const Src src, const int64_t* __restrict__ offsets, int n_scans, int64_t n_total, ProjParams P,
                  unsigned long long* __restrict__ keys, uint32_t* __restrict__ valid_words) {
  __shared__ int s_first_scan;
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (threadIdx.x == 0) {
    int64_t g0 = (int64_t)blockIdx.x * blockDim.x;
    s_first_scan = find_scan(offsets, n_scans, g0 < n_total ? g0 : n_total - 1);
  }
  __syncthreads();
  bool valid = false;
  if (g < n_total && g >= offsets[0] && g < offsets[n_scans]) {
    int b = s_first_scan;
    while (b + 1 < n_scans && g >= offsets[b + 1]) ++b;   // a block rarely spans > 2 scans
    const float4 p = src.point(b, g);
    const float depth = point_depth(p);
    const bool in_a = (depth > 0.0f) && (depth < P.max_range);   // utils.py:76-77
    valid = kCues ? (depth > 0.0f) && (depth < __int_as_float(0x7f800000)) : in_a;
    if (valid) {
      int bx, by;
      point_bins(p, depth, P, bx, by);
      const uint32_t local = src.key_index(b, g, offsets[b]);
      const unsigned long long key = ((unsigned long long)__float_as_uint(depth) << 32) | local;
      const size_t pix = (size_t)src.image(b) * P.H * P.W + (size_t)by * P.W + bx;
      if (!kCues || in_a) atomicMin(keys + pix, key);
      if (kCues) atomicMin(keys + (size_t)n_scans * P.H * P.W + pix, key);
    }
  }
  if (valid_words != nullptr) {
    const unsigned m = __ballot_sync(0xffffffffu, valid);
    if ((threadIdx.x & 31) == 0 && g < n_total) valid_words[g >> 5] = m;
  }
}

// ------------------------------------------------------------------------------------------
// Exclusive prefix sum of popcounts over the validity words (only when proj_idx / semantic
// output is requested): rank of a point among the valid points == index into the filtered cloud.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
k_scan_words_local(const uint32_t* __restrict__ words, int64_t n_words, uint32_t* __restrict__ prefix,
                   uint32_t* __restrict__ block_sums) {
  __shared__ uint32_t warp_tot[32];
  const int64_t i = (int64_t)blockIdx.x * 1024 + threadIdx.x;
  const uint32_t v = i < n_words ? __popc(words[i]) : 0u;
  uint32_t incl = v;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    uint32_t w = warp_tot[lane];
    uint32_t wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += t;
    }
    warp_tot[lane] = wi - w;   // exclusive
    if (lane == 31) block_sums[blockIdx.x] = wi;
  }
  __syncthreads();
  if (i < n_words) prefix[i] = warp_tot[wid] + incl - v;
}

__global__ void __launch_bounds__(1024)
k_scan_block_sums(uint32_t* __restrict__ block_sums, int n_blocks) {
  // single block, sequential over chunks of 1024
  __shared__ uint32_t warp_tot[32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int base = 0; base < n_blocks; base += 1024) {
    const int i = base + threadIdx.x;
    const uint32_t v = i < n_blocks ? block_sums[i] : 0u;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      uint32_t w = warp_tot[lane], wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += t;
      }
      warp_tot[lane] = wi - w;
    }
    __syncthreads();
    const uint32_t excl = carry + warp_tot[wid] + incl - v;
    if (i < n_blocks) block_sums[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(1024)
k_scan_add_offsets(uint32_t* __restrict__ prefix, int64_t n_words, const uint32_t* __restrict__ block_sums) {
  const int64_t i = (int64_t)blockIdx.x * 1024 + threadIdx.x;
  if (i < n_words) prefix[i] += block_sums[blockIdx.x];
}

__device__ __forceinline__ uint32_t valid_before(const uint32_t* __restrict__ words,
                                                 const uint32_t* __restrict__ prefix, int64_t g) {
  // number of valid points with global index < g
  const int64_t w = g >> 5;
  const uint32_t bit = (uint32_t)(g & 31);
  const uint32_t mask = bit ? (0xffffffffu >> (32 - bit)) : 0u;
  return prefix[w] + __popc(words[w] & mask);
}

// ------------------------------------------------------------------------------------------
// normal of one pixel, utils.py:166-173 with NumPy's rounding (oracle/projection.py:_norm3_vec)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float norm3_np(float a, float b, float c) {
  const double s = ((double)__fmul_rn(a, a) + (double)__fmul_rn(b, b)) + (double)__fmul_rn(c, c);
  return __fsqrt_rn(__double2float_rn(s));
}

__device__ __forceinline__ bool pixel_normal(const float4 p, const float4 u, const float4 v, float n[3]) {
  const float dux = __fsub_rn(u.x, p.x), duy = __fsub_rn(u.y, p.y), duz = __fsub_rn(u.z, p.z);
  const float dvx = __fsub_rn(v.x, p.x), dvy = __fsub_rn(v.y, p.y), dvz = __fsub_rn(v.z, p.z);
  const float nu = norm3_np(dux, duy, duz);
  const float nv = norm3_np(dvx, dvy, dvz);
  const float unx = __fdiv_rn(dux, nu), uny = __fdiv_rn(duy, nu), unz = __fdiv_rn(duz, nu);
  const float vnx = __fdiv_rn(dvx, nv), vny = __fdiv_rn(dvy, nv), vnz = __fdiv_rn(dvz, nv);
  // np.cross(v_norm, u_norm): each product rounded, then one subtraction (no FMA)
  const float wx = __fsub_rn(__fmul_rn(vny, unz), __fmul_rn(vnz, uny));
  const float wy = __fsub_rn(__fmul_rn(vnz, unx), __fmul_rn(vnx, unz));
  const float wz = __fsub_rn(__fmul_rn(vnx, uny), __fmul_rn(vny, unx));
  const float nw = norm3_np(wx, wy, wz);
  if (!(nw > 0.0f)) return false;                          // utils.py:171 (nan fails too)
  n[0] = __fdiv_rn(wx, nw);
  n[1] = __fdiv_rn(wy, nw);
  n[2] = __fdiv_rn(wz, nw);
  return true;
}

// ------------------------------------------------------------------------------------------
// K2: gather.  grid = (ceil(W/32), ceil(H/8), n_scans), block = 256 (8 rows x 32 columns).
// ------------------------------------------------------------------------------------------
struct GatherOut {
  float* range;       // [n][H][W]
  float* vertex;      // [n][H][W][4]
  float* intensity;   // [n][H][W]
  int32_t* idx;       // [n][H][W]
  float* normal;      // [n][H][W][3]
  float* packed;      // [n][H][W][C]
  int C, c_depth, c_normal, c_prob, n_prob, c_intensity;   // channel offsets in packed (-1 = absent)
  const float* probs; // [n_total][n_prob] raw per-point probabilities (quirk: indexed by filtered idx)
};

constexpr int TILE_R = 8, TILE_C = 32;

// kCues: keys holds A then B (k_project_scatter<true>); depth, normals and intensity come from A's winners, the
// probabilities from B's, indexed with B's rank (the validity bits are B's filter); out.idx is not written.
// Src::kRanked: out.idx is the winner's index in the filtered cloud (raw points); else the key's index.
template <bool kCues, class Src>
__global__ void __launch_bounds__(256)
k_project_gather(const Src src, ProjParams P, const unsigned long long* __restrict__ keys,
                 const uint32_t* __restrict__ valid_words, const uint32_t* __restrict__ word_prefix, GatherOut out) {
  __shared__ float4 s_pt[TILE_R + 1][TILE_C + 1];
  __shared__ float s_depth[TILE_R + 1][TILE_C + 1];
  __shared__ uint32_t s_local[TILE_R + 1][TILE_C + 1];
  const int b = blockIdx.z;
  const int x0 = blockIdx.x * TILE_C, y0 = blockIdx.y * TILE_R;
  const int64_t off = src.base(b);
  const unsigned long long* kb = keys + (size_t)b * P.H * P.W;
  for (int c = threadIdx.x; c < (TILE_R + 1) * (TILE_C + 1); c += blockDim.x) {
    const int ry = c / (TILE_C + 1), rx = c % (TILE_C + 1);
    const int y = y0 + ry;
    int x = x0 + rx;
    if (x >= P.W) x -= P.W;                                 // wrap(x+1, W), utils.py:155
    float depth = -1.0f;
    float4 p = make_float4(-1.f, -1.f, -1.f, -1.f);
    uint32_t local = 0;
    if (y < P.H && x < P.W) {
      const unsigned long long k = kb[(size_t)y * P.W + x];
      if (k != kEmptyKey) {
        depth = __uint_as_float((uint32_t)(k >> 32));
        local = (uint32_t)(k & 0xFFFFFFFFull);
        p = src.winner(b, off, local, y, x);
      }
    }
    s_pt[ry][rx] = p;
    s_depth[ry][rx] = depth;
    s_local[ry][rx] = local;
  }
  __syncthreads();
  const int ty = threadIdx.x / TILE_C, tx = threadIdx.x % TILE_C;
  const int y = y0 + ty, x = x0 + tx;
  if (y >= P.H || x >= P.W) return;
  const size_t pix = ((size_t)b * P.H + y) * P.W + x;
  const float depth = s_depth[ty][tx];
  const float4 p = s_pt[ty][tx];
  const bool has = depth > 0.0f;   // valid points have depth > 0; empty pixels hold -1

  int32_t fidx = -1;
  if (!kCues && has && (out.idx != nullptr || out.n_prob > 0)) {
    if constexpr (Src::kRanked) {
      // index into the FILTERED cloud (utils.py:76,117-118)
      fidx = (int32_t)(valid_before(valid_words, word_prefix, off + s_local[ty][tx]) -
                       valid_before(valid_words, word_prefix, off));
    } else {
      fidx = (int32_t)s_local[ty][tx];
    }
  }
  float nrm[3] = {-1.f, -1.f, -1.f};
  if ((out.normal != nullptr || out.c_normal >= 0) && has && y < P.H - 1 &&
      s_depth[ty][tx + 1] > 0.0f && s_depth[ty + 1][tx] > 0.0f) {
    float t[3];
    if (pixel_normal(p, s_pt[ty][tx + 1], s_pt[ty + 1][tx], t)) { nrm[0] = t[0]; nrm[1] = t[1]; nrm[2] = t[2]; }
  }
  if (out.range) out.range[pix] = has ? depth : -1.0f;
  if (out.vertex) reinterpret_cast<float4*>(out.vertex)[pix] = has ? make_float4(p.x, p.y, p.z, 1.0f)
                                                                     : make_float4(-1.f, -1.f, -1.f, -1.f);
  if (out.intensity) out.intensity[pix] = has ? p.w : -1.0f;
  if (out.idx) out.idx[pix] = fidx;
  if (out.normal) {
    float* o = out.normal + pix * 3;
    o[0] = nrm[0]; o[1] = nrm[1]; o[2] = nrm[2];
  }
  if (out.packed) {
    float* o = out.packed + pix * out.C;
    if (out.C == 4 && out.c_depth == 0 && out.c_normal == 1) {
      *reinterpret_cast<float4*>(o) = make_float4(has ? depth : -1.0f, nrm[0], nrm[1], nrm[2]);
    } else {
      if (out.c_depth >= 0) o[out.c_depth] = has ? depth : -1.0f;
      if (out.c_normal >= 0) { o[out.c_normal] = nrm[0]; o[out.c_normal + 1] = nrm[1]; o[out.c_normal + 2] = nrm[2]; }
      if (out.c_intensity >= 0) o[out.c_intensity] = has ? p.w : -1.0f;
      if (out.c_prob >= 0) {
        // gen_semantic_data.py:46 -- raw probs indexed with the filtered index (reference quirk)
        bool has_p = has;
        int32_t pidx = fidx;
        if (kCues) {   // B's winner and its rank among the points of 0 < depth < inf (gen_semantic_data.py:39-46)
          const unsigned long long k = keys[((size_t)gridDim.z + b) * P.H * P.W + (size_t)y * P.W + x];
          has_p = k != kEmptyKey;
          if (has_p)
            pidx = (int32_t)(valid_before(valid_words, word_prefix, off + (uint32_t)(k & 0xFFFFFFFFull)) -
                             valid_before(valid_words, word_prefix, off));
        }
        const float* src = out.probs + (size_t)(off + (has_p ? pidx : 0)) * out.n_prob;
        for (int c = 0; c < out.n_prob; ++c) o[out.c_prob + c] = has_p ? __ldg(src + c) : -1.0f;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// standalone normal map from range + vertex images (utils.py:137-175); one thread per pixel
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_normals_from_images(const float* __restrict__ range, const float4* __restrict__ vertex, int n_scans,
                      int H, int W, float* __restrict__ normal) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)n_scans * H * W;
  if (i >= total) return;
  const int x = (int)(i % W);
  const int y = (int)((i / W) % H);
  float n[3] = {-1.f, -1.f, -1.f};
  if (y < H - 1 && range[i] > 0.0f) {
    const int xw = (x + 1 >= W) ? x + 1 - W : x + 1;
    const size_t iu = i - x + xw, iv = i + W;
    if (range[iu] > 0.0f && range[iv] > 0.0f) {
      float t[3];
      if (pixel_normal(vertex[i], vertex[iu], vertex[iv], t)) { n[0] = t[0]; n[1] = t[1]; n[2] = t[2]; }
    }
  }
  normal[i * 3 + 0] = n[0];
  normal[i * 3 + 1] = n[1];
  normal[i * 3 + 2] = n[2];
}

// semantic gather from proj_idx (gen_semantic_data.py:41-46); one thread per (pixel, class)
__global__ void __launch_bounds__(256)
k_semantic_gather(const int32_t* __restrict__ idx, const float* __restrict__ probs,
                  const int64_t* __restrict__ offsets, int n_scans, int HW, int n_classes,
                  float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)n_scans * HW * n_classes;
  if (i >= total) return;
  const int c = (int)(i % n_classes);
  const size_t pix = i / n_classes;
  const int b = (int)(pix / HW);
  const int32_t id = idx[pix];
  out[i] = id >= 0 ? __ldg(probs + (size_t)(offsets[b] + id) * n_classes + c) : -1.0f;
}

// channel packing of separately computed cue images (prepareOneInput, Sequence.py:130-207)
__global__ void __launch_bounds__(256)
k_pack_input(const float* __restrict__ depth, const float* __restrict__ normal,
             const float* __restrict__ prob, const float* __restrict__ intensity, size_t n_pix,
             int C, int n_prob, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix) return;
  float* o = out + i * C;
  int c = 0;
  if (depth) o[c++] = depth[i];
  if (normal) { o[c] = normal[i * 3]; o[c + 1] = normal[i * 3 + 1]; o[c + 2] = normal[i * 3 + 2]; c += 3; }
  if (prob) { for (int k = 0; k < n_prob; ++k) o[c + k] = prob[i * n_prob + k]; c += n_prob; }
  if (intensity) o[c++] = intensity[i];
}

// out[i][y][x][c] = images[rows[i]][y][(x - shift[i]) mod W][c]: image i of the cloud rotated about z by
// theta = -2 pi shift / W (utils.py:86-90).  The normal channels [c_normal, c_normal + 3) of that image get
// (nx, ny) -> (cos nx - sin ny, sin nx + cos ny) in NumPy's float32 order (no FMA contraction); the
// gen_normal_map fill (-1, -1, -1) and every other channel are copied.  One thread per output float.
__global__ void __launch_bounds__(256)
k_gather_images(const float* __restrict__ images, int64_t n_images, const int32_t* __restrict__ rows,
                const int32_t* __restrict__ shift, const float* __restrict__ rot, size_t total, int H, int W, int C,
                int c_normal, float* __restrict__ out, int* __restrict__ err) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int c = (int)(e % C);
  const size_t pix = e / C;
  const int x = (int)(pix % W);
  const size_t iy = pix / W;
  const int y = (int)(iy % H);
  const int i = (int)(iy / H);
  int64_t r = rows[i];
  if (r < 0 || r >= n_images) {
    if (e == (size_t)i * H * W * C) atomicCAS(err, 0, kErrBadIndex);    // one thread per image raises the flag
    r = r < 0 ? 0 : n_images - 1;
  }
  int s = shift ? shift[i] % W : 0;
  if (s < 0) s += W;
  const int xs = x >= s ? x - s : x - s + W;
  const float* src = images + (((size_t)r * H + y) * W + xs) * C;
  float v = src[c];
  if (rot && c_normal >= 0 && c >= c_normal && c < c_normal + 2) {
    const float nx = src[c_normal], ny = src[c_normal + 1], nz = src[c_normal + 2];
    if (!(nx == -1.f && ny == -1.f && nz == -1.f)) {
      const float cs = rot[2 * i], sn = rot[2 * i + 1];
      v = c == c_normal ? __fsub_rn(__fmul_rn(cs, nx), __fmul_rn(sn, ny))
                        : __fadd_rn(__fmul_rn(sn, nx), __fmul_rn(cs, ny));
    }
  }
  out[e] = v;
}

// ------------------------------------------------------------------------------------------
// host-side drivers
// ------------------------------------------------------------------------------------------
// rank workspaces for n_total points; a grow leaves room for 1/8 more points + 1024.  What must fit is counted
// in bitmask words, on purpose: the kernels use ceil(n_total / 32) words and one block sum per 1024 words, so a
// count up to 31 points past the last grow's headroom still fits and does not reallocate.
static int ensure_point_capacity(ovn_handle* h, int64_t n_total) {
  const int64_t cap = n_total + n_total / 8 + 1024;
  const size_t need = n_total / 32 + 2, words = cap / 32 + 2;       // bitmask words
  int rc;
  if ((rc = h->d_valid_words.ensure(h, need * sizeof(uint32_t), words * sizeof(uint32_t))) != OVN_OK) return rc;
  if ((rc = h->d_word_prefix.ensure(h, need * sizeof(uint32_t), words * sizeof(uint32_t))) != OVN_OK) return rc;
  return h->d_scan_tmp.ensure(h, (need / 1024 + 2) * sizeof(uint32_t), (words / 1024 + 2) * sizeof(uint32_t));
}

// One projection of n_images images from the source's n_seg segments of g in [offsets[0], offsets[n_seg]).
// cues: the two key images of ovn_preprocess_cues_batch (k_project_scatter<true>); the handle's d_keys holds them
// only when it has probability channels (ovn_create).
template <class Src>
static int launch_projection(ovn_handle* h, const Src& src, const int64_t* d_offsets, int n_seg, int n_images,
                             int64_t n_total, float max_range, const GatherOut& out, cudaStream_t s, bool cues,
                             int prof_scatter, int prof_gather) {
  const ProjParams P = make_params(h, max_range);
  const bool need_rank = Src::kRanked && (cues || out.idx != nullptr || out.n_prob > 0);
  const size_t HW = (size_t)P.H * P.W;
  const size_t n_key_images = cues ? 2 : 1;
  OVN_CUDA(h, cudaMemsetAsync(h->d_keys, 0xFF, n_key_images * n_images * HW * sizeof(unsigned long long), s));
  int64_t n_words = (n_total + 31) / 32;
  if (need_rank) {
    int rc = ensure_point_capacity(h, n_total);
    if (rc != OVN_OK) return rc;
  }
  if (n_total > 0) {
    const int64_t blocks = (n_total + 255) / 256;
    prof_mark(h, prof_scatter, s);
    auto scatter = k_project_scatter<false, Src>;
    if constexpr (Src::kRanked) if (cues) scatter = k_project_scatter<true, Src>;
    scatter<<<(unsigned)blocks, 256, 0, s>>>(src, d_offsets, n_seg, n_total, P, h->d_keys,
                                             need_rank ? h->d_valid_words.get() : nullptr);
    prof_mark(h, prof_scatter, s);
    OVN_LAUNCH_CHECK(h);
    if (need_rank) {
      const int nb = (int)((n_words + 1023) / 1024);
      k_scan_words_local<<<nb, 1024, 0, s>>>(h->d_valid_words, n_words, h->d_word_prefix, h->d_scan_tmp);
      OVN_LAUNCH_CHECK(h);
      k_scan_block_sums<<<1, 1024, 0, s>>>(h->d_scan_tmp, nb);
      OVN_LAUNCH_CHECK(h);
      k_scan_add_offsets<<<nb, 1024, 0, s>>>(h->d_word_prefix, n_words, h->d_scan_tmp);
      OVN_LAUNCH_CHECK(h);
    }
  }
  dim3 grid((P.W + TILE_C - 1) / TILE_C, (P.H + TILE_R - 1) / TILE_R, n_images);
  prof_mark(h, prof_gather, s);
  auto gather = k_project_gather<false, Src>;
  if constexpr (Src::kRanked) if (cues) gather = k_project_gather<true, Src>;
  gather<<<grid, 256, 0, s>>>(src, P, h->d_keys, h->d_valid_words, h->d_word_prefix, out);
  prof_mark(h, prof_gather, s);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

static int run_projection(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans,
                          int64_t n_total, float max_range, const GatherOut& out, cudaStream_t s,
                          bool cues = false) {
  if (n_scans <= 0) return OVN_OK;
  if (n_scans > h->cfg.max_batch_scans)
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "n_scans=%d exceeds max_batch_scans=%d", n_scans, h->cfg.max_batch_scans);
  const RawPoints src = {reinterpret_cast<const float4*>(d_points), d_offsets};
  return launch_projection(h, src, d_offsets, n_scans, n_scans, n_total, max_range, out, s, cues, PROF_SCATTER,
                           PROF_GATHER);
}

int project_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans,
                  int64_t n_total, float max_range, float* d_range, float* d_vertex,
                  float* d_intensity, int32_t* d_idx, cudaStream_t s) {
  GatherOut out = {};
  out.range = d_range; out.vertex = d_vertex; out.intensity = d_intensity; out.idx = d_idx;
  out.c_depth = out.c_normal = out.c_prob = out.c_intensity = -1;
  return run_projection(h, d_points, d_offsets, n_scans, n_total,
                        max_range < 0 ? h->cfg.max_range : max_range, out, s);
}

// the packed input's channels in prepareOneInput's order (Sequence.py:143-207): depth, normals, probabilities,
// intensity
static GatherOut packed_channels(const ovn_handle* h, const float* d_probs, float* d_input) {
  GatherOut out = {};
  out.packed = d_input;
  out.C = h->C;
  int c = 0;
  out.c_depth = out.c_normal = out.c_prob = out.c_intensity = -1;
  if (h->cfg.use_depth) { out.c_depth = c; c += 1; }
  if (h->cfg.use_normals) { out.c_normal = c; c += 3; }
  if (h->cfg.n_prob_channels > 0) {
    out.c_prob = c; out.n_prob = h->cfg.n_prob_channels; out.probs = d_probs; c += out.n_prob;
  }
  if (h->cfg.use_intensity) { out.c_intensity = c; c += 1; }
  return out;
}

int preprocess_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans,
                     int64_t n_total, const float* d_probs, float* d_input, cudaStream_t s) {
  if (h->cfg.n_prob_channels > 0 && d_probs == nullptr)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "d_probs is NULL but n_prob_channels=%d", h->cfg.n_prob_channels);
  // semantic channels are generated with max_range=inf in the reference (gen_semantic_data.py:39)
  // while depth/normal/intensity use max_range=50; this path uses the configured max_range
  // for every cue, so it is bit-identical to the reference only for the geometric cues.
  // preprocess_cues_batch gives every cue the reference's range.
  return run_projection(h, d_points, d_offsets, n_scans, n_total, h->cfg.max_range,
                        packed_channels(h, d_probs, d_input), s);
}

// Every channel as the reference's cue files give it (gen_depth/normal/intensity_data.py at max_range,
// gen_semantic_data.py:33-46 at max_range = inf), in one scatter and one gather: see k_project_scatter<true>.
int preprocess_cues_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans,
                          int64_t n_total, const float* d_probs, float* d_input, cudaStream_t s) {
  if (h->cfg.n_prob_channels == 0) {
    if (d_probs != nullptr)
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "d_probs must be NULL: the handle has no probability channels");
    return preprocess_batch(h, d_points, d_offsets, n_scans, n_total, nullptr, d_input, s);
  }
  if (d_probs == nullptr)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "d_probs is NULL but n_prob_channels=%d", h->cfg.n_prob_channels);
  return run_projection(h, d_points, d_offsets, n_scans, n_total, h->cfg.max_range,
                        packed_channels(h, d_probs, d_input), s, true);
}

// ---- the render: range images of resident clouds moved into virtual frames ----------------------------------
// Reads and checks the host tables (nothing is launched on a refusal), uploads the entry table to d_render and
// projects each image from its entries' transformed points in entry order (PosedPoints).
static int render(ovn_handle* h, const float* d_points, const int64_t* h_offsets, int n_clouds, int n_virtual,
                  const int64_t* h_entry_offsets, const int32_t* h_entry_cloud, const double* h_entry_pose,
                  float max_range, const GatherOut& out, cudaStream_t s) {
  if (n_virtual > h->cfg.max_batch_scans)
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "n_virtual=%d exceeds max_batch_scans=%d", n_virtual, h->cfg.max_batch_scans);
  if (n_virtual <= 0) return OVN_OK;
  if (h_offsets[0] < 0) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render: h_offsets[0] < 0");
  for (int c = 0; c < n_clouds; ++c)
    if (h_offsets[c + 1] < h_offsets[c])
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render: h_offsets decreases at cloud %d", c);
  if (h_entry_offsets[0] != 0) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render: h_entry_offsets[0] must be 0");
  for (int v = 0; v < n_virtual; ++v)
    if (h_entry_offsets[v + 1] < h_entry_offsets[v])
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render: h_entry_offsets decreases at image %d", v);
  const int64_t n_entries = h_entry_offsets[n_virtual];
  if (n_entries >= INT32_MAX) OVN_SET_ERR(h, OVN_ERR_CAPACITY, "render: %lld entries", (long long)n_entries);
  std::vector<RenderEntry> ent((size_t)n_entries);
  std::vector<int64_t> seg((size_t)n_entries + 1), first(h_entry_offsets, h_entry_offsets + n_virtual + 1);
  seg[0] = 0;
  for (int v = 0; v < n_virtual; ++v) {
    for (int64_t e = h_entry_offsets[v]; e < h_entry_offsets[v + 1]; ++e) {
      const int32_t c = h_entry_cloud[e];
      if (c < 0 || c >= n_clouds)
        OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render: entry %lld names cloud %d, outside [0, %d)", (long long)e, c,
                    n_clouds);
      const double* M = h_entry_pose + 16 * e;
      for (int i = 0; i < 16; ++i)
        if (!std::isfinite(M[i])) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render: the pose of entry %lld is not finite",
                                              (long long)e);
      if (M[12] != 0.0 || M[13] != 0.0 || M[14] != 0.0 || M[15] != 1.0)
        OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render: the pose of entry %lld does not end in the row 0 0 0 1",
                    (long long)e);
      RenderEntry& E = ent[(size_t)e];
      memcpy(E.M, M, sizeof(E.M));
      E.cloud_start = h_offsets[c];
      E.image_base = seg[(size_t)h_entry_offsets[v]];
      E.image = v;
      E.pad = 0;
      seg[(size_t)e + 1] = seg[(size_t)e] + (h_offsets[c + 1] - h_offsets[c]);
    }
    // the key's index field holds the concatenated index
    const int64_t n_image = seg[(size_t)h_entry_offsets[v + 1]] - seg[(size_t)h_entry_offsets[v]];
    if (n_image >= (int64_t(1) << 32))
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render: image %d concatenates %lld points, 2^32 or more", v,
                  (long long)n_image);
  }
  const int64_t n_total = seg[(size_t)n_entries];
  if (n_total > (int64_t)INT32_MAX * 256)
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "render: %lld points in one call exceed the scatter grid", (long long)n_total);
  if (n_total > 0 && d_points == nullptr) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render: d_points is NULL");
  const size_t b_ent = ent.size() * sizeof(RenderEntry), b_seg = seg.size() * sizeof(int64_t);
  const size_t b_first = first.size() * sizeof(int64_t);
  std::vector<uint8_t> table(b_ent + b_seg + b_first);
  if (b_ent) memcpy(table.data(), ent.data(), b_ent);
  memcpy(table.data() + b_ent, seg.data(), b_seg);
  memcpy(table.data() + b_ent + b_seg, first.data(), b_first);
  int rc = h->d_render.ensure(h, table.size());
  if (rc != OVN_OK) return rc;
  // pageable source: the copy is staged before the call returns, after the stream's earlier work
  OVN_CUDA(h, cudaMemcpyAsync(h->d_render, table.data(), table.size(), cudaMemcpyHostToDevice, s));
  const uint8_t* base = h->d_render;
  PosedPoints src;
  src.pts = reinterpret_cast<const float4*>(d_points);
  src.ent = reinterpret_cast<const RenderEntry*>(base);
  src.seg = reinterpret_cast<const int64_t*>(base + b_ent);
  src.first = reinterpret_cast<const int64_t*>(base + b_ent + b_seg);
  return launch_projection(h, src, src.seg, (int)n_entries, n_virtual, n_total,
                           max_range < 0 ? h->cfg.max_range : max_range, out, s, false, PROF_RENDER_SCATTER,
                           PROF_RENDER_GATHER);
}

int render_batch(ovn_handle* h, const float* d_points, const int64_t* h_offsets, int n_clouds, int n_virtual,
                 const int64_t* h_entry_offsets, const int32_t* h_entry_cloud, const double* h_entry_pose,
                 float max_range, float* d_range, float* d_vertex, float* d_intensity, int32_t* d_winner,
                 cudaStream_t s) {
  GatherOut out = {};
  out.range = d_range; out.vertex = d_vertex; out.intensity = d_intensity; out.idx = d_winner;
  out.c_depth = out.c_normal = out.c_prob = out.c_intensity = -1;
  return render(h, d_points, h_offsets, n_clouds, n_virtual, h_entry_offsets, h_entry_cloud, h_entry_pose, max_range,
                out, s);
}

int render_preprocess_batch(ovn_handle* h, const float* d_points, const int64_t* h_offsets, int n_clouds,
                            int n_virtual, const int64_t* h_entry_offsets, const int32_t* h_entry_cloud,
                            const double* h_entry_pose, float* d_input, cudaStream_t s) {
  if (h->cfg.n_prob_channels > 0)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "render_preprocess: the handle has probability channels, which renders lack");
  return render(h, d_points, h_offsets, n_clouds, n_virtual, h_entry_offsets, h_entry_cloud, h_entry_pose,
                h->cfg.max_range, packed_channels(h, nullptr, d_input), s);
}

// ---- surfel renders: oriented disks from the keyframes' range images (DESIGN.md section 7, "Surfel renders") ------
// A keyframe's surfels are its projection's pixels: slot y W + x of its [H][W] bank holds two float4, (cx, cy, cz, r)
// and (nx, ny, nz, intensity); an empty pixel is an all-zero slot (r = 0, never drawn).
struct SurfelBuild {
  double kappa, c_min, delta;   // r = fl32(((kappa d) delta) / max(|n.c| / d, c_min)), delta = max(2 pi / W, fov / H)
};

// One thread per pixel of the projection's outputs.  Every float64 operation is rounded once (no contraction).
__global__ void __launch_bounds__(256)
k_surfel_build(const float* __restrict__ range, const float4* __restrict__ vertex, const float* __restrict__ intensity,
               const float* __restrict__ normal, size_t n_pix, SurfelBuild B, float4* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix) return;
  const float d = range[i];
  if (!(d > 0.0f)) {
    out[2 * i] = make_float4(0.f, 0.f, 0.f, 0.f);
    out[2 * i + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const float4 c = vertex[i];
  const double cx = c.x, cy = c.y, cz = c.z;
  float n0 = normal[3 * i], n1 = normal[3 * i + 1], n2 = normal[3 * i + 2];
  if (n0 == -1.f && n1 == -1.f && n2 == -1.f) {   // gen_normal_map's fill: the sensor-facing unit vector -c / |c|
    const double nc = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz)));
    n0 = __double2float_rn(__ddiv_rn(-cx, nc));
    n1 = __double2float_rn(__ddiv_rn(-cy, nc));
    n2 = __double2float_rn(__ddiv_rn(-cz, nc));
  }
  const double dot = __dadd_rn(__dadd_rn(__dmul_rn((double)n0, cx), __dmul_rn((double)n1, cy)),
                               __dmul_rn((double)n2, cz));
  const double den = fmax(__ddiv_rn(fabs(dot), (double)d), B.c_min);
  const float r = __double2float_rn(__ddiv_rn(__dmul_rn(__dmul_rn(B.kappa, (double)d), B.delta), den));
  out[2 * i] = make_float4(c.x, c.y, c.z, r);
  out[2 * i + 1] = make_float4(n0, n1, n2, intensity[i]);
}

// The entries of a surfel render (RenderEntry: M, cloud_start = the first slot of its keyframe's bank, image_base =
// the first entry of its image, image) with the banks, the pixel rays and the window's scales.
struct SurfelRender {
  const float4* __restrict__ surfels;   // [n_clouds][H][W][2]
  const RenderEntry* __restrict__ ent;  // [n_entries]
  const int64_t* __restrict__ first;    // [n_images + 1] first entry of each image
  const double* __restrict__ rays;      // [H][W][3] unit directions of the pixel centres
  double rows_per_rad, cols_per_rad;    // H / fov, W / (2 pi)
  int S;                                // max_splat
};

// q = M (c, 1) in mat4_apply's order, m = R n: float64, every product and sum rounded once
__device__ __forceinline__ void surfel_pose(const double* __restrict__ M, const float4 a, const float4 b, double q[3],
                                            double m[3]) {
  const double cx = a.x, cy = a.y, cz = a.z, nx = b.x, ny = b.y, nz = b.z;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    q[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(M[4 * i], cx), __dmul_rn(M[4 * i + 1], cy)),
                               __dmul_rn(M[4 * i + 2], cz)), M[4 * i + 3]);
    m[i] = __dadd_rn(__dadd_rn(__dmul_rn(M[4 * i], nx), __dmul_rn(M[4 * i + 1], ny)), __dmul_rn(M[4 * i + 2], nz));
  }
}

__device__ __forceinline__ double dot3_rn(const double a[3], const double* b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

// The ray u meets the plane (q, m) at t = (m.q) / (m.u); the pixel is drawn when |m.u| > 1e-6, t > 0,
// fl32(t) < max_range and |t u - q|^2 <= r^2.
__device__ __forceinline__ bool surfel_hit(const double q[3], const double m[3], double r2, const double* u,
                                           float max_range, double& t) {
  const double uu[3] = {__ldg(u), __ldg(u + 1), __ldg(u + 2)};
  const double den = dot3_rn(m, uu), num = dot3_rn(m, q);
  if (!(fabs(den) > 1e-6)) return false;
  t = __ddiv_rn(num, den);
  if (!(t > 0.0) || !(__double2float_rn(t) < max_range)) return false;
  const double d0 = __dsub_rn(__dmul_rn(t, uu[0]), q[0]), d1 = __dsub_rn(__dmul_rn(t, uu[1]), q[1]);
  const double d2 = __dsub_rn(__dmul_rn(t, uu[2]), q[2]);
  return __dadd_rn(__dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1)), __dmul_rn(d2, d2)) <= r2;
}

// Half-widths (rows hy, columns hx) of the box around the centre pixel that holds every pixel the surfel can draw,
// at most S.  A drawn ray lies within a = asin(r / |q|) of q (r < |q|), so its pitch differs from q's by at most a
// and its azimuth by at most 2 asin(sin(a / 2) / cos(|pitch_q| + a)) (haversine); in pixels that is at most
// a H / fov + 1/2 rows and that azimuth W / (2 pi) + 1/2 columns from the centre pixel.  ceil(.) + 1 adds at least
// 1/2 pixel more than that, which covers libm's errors here and the float32 bins of the centre many times over
// (DESIGN.md section 7).  NaN anywhere gives the full window.
__device__ __forceinline__ void surfel_window(double qz, double nq, double r, const SurfelRender& R, int& hy,
                                             int& hx) {
  hy = hx = R.S;
  if (!(r < nq)) return;
  const double a = asin(r / nq);
  hy = (int)fmin((double)R.S, ceil(a * R.rows_per_rad) + 1.0);
  const double p = fabs(asin(qz / nq)) + a;
  if (p < 1.5707963267948966) {
    const double s = sin(0.5 * a) / cos(p);
    if (s < 1.0) hx = (int)fmin((double)R.S, ceil(2.0 * asin(s) * R.cols_per_rad) + 1.0);
  }
}

// One lane's surfel in the scatter's flattened pixel loop.
struct SurfelLane {
  double q[3], m[3], r2;
  int y0, x0, ncols, image;   // box rows y0 .., columns x0 .. x0 + ncols - 1 (mod W)
  uint32_t key;               // the entry's ordinal in its image * H W + slot
};

// K1 of the surfel render.  grid = ceil(n_entries H W / 256), block = 256; thread i takes (entry, slot) = (i / HW,
// i % HW).  Each lane moves its surfel, culls it and forms its box; a warp prefix over the box areas flattens the
// warp's (surfel, pixel) list, and the 32 lanes stride over it, so a warp's lanes stay busy whatever the boxes'
// sizes (0 to (2S + 1)^2 pixels).  Key: float_bits(fl32(t)) << 32 | key, 64-bit atomicMin.
__global__ void __launch_bounds__(256)
k_surfel_scatter(const SurfelRender R, int64_t n_items, ProjParams P, unsigned long long* __restrict__ keys) {
  __shared__ SurfelLane s_lane[8][32];
  __shared__ int s_start[8][32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int HW = P.H * P.W;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int area = 0;
  if (i < n_items) {
    const int64_t e = i / HW;
    const int slot = (int)(i - e * HW);
    const RenderEntry& E = R.ent[e];
    const float4* rec = R.surfels + 2 * (E.cloud_start + slot);
    const float4 a = __ldg(rec);
    if (a.w > 0.0f) {
      SurfelLane& L = s_lane[wid][lane];
      surfel_pose(E.M, a, __ldg(rec + 1), L.q, L.m);
      const double nq = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(L.q[0], L.q[0]), __dmul_rn(L.q[1], L.q[1])),
                                             __dmul_rn(L.q[2], L.q[2])));
      const double r = (double)a.w;
      if (nq > 0.0 && __dsub_rn(nq, r) < (double)P.max_range) {
        const float4 c = make_float4(__double2float_rn(L.q[0]), __double2float_rn(L.q[1]), __double2float_rn(L.q[2]),
                                     0.f);
        const float depth = point_depth(c);
        if (depth > 0.0f) {
          int bx, by, hy, hx;
          point_bins(c, depth, P, bx, by);
          surfel_window(L.q[2], nq, r, R, hy, hx);
          const int y0 = max(0, by - hy), y1 = min(P.H - 1, by + hy);
          L.r2 = __dmul_rn(r, r);
          L.y0 = y0;
          L.x0 = bx - hx;
          L.ncols = 2 * hx + 1;
          L.image = E.image;
          L.key = (uint32_t)((e - E.image_base) * HW + slot);
          area = (y1 - y0 + 1) * L.ncols;
        }
      }
    }
  }
  int incl = area;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  s_start[wid][lane] = incl - area;
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  __syncwarp();
  for (int k = lane; k < total; k += 32) {
    // the owner: the last lane whose box starts at or before k (a lane with an empty box shares its start with the
    // next lane, so the last such lane has a box)
    int o = 0;
#pragma unroll
    for (int step = 16; step > 0; step >>= 1)
      if (s_start[wid][o + step] <= k) o += step;
    const SurfelLane& L = s_lane[wid][o];
    const int local = k - s_start[wid][o];
    const int row = local / L.ncols;
    const int y = L.y0 + row;
    int x = (L.x0 + (local - row * L.ncols)) % P.W;
    if (x < 0) x += P.W;
    double t;
    if (surfel_hit(L.q, L.m, L.r2, R.rays + 3 * ((size_t)y * P.W + x), P.max_range, t)) {
      const unsigned long long key = ((unsigned long long)__float_as_uint(__double2float_rn(t)) << 32) | L.key;
      atomicMin(keys + (size_t)L.image * HW + (size_t)y * P.W + x, key);
    }
  }
}

// The gather's source of a surfel render: image b's key index k is (entry ordinal) H W + slot; the winner's point is
// its hit on the pixel's ray, recomputed as the scatter computed it: (fl32(t u), intensity).
struct SurfelHits {
  static constexpr bool kRanked = false;     // d_winner is the key's index itself
  SurfelRender R;
  int HW, W;
  __device__ __forceinline__ int64_t base(int b) const { return R.first[b]; }
  __device__ __forceinline__ float4 winner(int b, int64_t base, uint32_t k, int y, int x) const {
    const int64_t e = base + k / (uint32_t)HW;
    const int slot = (int)(k % (uint32_t)HW);
    const RenderEntry& E = R.ent[e];
    const float4* rec = R.surfels + 2 * (E.cloud_start + slot);
    const float4 b1 = __ldg(rec + 1);
    double q[3], m[3];
    surfel_pose(E.M, __ldg(rec), b1, q, m);
    const double* u = R.rays + 3 * ((size_t)y * W + x);
    const double uu[3] = {__ldg(u), __ldg(u + 1), __ldg(u + 2)};
    const double t = __ddiv_rn(dot3_rn(m, q), dot3_rn(m, uu));
    return make_float4(__double2float_rn(__dmul_rn(t, uu[0])), __double2float_rn(__dmul_rn(t, uu[1])),
                       __double2float_rn(__dmul_rn(t, uu[2])), b1.w);
  }
};

static double surfel_delta(const ovn_handle* h) {
  const double pi = 3.14159265358979323846;
  const double fu = (double)h->cfg.fov_up_deg / 180.0 * pi, fd = (double)h->cfg.fov_down_deg / 180.0 * pi;
  return fmax(2.0 * pi / h->cfg.proj_W, (fabs(fd) + fabs(fu)) / h->cfg.proj_H);
}

int surfels_batch(ovn_handle* h, const float* d_points, const int64_t* d_offsets, int n_scans, int64_t n_total,
                  const ovn_surfel_params& prm, float* d_surfels, cudaStream_t s) {
  if (n_scans <= 0) return OVN_OK;
  if (n_scans > h->cfg.max_batch_scans)
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "n_scans=%d exceeds max_batch_scans=%d", n_scans, h->cfg.max_batch_scans);
  const size_t n_pix = (size_t)n_scans * h->cfg.proj_H * h->cfg.proj_W;
  // the projection's outputs: vertex (16 B), range, intensity (4 B) and normal (12 B) per pixel
  int rc = h->d_surfel.ensure(h, n_pix * 36);
  if (rc != OVN_OK) return rc;
  GatherOut out = {};
  out.vertex = reinterpret_cast<float*>(h->d_surfel.get());
  out.range = out.vertex + 4 * n_pix;
  out.intensity = out.range + n_pix;
  out.normal = out.intensity + n_pix;
  out.c_depth = out.c_normal = out.c_prob = out.c_intensity = -1;
  rc = run_projection(h, d_points, d_offsets, n_scans, n_total, h->cfg.max_range, out, s);
  if (rc != OVN_OK) return rc;
  const SurfelBuild B = {prm.kappa, prm.c_min, surfel_delta(h)};
  prof_mark(h, PROF_SURFEL_BUILD, s);
  k_surfel_build<<<(unsigned)((n_pix + 255) / 256), 256, 0, s>>>(out.range, reinterpret_cast<const float4*>(out.vertex),
                                                                 out.intensity, out.normal, n_pix, B,
                                                                 reinterpret_cast<float4*>(d_surfels));
  prof_mark(h, PROF_SURFEL_BUILD, s);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

// Reads and checks the host tables (nothing is launched on a refusal), uploads the entry table to d_render, and
// z-buffers each image's entries' surfels (k_surfel_scatter) before the projection's gather reads the winners.
static int render_surfels(ovn_handle* h, const float* d_surfels, int n_clouds, const double* d_rays, int n_virtual,
                          const int64_t* h_entry_offsets, const int32_t* h_entry_cloud, const double* h_entry_pose,
                          int max_splat, float max_range, const GatherOut& out, cudaStream_t s) {
  if (n_virtual > h->cfg.max_batch_scans)
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "n_virtual=%d exceeds max_batch_scans=%d", n_virtual, h->cfg.max_batch_scans);
  if (n_virtual <= 0) return OVN_OK;
  const int64_t HW = (int64_t)h->cfg.proj_H * h->cfg.proj_W;
  if (h_entry_offsets[0] != 0) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render_surfels: h_entry_offsets[0] must be 0");
  for (int v = 0; v < n_virtual; ++v) {
    if (h_entry_offsets[v + 1] < h_entry_offsets[v])
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render_surfels: h_entry_offsets decreases at image %d", v);
    // the key's index field holds (entry ordinal) H W + slot
    if ((h_entry_offsets[v + 1] - h_entry_offsets[v]) * HW >= (int64_t(1) << 32))
      OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render_surfels: image %d has %lld entries, 2^32 / (H W) or more", v,
                  (long long)(h_entry_offsets[v + 1] - h_entry_offsets[v]));
  }
  const int64_t n_entries = h_entry_offsets[n_virtual];
  if (n_entries >= INT32_MAX) OVN_SET_ERR(h, OVN_ERR_CAPACITY, "render_surfels: %lld entries", (long long)n_entries);
  const int64_t n_items = n_entries * HW;
  if (n_items > (int64_t)INT32_MAX * 256)
    OVN_SET_ERR(h, OVN_ERR_CAPACITY, "render_surfels: %lld surfel slots in one call exceed the scatter grid",
                (long long)n_items);
  std::vector<RenderEntry> ent((size_t)n_entries);
  for (int v = 0; v < n_virtual; ++v) {
    for (int64_t e = h_entry_offsets[v]; e < h_entry_offsets[v + 1]; ++e) {
      const int32_t c = h_entry_cloud[e];
      if (c < 0 || c >= n_clouds)
        OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render_surfels: entry %lld names cloud %d, outside [0, %d)", (long long)e,
                    c, n_clouds);
      const double* M = h_entry_pose + 16 * e;
      for (int i = 0; i < 16; ++i)
        if (!std::isfinite(M[i]))
          OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render_surfels: the pose of entry %lld is not finite", (long long)e);
      if (M[12] != 0.0 || M[13] != 0.0 || M[14] != 0.0 || M[15] != 1.0)
        OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render_surfels: the pose of entry %lld does not end in the row 0 0 0 1",
                    (long long)e);
      RenderEntry& E = ent[(size_t)e];
      memcpy(E.M, M, sizeof(E.M));
      E.cloud_start = (int64_t)c * HW;
      E.image_base = h_entry_offsets[v];
      E.image = v;
      E.pad = 0;
    }
  }
  if (n_entries > 0 && (d_surfels == nullptr || d_rays == nullptr))
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "render_surfels: d_surfels or d_rays is NULL");
  const size_t b_ent = ent.size() * sizeof(RenderEntry), b_first = (size_t)(n_virtual + 1) * sizeof(int64_t);
  std::vector<uint8_t> table(b_ent + b_first);
  if (b_ent) memcpy(table.data(), ent.data(), b_ent);
  memcpy(table.data() + b_ent, h_entry_offsets, b_first);
  int rc = h->d_render.ensure(h, table.size());
  if (rc != OVN_OK) return rc;
  // pageable source: the copy is staged before the call returns, after the stream's earlier work
  OVN_CUDA(h, cudaMemcpyAsync(h->d_render, table.data(), table.size(), cudaMemcpyHostToDevice, s));
  const ProjParams P = make_params(h, max_range < 0 ? h->cfg.max_range : max_range);
  const double pi = 3.14159265358979323846;
  const double fov = fabs((double)h->cfg.fov_down_deg / 180.0 * pi) + fabs((double)h->cfg.fov_up_deg / 180.0 * pi);
  SurfelHits src;
  src.R.surfels = reinterpret_cast<const float4*>(d_surfels);
  src.R.ent = reinterpret_cast<const RenderEntry*>(h->d_render.get());
  src.R.first = reinterpret_cast<const int64_t*>(h->d_render.get() + b_ent);
  src.R.rays = d_rays;
  src.R.rows_per_rad = P.H / fov;
  src.R.cols_per_rad = P.W / (2.0 * pi);
  src.R.S = max_splat;
  src.HW = (int)HW;
  src.W = P.W;
  OVN_CUDA(h, cudaMemsetAsync(h->d_keys, 0xFF, (size_t)n_virtual * HW * sizeof(unsigned long long), s));
  if (n_items > 0) {
    prof_mark(h, PROF_SURFEL_SCATTER, s);
    k_surfel_scatter<<<(unsigned)((n_items + 255) / 256), 256, 0, s>>>(src.R, n_items, P, h->d_keys);
    prof_mark(h, PROF_SURFEL_SCATTER, s);
    OVN_LAUNCH_CHECK(h);
  }
  dim3 grid((P.W + TILE_C - 1) / TILE_C, (P.H + TILE_R - 1) / TILE_R, n_virtual);
  prof_mark(h, PROF_SURFEL_GATHER, s);
  k_project_gather<false, SurfelHits><<<grid, 256, 0, s>>>(src, P, h->d_keys, nullptr, nullptr, out);
  prof_mark(h, PROF_SURFEL_GATHER, s);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

int render_surfels_batch(ovn_handle* h, const float* d_surfels, int n_clouds, const double* d_rays, int n_virtual,
                         const int64_t* h_entry_offsets, const int32_t* h_entry_cloud, const double* h_entry_pose,
                         const ovn_surfel_params& prm, float max_range, float* d_range, float* d_vertex,
                         float* d_intensity, int32_t* d_winner, cudaStream_t s) {
  GatherOut out = {};
  out.range = d_range; out.vertex = d_vertex; out.intensity = d_intensity; out.idx = d_winner;
  out.c_depth = out.c_normal = out.c_prob = out.c_intensity = -1;
  return render_surfels(h, d_surfels, n_clouds, d_rays, n_virtual, h_entry_offsets, h_entry_cloud, h_entry_pose,
                        prm.max_splat, max_range, out, s);
}

int render_surfels_preprocess_batch(ovn_handle* h, const float* d_surfels, int n_clouds, const double* d_rays,
                                    int n_virtual, const int64_t* h_entry_offsets, const int32_t* h_entry_cloud,
                                    const double* h_entry_pose, const ovn_surfel_params& prm, float* d_input,
                                    cudaStream_t s) {
  if (h->cfg.n_prob_channels > 0)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG,
                "render_surfels_preprocess: the handle has probability channels, which renders lack");
  return render_surfels(h, d_surfels, n_clouds, d_rays, n_virtual, h_entry_offsets, h_entry_cloud, h_entry_pose,
                        prm.max_splat, h->cfg.max_range, packed_channels(h, nullptr, d_input), s);
}

int normals_batch(ovn_handle* h, const float* d_range, const float* d_vertex, int n_scans,
                  float* d_normal, cudaStream_t s) {
  if (n_scans <= 0) return OVN_OK;
  const size_t total = (size_t)n_scans * h->cfg.proj_H * h->cfg.proj_W;
  k_normals_from_images<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(
      d_range, reinterpret_cast<const float4*>(d_vertex), n_scans, h->cfg.proj_H, h->cfg.proj_W, d_normal);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

int semantic_batch(ovn_handle* h, const int32_t* d_idx, const float* d_probs, const int64_t* d_offsets,
                   int n_scans, int n_classes, float* d_out, cudaStream_t s) {
  if (n_scans <= 0) return OVN_OK;
  const int HW = h->cfg.proj_H * h->cfg.proj_W;
  const size_t total = (size_t)n_scans * HW * n_classes;
  k_semantic_gather<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(d_idx, d_probs, d_offsets, n_scans, HW,
                                                                   n_classes, d_out);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

int pack_input(ovn_handle* h, const float* d_depth, const float* d_normal, const float* d_prob,
               const float* d_intensity, int n_scans, float* d_input, cudaStream_t s) {
  if (n_scans <= 0) return OVN_OK;
  const size_t n_pix = (size_t)n_scans * h->cfg.proj_H * h->cfg.proj_W;
  k_pack_input<<<(unsigned)((n_pix + 255) / 256), 256, 0, s>>>(d_depth, d_normal, d_prob, d_intensity, n_pix,
                                                              h->C, h->cfg.n_prob_channels, d_input);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

int gather_images(ovn_handle* h, const float* d_images, int64_t n_images, const int32_t* d_rows,
                  const int32_t* d_shift, const float* d_rot, int n, float* d_out, cudaStream_t s) {
  const size_t total = (size_t)n * h->cfg.proj_H * h->cfg.proj_W * h->C;
  const int c_normal = h->cfg.use_normals ? (h->cfg.use_depth ? 1 : 0) : -1;
  k_gather_images<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(d_images, n_images, d_rows, d_shift, d_rot, total,
                                                                  h->cfg.proj_H, h->cfg.proj_W, h->C, c_normal, d_out,
                                                                  h->d_err);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

}  // namespace ovn
