// network_tc.cu -- tensor-core path (precision f16_tc) of the leg and the two heads, for Hopper (sm_90a).
//
// Replaces: DeltaLayer + c_conv1 (generateNet.py:15-61,96-100)      -> k_delta_conv1_wgmma
//           c_conv2 (+ReLU) (generateNet.py:102-105)                -> k_conv2_wgmma
//           c_conv3 (+ReLU), Flatten + Dense(1, sigmoid) (:107-114) -> k_conv3_wgmma + k_dense_finalize
//           NormalizedCorrelation2D + argmax (:117-143, infer.py)   -> k_corr_wgmma + k_corr_finalize
//           leg Conv2D stack (generateNet.py:149-230)               -> layer 1: k_leg_layer1_small (1-2 scans) /
//                                                                      k_leg_layer1_direct (batches), SIMT fp32;
//                                                                      layers 2..: k_leg_mma (+ k_leg_splitk_reduce,
//                                                                      1-2 scans)
//
// Every GEMM runs on tensor cores (fp16 operands, fp32 accumulators) and reads packed operand layouts (8
// consecutive K values per 16-byte chunk).  The delta head is three persistent, warp-specialised wgmma kernels
// fed by bulk copies through mbarrier rings: k_delta_conv1_wgmma (83 % of the FLOPs of a pair) synthesises its
// A operand |l - r| in registers, so the 66 MB delta tensor of a pair (the reference's DeltaLayer output) is
// never materialised; k_conv2_wgmma and k_conv3_wgmma take both operands from shared memory.  The correlation
// head k_corr_wgmma is built the same way.  The leg is a warp-level mma.sync m16n8k16 kernel whose fragments are
// loaded straight from global; a single scan splits its K over more CTAs.
// Operands that must be fp32-grade are split into hi + lo fp16 halves (x = hi + lo exactly to 2^-22).
#include "common.cuh"
#include "hopper.cuh"

#include <cuda_fp16.h>
#include <stddef.h>
#include <stdlib.h>

namespace ovn {

using namespace hopper;

constexpr int WF = 360;                 // leg_output_width (the TC path is specialised to the
constexpr int CF = 128;                 //   reference geometry: 360 x 128 volumes, conv1size 15)
constexpr int S15 = 15;
constexpr int NB = 24;                  // 360 / 15
constexpr int PAIR_ROWS = NB * NB;      // 576 rows of c_conv2 output per pair
constexpr int K4_PITCH = CF;            // fp16 row pitch of the L / R operand copies of k_delta_conv1_wgmma (k4_pos)

struct TcState {
  Buffer<__half> w1p;           // [60 steps][4][64][8]
  Buffer<__half> w2p;           // [15 di][hi, lo][128 n][64 o] SWIZZLE_128B tiles (W2 = hi + lo in fp16)
  Buffer<__half> w3p;           // [2 halves][36 slabs][4][128][8]
  Buffer<float> b2eff;          // c_conv2 bias + the c_conv1 bias pushed through W2 (both layers are linear)
  // tensor-core leg (layers 2..): packed weights per layer, ping-pong activation planes
  Buffer<__half> wres[kMaxLegLayers];    // [cout/64][kh*kw*3 slabs (tap, term)][C_in/8][64][8]; term 0, 1 = hi, 2 = lo
  Buffer<__half> actp[2];
  Buffer<float> leg_part;       // K-slice sums of the single-scan leg: [n_split][rows][w_out][cout] fp32
  Buffer<__half> l16;           // [max_pairs][360][128]
  Buffer<__half> r16;           // [max_pairs][360][128] (pair mode) / [1][360][128] (query mode)
  Buffer<__half> o1;            // [rows_pad/128][15 di][128][64]: SWIZZLE_128B A tiles of c_conv2 (o1_chunk_offset)
  Buffer<__half> x3;            // [16 planes][rows_pad][8], row = pair*576 + jb*24 + ib
  Buffer<float> partial;        // [rows_pad][2]
  Buffer<__half> lc;            // correlation operands: [max_pairs][6 tiles][hi,lo][16][64][8]
  Buffer<__half> rc;            // [max_pairs or 1][3 thirds][hi,lo][16][128][8]
  Buffer<float> corr_part;      // [max_pairs][6 LEFT tiles][3 RIGHT thirds][360]
  // resident bank (ovn_bank_prepare): operand copies of the LEFT volumes, indexed by bank row
  const float* pb_key = nullptr;
  int64_t pb_rows = 0;                  // rows [0, pb_rows) prepared
  Buffer<__half> pb_l16;                // [cap][360][K4_PITCH]
  Buffer<__half> pb_lc;                 // [cap] x C6_VOL_L_BYTES
  Buffer<int32_t> pb_bad;               // [cap] 1: the row holds a value its fp16 copies cannot (kErrNonFiniteOperand)
  // per-channel centre of the feature volumes: the delta head only sees |l - r|, which is invariant
  // to a common offset, so both operands are stored as fp16(x - mu[c]) -- smaller magnitudes, smaller
  // fp16 rounding error of the (coherently re-used) volumes.  mu is calibrated once (first bank rows /
  // first RIGHT volume seen) or set through ovn_set_feature_center; values are fp16-representable.
  Buffer<float> mu;             // [128] device
  bool mu_set = false;
  // The same trick one and two layers further on: c_conv2 and c_conv3 are linear in their inputs, so
  // o1 and x3 are stored as fp16(x - mean[channel]) and the mean's image under the layer is folded into
  // that layer's bias (b2eff / b3eff).  Calibrated on the first pairs the handle scores.
  Buffer<float> mu_o1;          // [64]
  Buffer<float> mu_x3;          // [128]
  Buffer<float> b2base;         // c_conv2 bias + c_conv1 bias pushed through W2
  Buffer<float> b3eff;          // c_conv3 bias + mu_x3 pushed through the fp16 W3
  bool act_set = false;
  int64_t rows_pad = 0;
  int64_t last_n = 0;           // pairs of the last heads chunk whose o1 / x3 / partial are stored (0: none or unknown)
};

void TcStateDelete::operator()(TcState* t) const { delete t; }

// ------------------------------------------------------------------------------------------------
// fp32 feature volumes -> fp16 rows gathered by index (the tensor-core operands)
// ------------------------------------------------------------------------------------------------
// Storage order of a row of these copies (what k_delta_conv1_wgmma reads; the logical K order is unchanged).  Lane
// t of an A fragment needs the channel pairs 2t, 2t + 8, 2t + 16 and 2t + 24 of a 32-channel chunk: they are stored
// adjacent, 16 bytes at t * 16 of the chunk, so a fragment row is one 128-bit shared load.  Chunk cc of row r sits at
// chunk position cc ^ (r & 1): the two rows of a quarter-warp's load then fall in different halves of the banks.
__host__ __device__ __forceinline__ int k4_pos(int r, int c) {
  const int k = c & 31;
  return (((c >> 5) ^ (r & 1)) << 5) + ((k & 7) >> 1) * 8 + (k >> 3) * 2 + (k & 1);
}

// An fp16 value that is not finite (exponent field all ones): its source was NaN, inf or beyond fp16's range.  The
// heads' ReLUs (fmaxf) turn NaN into 0 and the argmax skips it, so such an operand would give plausible outputs:
// the operand kernels raise kErrNonFiniteOperand instead, which poisons the outputs of the call.
__device__ __forceinline__ bool h2_nonfinite(__half2 v) {
  const uint32_t b = *reinterpret_cast<const uint32_t*>(&v);
  return (b & 0x7c00u) == 0x7c00u || (b & 0x7c000000u) == 0x7c000000u;
}

__global__ void __launch_bounds__(256)
k_gather_rows_f16(const float* __restrict__ bank, const int32_t* __restrict__ idx, int n, const float* __restrict__ mu,
                  int row_shift, __half* __restrict__ out, int* __restrict__ err, int32_t* __restrict__ row_bad) {
  const int64_t per = (int64_t)WF * CF / 4;            // float4 per volume
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * per) return;
  const int p = (int)(i / per);
  const int64_t e = i % per;
  const int64_t row = idx ? idx[p] : p;
  const int r = (int)(e / (CF / 4)), c4 = (int)(e % (CF / 4));
  int64_t rs = r + row_shift;                                   // circular row shift (calibration pair only)
  if (rs >= WF) rs -= WF;
  const float4 v = __ldg(reinterpret_cast<const float4*>(bank + (row * WF + rs) * CF) + c4);
  const float4 m = __ldg(reinterpret_cast<const float4*>(mu) + c4);
  __half2 a = __floats2half2_rn(v.x - m.x, v.y - m.y), b = __floats2half2_rn(v.z - m.z, v.w - m.w);
  if (h2_nonfinite(a) || h2_nonfinite(b)) {
    if (row_bad) row_bad[p] = 1;          // a resident bank row: the heads calls that read it raise the flag
    else atomicCAS(err, 0, kErrNonFiniteOperand);
  }
  __half* o = out + ((int64_t)p * WF + r) * K4_PITCH;
  *reinterpret_cast<uint32_t*>(o + k4_pos(r, 4 * c4)) = *reinterpret_cast<uint32_t*>(&a);
  *reinterpret_cast<uint32_t*>(o + k4_pos(r, 4 * c4 + 2)) = *reinterpret_cast<uint32_t*>(&b);
}

// Per-channel mean over the rows of n volumes (bank rows idx[0..n) or 0..n-1), rounded to fp16:
// one block, fixed summation order (bit-reproducible).  Only runs when the centre is calibrated.
__global__ void __launch_bounds__(1024)
k_channel_mean(const float* __restrict__ bank, const int32_t* __restrict__ idx, int n, float* __restrict__ mu) {
  __shared__ float part[8][CF];
  const int c = threadIdx.x & (CF - 1), g = threadIdx.x >> 7;
  float acc = 0.f;
  for (int v = 0; v < n; ++v) {
    const float* vol = bank + (int64_t)(idx ? idx[v] : v) * WF * CF;
    for (int r = g; r < WF; r += 8) acc += __ldg(vol + (int64_t)r * CF + c);
  }
  part[g][c] = acc;
  __syncthreads();
  if (g == 0) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += part[k][c];
    mu[c] = __half2float(__float2half_rn(t / (float)((int64_t)n * WF)));
  }
}

constexpr int K4_STEPS = 60;            // W1 slices: 4 channel chunks x 15 dj

// o1 layout ("SWIZZLE_128B tiles", kept from the bulk-copy design: [128 rows x 64 K] tiles whose 16-byte
// chunks are XOR-swizzled by the row):
//   row m = pair*576 + jb*24 + ib (i = ib*15 + di), K = di*64 + o
//   o1[(m / 128) * 15 + di][m % 128][chunk (o/8) ^ (m & 7)][o % 8]
__host__ __device__ __forceinline__ size_t o1_row_offset(int64_t m, int di) {
  return ((size_t)((m >> 7) * S15 + di) * 128 + (size_t)(m & 127)) * 64;
}
__host__ __device__ __forceinline__ size_t o1_chunk_offset(int64_t m, int di, int c8) {
  return o1_row_offset(m, di) + (size_t)((c8 ^ (int)(m & 7)) * 8);
}

struct LegArgs {
  const __half* A; int64_t a_pitch;
  int runs_per_img, in_img_planes, in_run_planes;
  int kh, kw, c8in;
  const __half* Bp;           // [cout/64][kh*kw*3][c8in][64][8]
  const float* bias; int n_valid;
  int64_t M;                  // output pixels per run
  __half* out_planes; int64_t out_pitch; int out_run_planes;   // EPI 4
  float* out_f32;                                               // EPI 3
  int n_split; float* part;                                     // K slices; EPI 5: [n_split][rows][M][n_valid] fp32
  int* err;                                                     // ovn_handle::d_err (EPI 4: kErrNonFiniteOperand)
};

// A leg pre-activation v whose ReLU the hi / lo planes cannot hold: NaN, +-inf, or a value that rounds to an infinite
// fp16 (hi = inf, lo = -inf: the next layer's MMAs make NaN of them).  fmaxf returns 0 for NaN, so without this test
// such a layer hands on ordinary-looking zeros; the kernels that write planes raise kErrNonFiniteOperand instead.
__device__ __forceinline__ bool leg_act_unstorable(float v) { return !(v < 65520.f) || v == -INFINITY; }

// Correlation operands (k_corr_wgmma): a volume is cut into row tiles of TR rows (64 for LEFT, 128 for RIGHT),
// each tile one contiguous [hi, lo][16 planes = c / 8][TR rows][8] block of fp16, zero rows past 360: the
// no-swizzle K-major layout a wgmma descriptor reads (LBO = plane pitch, SBO = 128 B).
constexpr int C6_LROWS = 64, C6_RROWS = 128;
constexpr int C6_LT = 6, C6_RT = 3;                    // LEFT tiles, RIGHT thirds (6 x 64 = 3 x 128 = 384 >= 360)
constexpr int C6_L_BYTES = 2 * 16 * C6_LROWS * 16;     // 32 KB
constexpr int C6_R_BYTES = 2 * 16 * C6_RROWS * 16;     // 64 KB
constexpr int C6_VOL_L_BYTES = C6_LT * C6_L_BYTES;
constexpr int C6_VOL_R_BYTES = C6_RT * C6_R_BYTES;

// fp32 volumes -> hi/lo fp16 split in the tiled operand layout above; one thread per (volume, plane, row)
template <int TR, int NT>
__global__ void __launch_bounds__(256)
k_pack_corr(const float* __restrict__ bank, const int32_t* __restrict__ idx, int n, __half* __restrict__ out,
            int* __restrict__ err, int32_t* __restrict__ row_bad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t per = 16 * NT * TR;
  if (i >= (int64_t)n * per) return;
  const int p = (int)(i / per);
  int r = (int)(i % per);
  const int vrow = r % (NT * TR); r /= NT * TR;
  const int pl = r;
  const int tile = vrow / TR, row = vrow % TR;
  float v[8];
  if (vrow < WF) {
    const int64_t src = (idx ? idx[p] : p);
    const float4 a = __ldg(reinterpret_cast<const float4*>(bank + (src * WF + vrow) * CF + pl * 8));
    const float4 b = __ldg(reinterpret_cast<const float4*>(bank + (src * WF + vrow) * CF + pl * 8 + 4));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
  }
  __half hi[8], lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    hi[e] = __float2half_rn(v[e]);
    lo[e] = __float2half_rn(v[e] - __half2float(hi[e]));
  }
  bool bad = false;                       // lo is finite whenever hi is
#pragma unroll
  for (int e = 0; e < 8; e += 2) bad |= h2_nonfinite(__halves2half2(hi[e], hi[e + 1]));
  if (bad) {
    if (row_bad) row_bad[p] = 1;
    else atomicCAS(err, 0, kErrNonFiniteOperand);
  }
  __half* base = out + ((size_t)p * NT + tile) * (2 * 16 * TR * 8);
  *reinterpret_cast<uint4*>(base + ((size_t)pl * TR + row) * 8) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(base + ((size_t)(16 + pl) * TR + row) * 8) = *reinterpret_cast<const uint4*>(lo);
}

// ------------------------------------------------------------------------------------------------
// Warp-level tensor-core building blocks (mma.sync m16n8k16, f16 x f16 -> f32).
// Fragment ownership (PTX ISA, "Matrix fragments for mma.m16n8k16"): g = lane / 4, t = lane % 4;
//   A (16 x 16, row-major): a0 = (g, 2t..2t+1), a1 = (g + 8, 2t..), a2 = (g, 2t + 8..), a3 = (g + 8, 2t + 8..)
//   B (16 x 8, K-major):    b0 = (k = 2t..2t+1, n = g), b1 = (k = 2t + 8.., n = g)
//   D (16 x 8):             d0, d1 = (g, 2t..2t+1), d2, d3 = (g + 8, 2t..2t+1)
// Every operand below is stored with 8 consecutive K values (16 bytes) contiguous, so each fragment
// register is one aligned 32-bit load.  A block is 4 warps; a warp owns 16 output rows.
// ------------------------------------------------------------------------------------------------
constexpr int MMA_THREADS = 128;
constexpr int MMA_ROWS = 64;                       // output rows per block (4 warps x 16)

__device__ __forceinline__ void mma16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                         uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t ld_h2(const __half* p) { return __ldg(reinterpret_cast<const unsigned int*>(p)); }

// |a - b| of two packed fp16 pairs: subtract, then clear both sign bits
__device__ __forceinline__ uint32_t absdiff_h2(uint32_t a, uint32_t b) {
  const __half2 d = __hsub2(*reinterpret_cast<const __half2*>(&a), *reinterpret_cast<const __half2*>(&b));
  return *reinterpret_cast<const uint32_t*>(&d) & 0x7fff7fffu;
}

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// ------------------------------------------------------------------------------------------------
// k_delta_conv1_wgmma -- DeltaLayer + c_conv1 without the delta tensor (83 % of the FLOPs of a pair).
//   GEMM per work unit (block, jb):  o1[g, o] = sum_{dj < 15, c < 128} |L[g, c] - R[15 jb + dj, c]| W1[dj, c, o] - mu_o1[o]
//   M = the LEFT rows g of a block (6 row tiles of 64, rows past the block masked), N = 64, K = 1920 (60 W1 slices
//   of 32 channels).  A block is a range of the flat LEFT rows g = pair * 360 + i (k4_block): in pair mode one pair's
//   360 rows; in query mode, where every pair meets the same RIGHT volume, 384 consecutive rows that may straddle
//   two pairs, so that no row tile multiplies padding except in the last block.
// Warp specialisation: warpgroup 3 is the producer (one lane issues bulk copies; the warpgroup hands its registers
// to the consumers with setmaxnreg): the LEFT rows of the current block (96 KB at most, once per block, one bulk
// copy per pair it touches), the 15 RIGHT rows of a unit (double-buffered) and W1 in groups of 5 slices (20 KB)
// through a 3-deep ring, each buffer guarded by a
// full / empty mbarrier pair.  Warpgroups 0-2 are the consumers (160 registers): warpgroup w owns row tiles w and
// w + 3 (2 x 32 fp32 accumulators per thread) and commits one group of 2 wgmma per K16 step.  The A
// operand |l - r| is synthesised in registers from the LEFT rows (kept in registers for a 32-channel chunk)
// and the broadcast RIGHT row, and multiplied by wgmma in register-A mode against the W1 slice in shared
// memory: the 66 MB delta tensor of a pair is never written.  A group of 5 slices never straddles a 32-channel
// chunk (15 dj each), so the slice loop is unrolled straight-line code whose W1 descriptors and RIGHT rows are
// fixed offsets from bases computed once per group; a RIGHT row is one 128-bit load (k4_pos).  The accumulators
// start at the fp16-rounded -mu_o1 (the centre that k_fold_bias2 pushes through c_conv2).  Output: fp16 o1 tiles,
// written by the consumers into a staging buffer laid out as the tiles and stored with bulk copies by 15 lanes of a
// second producer warp, while the consumers go on with the next unit.
// Persistent: each CTA takes a contiguous range of the blocks * 24 units, ordered (block, jb).
// ------------------------------------------------------------------------------------------------
constexpr int K4_WG = 3;                               // consumer warpgroups
constexpr int K4_THREADS = (K4_WG + 1) * 128;          // + the producer warpgroup
constexpr uint32_t K4_REG_PRODUCER = 32, K4_REG_CONSUMER = 160;   // per thread: 3 x 160 + 32 = 512 per SM quarter
constexpr int K4_GROUP = 5;                            // W1 slices per bulk copy (divides the 15 dj of a chunk)
constexpr int K4_CHUNK_GROUPS = S15 / K4_GROUP;        // W1 groups per 32-channel chunk
constexpr int K4_NGROUPS = K4_STEPS / K4_GROUP;        // 12 per unit
static_assert(S15 % K4_GROUP == 0, "a W1 group within one 32-channel chunk");
constexpr int K4_RING = 3;
constexpr int K4_BSLICE = 4096;                        // bytes of W1 per slice: [4 k8][64 o][8]
constexpr int K4_BLOCK_ROWS = 2 * K4_WG * 64;          // LEFT rows of a query-mode block: the 6 row tiles
constexpr uint32_t K4_RWIN_BYTES = S15 * K4_PITCH * 2;
// Blocks start on a multiple of 24 rows (360 and 384 are), so a block row has the parity of its volume row (the
// k4_pos chunk order carries over), a block spans at most two pairs and at most 27 values of q = g / 15.
static_assert(WF % NB == 0 && K4_BLOCK_ROWS % NB == 0, "blocks start on a multiple of 24 rows");
constexpr int K4_O1S_Q = (K4_BLOCK_ROWS + S15 - 2) / S15 + 1;     // 27
// o1 staging of a unit: per di, the rows g = 15 q + di of the block at slot q - g0 / 15, exactly as they land in the
// o1 tiles (128 B each, chunk-swizzled), then 16 bytes of padding, so that the 8 rows of a fragment store (8
// consecutive g, i.e. 8 different di) hit 8 different 16-byte bank groups
constexpr int K4_O1S_PITCH = K4_O1S_Q * 64 + 8;        // fp16 per di

// Block b of the n_pairs x 360 flat LEFT rows g = pair * 360 + i: rows [g0, g0 + rows).  Pair mode (a RIGHT volume
// per pair) keeps one pair per block; query mode packs 384 rows per block, the last one partial.
struct K4Block { int g0, rows; };
__host__ __device__ __forceinline__ int k4_blocks(int n_pairs, int r_per_pair) {
  return r_per_pair ? n_pairs : (n_pairs * WF + K4_BLOCK_ROWS - 1) / K4_BLOCK_ROWS;
}
__device__ __forceinline__ K4Block k4_block(int b, int r_per_pair, int n_pairs) {
  if (r_per_pair) return {b * WF, WF};
  const int g0 = b * K4_BLOCK_ROWS;
  return {g0, min(K4_BLOCK_ROWS, n_pairs * WF - g0)};
}

struct K4Smem {
  __half L[K4_BLOCK_ROWS * K4_PITCH];
  __half Rw[2][S15 * K4_PITCH];
  __half B[K4_RING][K4_GROUP * K4_BSLICE / 2];
  __half O1s[S15 * K4_O1S_PITCH];
  MbarRing<K4_RING> w1;
  MbarRing<1> left;
  MbarRing<2> right;
  MbarRing<1> o1s;
};
static_assert(sizeof(K4Smem) <= 232448, "k_delta_conv1_wgmma shared memory");
static_assert(offsetof(K4Smem, B) % 16 == 0 && offsetof(K4Smem, Rw) % 16 == 0 && offsetof(K4Smem, O1s) % 16 == 0 &&
              K4_O1S_PITCH * 2 % 16 == 0, "bulk-copy alignment");

// [begin, end) of the contiguous share of n work items that part `part` of `parts` takes (a persistent CTA)
struct Share { int64_t begin, end; };
__device__ __forceinline__ Share work_share(int64_t n, uint32_t part, uint32_t parts) {
  return {n * part / parts, n * (part + 1) / parts};
}

__global__ void __launch_bounds__(K4_THREADS, 1)
k_delta_conv1_wgmma(const __half* __restrict__ L16, const int32_t* __restrict__ l_idx, const __half* __restrict__ R16,
                    int r_per_pair, const __half* __restrict__ W1p, const float* __restrict__ mu_o1,
                    __half* __restrict__ o1, int n_pairs, int* __restrict__ err) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  K4Smem& S = *reinterpret_cast<K4Smem*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const Share share = work_share((int64_t)k4_blocks(n_pairs, r_per_pair) * NB, blockIdx.x, gridDim.x);
  const int u_begin = (int)share.begin, u_end = (int)share.end;
  if (tid == 0) {
    S.w1.init(K4_WG * 4);
    S.left.init(K4_WG * 4);
    S.right.init(K4_WG * 4);
    S.o1s.init(1, K4_WG * 4);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= K4_WG * 4) {
    // ===================== producer ==========================================================
    setmaxnreg_dec<K4_REG_PRODUCER>();
    if (warp == K4_WG * 4 && lane == 0) {
      uint32_t pi = 0, gi = 0, ui = 0;
      for (int u = u_begin; u < u_end; ++u, ++ui) {
        const int b = u / NB, jb = u - b * NB;
        if (u == u_begin || jb == 0) {
          // rows [i0, i0 + n1) of pair p, then the block's rest from the start of pair p + 1
          const K4Block blk = k4_block(b, r_per_pair, n_pairs);
          const int p = blk.g0 / WF, i0 = blk.g0 - p * WF, n1 = min(blk.rows, WF - i0);
          PIPE_WAIT(S.left.acquire(pi, blk.rows * K4_PITCH * 2), kErrDeltaLeftProducer);
          bulk_g2s(S.L, L16 + ((size_t)(l_idx ? l_idx[p] : p) * WF + i0) * K4_PITCH, n1 * K4_PITCH * 2, S.left.bar(pi));
          if (n1 < blk.rows)
            bulk_g2s(S.L + n1 * K4_PITCH, L16 + (size_t)(l_idx ? l_idx[p + 1] : p + 1) * WF * K4_PITCH,
                     (blk.rows - n1) * K4_PITCH * 2, S.left.bar(pi));
          ++pi;
        }
        PIPE_WAIT(S.right.acquire(ui, K4_RWIN_BYTES), kErrDeltaRightProducer);
        bulk_g2s(S.Rw[S.right.slot(ui)], R16 + (r_per_pair ? (size_t)b * WF * K4_PITCH : 0) + (size_t)jb * S15 * K4_PITCH,
                 K4_RWIN_BYTES, S.right.bar(ui));
        for (int grp = 0; grp < K4_NGROUPS; ++grp, ++gi) {
          PIPE_WAIT(S.w1.acquire(gi, K4_GROUP * K4_BSLICE), kErrDeltaW1Producer);
          bulk_g2s(S.B[S.w1.slot(gi)], W1p + (size_t)grp * K4_GROUP * (K4_BSLICE / 2), K4_GROUP * K4_BSLICE, S.w1.bar(gi));
        }
      }
    } else if (warp == K4_WG * 4 + 1) {
      // o1 stores, lane di of producer warp 1 for di < 15 (the warp shares its SM sub-partition's issue slots with
      // consumer warps, so the 15 store loops run side by side): per unit, the block's rows g = 15 q + di,
      // q in [qa, qb], land at o1 rows m = (q / 24) * 576 + jb * 24 + q % 24, one contiguous run per pair, each
      // split in two where it crosses a 128-row o1 block (576 = 4.5 x 128), so up to 4 bulk copies per lane.  Each
      // lane waits for its own copies to have read the staging buffer; lane 0 then frees it.
      const int di = lane;
      uint32_t ui = 0;
      for (int u = u_begin; u < u_end; ++u, ++ui) {
        const int b = u / NB, jb = u - b * NB;
        const K4Block blk = k4_block(b, r_per_pair, n_pairs);
        if (!__all_sync(0xffffffffu, S.o1s.wait(ui))) {
          if (lane == 0) atomicExch(err, kErrDeltaO1Producer);
          break;
        }
        if (di < S15) {
          const int q0 = blk.g0 / S15, qb = (blk.g0 + blk.rows - 1 - di) / S15;
#pragma unroll 1
          for (int q = (blk.g0 + S15 - 1 - di) / S15; q <= qb;) {
            const int p = q / NB, ib = q - p * NB, len = min(qb - q + 1, NB - ib);
            const int64_t m = (int64_t)p * PAIR_ROWS + jb * NB + ib;
            const int n0 = min(len, 128 - (int)(m & 127));
            const __half* src = S.O1s + di * K4_O1S_PITCH + (q - q0) * 64;
            bulk_s2g(o1 + o1_row_offset(m, di), src, n0 * 128);
            if (n0 < len) bulk_s2g(o1 + o1_row_offset(m + n0, di), src + n0 * 64, (len - n0) * 128);
            q += len;
          }
          bulk_commit();
          bulk_wait_read<0>();
        }
        __syncwarp();
        if (lane == 0) S.o1s.release_thread(ui);
      }
      if (di < S15) bulk_wait<0>();           // the next kernel reads o1
    }
  } else {
    // ===================== consumers ==========================================================
    setmaxnreg_inc<K4_REG_CONSUMER>();
    const int wg = warp >> 2, wi = warp & 3, g = lane >> 2, t = lane & 3;
    int rows[2][2];                         // [tile][a / b]: this thread's fragment rows
#pragma unroll
    for (int tt = 0; tt < 2; ++tt) {
      const int r = (wg + 3 * tt) * 64 + wi * 16 + g;
      rows[tt][0] = r;
      rows[tt][1] = r + 8;
    }
    const uint32_t b_base = smem_u32(S.B[0]);
    uint32_t pi = 0, gi = 0, ui = 0;
    uint32_t sto[2][2][8];                  // byte offsets of this thread's 32 o1 staging stores, set once per block
    for (int u = u_begin; u < u_end; ++u, ++ui) {
      const int b = u / NB, jb = u - b * NB;
      const K4Block blk = k4_block(b, r_per_pair, n_pairs);
      if (u == u_begin || jb == 0) {
        PIPE_WAIT(S.left.wait(pi), kErrDeltaLeftConsumer);
        ++pi;
        // Row g = 15 q + di of the block is staged at slot q - g0 / 15 of di and lands at o1 row
        // m = (q / 24) * 576 + jb * 24 + ib with ib = q % 24, so its chunk swizzle m & 7 is ib & 7 for every jb.
#pragma unroll
        for (int tt = 0; tt < 2; ++tt)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int g = blk.g0 + rows[tt][h], q = g / S15, di = g - q * S15, ib = q % NB;
            const uint32_t st = (uint32_t)offsetof(K4Smem, O1s) + 2 * (di * K4_O1S_PITCH + (q - blk.g0 / S15) * 64 + 2 * t);
#pragma unroll
            for (int j = 0; j < 8; ++j) sto[tt][h][j] = st + ((j ^ (ib & 7)) << 4);
          }
      }
      const uint32_t wb = S.right.slot(ui);
      PIPE_WAIT(S.right.wait(ui), kErrDeltaRightConsumer);
      float acc[2][32];
#pragma unroll
      for (int j = 0; j < 8; ++j) {             // read per unit rather than held in 16 registers across the loop
        const float m0 = __half2float(__float2half_rn(-__ldg(mu_o1 + j * 8 + 2 * t)));
        const float m1 = __half2float(__float2half_rn(-__ldg(mu_o1 + j * 8 + 2 * t + 1)));
#pragma unroll
        for (int tt = 0; tt < 2; ++tt) {
          acc[tt][4 * j + 0] = m0; acc[tt][4 * j + 1] = m1;
          acc[tt][4 * j + 2] = m0; acc[tt][4 * j + 3] = m1;
        }
      }
      uint32_t Lr[2][2][4];                   // LEFT values of the chunk: [tile][row a / b][kk0 lo, hi, kk1 lo, hi]
#pragma unroll 1
      for (int grp = 0; grp < K4_NGROUPS; ++grp, ++gi) {
        const int cc = grp / K4_CHUNK_GROUPS, dj0 = (grp - K4_CHUNK_GROUPS * cc) * K4_GROUP;
        if (dj0 == 0) {
#pragma unroll
          for (int tt = 0; tt < 2; ++tt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = rows[tt][h] < blk.rows ? rows[tt][h] : blk.rows - 1;
              const uint4 v = *reinterpret_cast<const uint4*>(S.L + r * K4_PITCH + ((cc ^ (r & 1)) << 5) + 8 * t);
              Lr[tt][h][0] = v.x; Lr[tt][h][1] = v.y; Lr[tt][h][2] = v.z; Lr[tt][h][3] = v.w;
            }
        }
        const uint32_t s = S.w1.slot(gi);
        // slice sl of the stage, K16 step kk: W1 chunks k8 = 2 kk, 2 kk + 1 (LBO = 1024 B between them, SBO = 128 B
        // per 8 outputs) at sl * 4096 + kk * 2048 bytes, i.e. (sl * 4096 + kk * 2048) >> 4 in the descriptor
        const uint64_t bdesc = desc_kmajor(b_base + s * (K4_GROUP * K4_BSLICE), 1024, 128, kNoSwizzle);
        // RIGHT row dj0 + sl of the window is row 15 jb + dj0 + sl of the volume: its chunks are swapped when odd
        const int par = (jb + dj0) & 1;
        const __half* rw = S.Rw[wb] + dj0 * K4_PITCH + 8 * t;
        const __half* rp[2] = {rw + ((cc ^ par) << 5), rw + ((cc ^ par ^ 1) << 5)};
        uint4 rv = *reinterpret_cast<const uint4*>(rp[0]);
        PIPE_WAIT(S.w1.wait(gi), kErrDeltaW1Consumer);
        // One commit group per K16 step, waited for with wait_group 1: a warpgroup forms step kk's A while its
        // previous step's MMAs run.  A[.][kk] is rewritten only after the group that last read it (two groups back)
        // has retired.  Every group is drained at the end of the W1 group: ptxas keeps register-A wgmmas pipelined
        // only when no group is in flight across the loop's back edge or a barrier wait.
        uint32_t A[2][2][4];                  // [tile][kk]
#pragma unroll
        for (int sl = 0; sl < K4_GROUP; ++sl)
#pragma unroll
          for (int kk = 0; kk < 2; ++kk) {
            const uint32_t r0 = kk ? rv.z : rv.x, r1 = kk ? rv.w : rv.y;
#pragma unroll
            for (int tt = 0; tt < 2; ++tt) {
              A[tt][kk][0] = absdiff_h2(Lr[tt][0][2 * kk], r0);
              A[tt][kk][1] = absdiff_h2(Lr[tt][1][2 * kk], r0);
              A[tt][kk][2] = absdiff_h2(Lr[tt][0][2 * kk + 1], r1);
              A[tt][kk][3] = absdiff_h2(Lr[tt][1][2 * kk + 1], r1);
            }
            wgmma_fence();
#pragma unroll
            for (int tt = 0; tt < 2; ++tt)
              wgmma_m64n64k16_rs(acc[tt], A[tt][kk], bdesc + ((sl * K4_BSLICE + kk * 2048) >> 4));
            wgmma_commit();
            // the next RIGHT row loads while the MMAs run
            if (kk == 1 && sl + 1 < K4_GROUP) rv = *reinterpret_cast<const uint4*>(rp[(sl + 1) & 1] + (sl + 1) * K4_PITCH);
            wgmma_wait<1>();
          }
        wgmma_wait<0>();
        S.w1.release(gi);
      }
      S.right.release(ui);
      if (jb == NB - 1 || u == u_end - 1) S.left.release(pi - 1);
      // o1 into the staging buffer, once the store warp's copies of the previous unit have read it
      if (!S.o1s.wait_free(ui)) { atomicExch(err, kErrDeltaO1Consumer); goto done; }
#pragma unroll
      for (int tt = 0; tt < 2; ++tt)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (rows[tt][h] >= blk.rows) continue;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<uint32_t*>(smem_raw + sto[tt][h][j]) = pack_h2(acc[tt][4 * j + 2 * h], acc[tt][4 * j + 2 * h + 1]);
        }
      fence_proxy_async_smem();
      S.o1s.publish(ui);
    }
  }
done:
  return;
}

// ------------------------------------------------------------------------------------------------
// k_conv2_wgmma -- c_conv2 (15x1 stride 15, 64 -> 128, ReLU) as a GEMM [M x 960] x [960 x 128], W2 applied as
// hi + lo (two MMAs per K16 step into the same accumulators: the fp16 rounding of W2 was the largest term of
// the logit error budget after the feature volumes).  A = the o1 tiles k_delta_conv1_wgmma wrote; output = the
// centred fp16 x3 planes.
// Persistent and warp-specialised: a CTA walks a contiguous range of 256-row tiles.  Warp 8 is the producer
// (one lane): per di it bulk-copies the two 16 KB o1 tiles of the 256 rows and the 32 KB W2 hi + lo tiles of
// that di into a 3-deep ring (full / empty mbarrier pairs).  Warpgroups 0 and 1 own 128 rows each (2 x m64n128
// fp32 accumulators) and multiply straight out of the SWIZZLE_128B tiles (wgmma, both operands in shared
// memory), one commit group per di with the previous di's group still in flight.  256 rows per tile because
// W2 hi + lo (480 KB) is re-read from L2 for every tile: at 128 rows that traffic would be twice the o1 read.
// `fault` != 0 is the test hook of ovn_debug_inject_fault: the kernel computes nothing and raises the
// pipeline-failure flag, so that the finalize kernels poison the outputs of the call.
// ------------------------------------------------------------------------------------------------
constexpr int TC_WG = 2;                               // consumer warpgroups of k_conv2_wgmma / k_conv3_wgmma
constexpr int TC_THREADS = TC_WG * 128 + 32;           // + the producer warp
constexpr int TC_ROWS = TC_WG * 128;                   // output rows per tile
constexpr uint32_t C2_TILE = 128 * 64 * 2;             // bytes of one SWIZZLE_128B tile: 128 rows x 64 fp16
constexpr int C2_RING = 3;

struct C2Smem {
  __half A[C2_RING][TC_WG][C2_TILE / 2];               // o1 of one di: rows [r0, r0 + 128), [r0 + 128, r0 + 256)
  __half B[C2_RING][2][C2_TILE / 2];                   // W2 of that di: hi, lo
  MbarRing<C2_RING> ring;
};
constexpr size_t C2_SMEM = sizeof(C2Smem) + 1024;      // + the round-up of the base to a 1024-byte swizzle atom
static_assert(C2_SMEM <= 232448, "k_conv2_wgmma shared memory");
static_assert(offsetof(C2Smem, B) % 1024 == 0 && C2_TILE % 1024 == 0, "SWIZZLE_128B tiles on 1024-byte boundaries");

__global__ void __launch_bounds__(TC_THREADS, 1)
k_conv2_wgmma(const __half* __restrict__ o1, const __half* __restrict__ W2s, const float* __restrict__ bias2,
              const float* __restrict__ mu_x3, __half* __restrict__ x3, int64_t out_pitch, int64_t M, int fault,
              int* __restrict__ err) {
  if (fault) {
    if (threadIdx.x == 0 && blockIdx.x == 0) atomicExch(err, kErrInjectedFault);
    return;
  }
  extern __shared__ __align__(128) uint8_t smem_raw[];
  C2Smem& S = *reinterpret_cast<C2Smem*>(smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const Share tiles = work_share((M + TC_ROWS - 1) / TC_ROWS, blockIdx.x, gridDim.x);
  if (tid == 0) {
    S.ring.init(TC_WG * 4);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == TC_WG * 4) {
    // ===================== producer ==========================================================
    if (lane == 0) {
      uint32_t gi = 0;
      for (int64_t tile = tiles.begin; tile < tiles.end; ++tile)
        for (int di = 0; di < S15; ++di, ++gi) {
          const uint32_t s = S.ring.slot(gi);
          PIPE_WAIT(S.ring.acquire(gi, 4 * C2_TILE), kErrConv2Producer);
          for (int h = 0; h < TC_WG; ++h)      // o1 tile (m / 128, di) of the rows m = 256 tile + 128 h + [0, 128)
            bulk_g2s(S.A[s][h], o1 + ((size_t)(tile * TC_WG + h) * S15 + di) * (C2_TILE / 2), C2_TILE, S.ring.bar(gi));
          bulk_g2s(S.B[s], W2s + (size_t)di * C2_TILE, 2 * C2_TILE, S.ring.bar(gi));
        }
    }
  } else {
    // ===================== consumers ==========================================================
    const int wg = warp >> 2, wi = warp & 3, g = lane >> 2, t = lane & 3;
    uint32_t gi = 0;
    bool failed = false;
    for (int64_t tile = tiles.begin; tile < tiles.end; ++tile) {
      float acc[2][64];                       // [m64 sub-tile][D fragment]
#pragma unroll
      for (int sub = 0; sub < 2; ++sub)
#pragma unroll
        for (int e = 0; e < 64; ++e) acc[sub][e] = 0.f;
#pragma unroll 1
      for (int di = 0; di < S15; ++di, ++gi) {
        const uint32_t s = S.ring.slot(gi);
        INFLIGHT_WAIT(S.ring.wait(gi), kErrConv2Consumer);
        const uint32_t a_base = smem_u32(S.A[s][wg]), b_base = smem_u32(S.B[s][0]);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
          for (int part = 0; part < 2; ++part) {  // W2 hi, then lo
            const uint64_t bd = desc_kmajor(b_base + part * C2_TILE + kk * 32, 16, 1024, kSwizzle128B);
#pragma unroll
            for (int sub = 0; sub < 2; ++sub)     // rows 64 sub + [0, 64) of this warpgroup: 8 KB into the tile
              wgmma_m64n128k16_ss(acc[sub], desc_kmajor(a_base + sub * (C2_TILE / 2) + kk * 32, 16, 1024, kSwizzle128B), bd);
          }
        wgmma_commit();
        wgmma_wait<1>();                      // the previous di's group is done: its stage can be refilled
        if (di > 0) S.ring.release(gi - 1);
      }
      wgmma_wait<0>();
      if (failed) goto done;
      S.ring.release(gi - 1);
      // b2eff, ReLU, minus the x3 centre, fp16 into the C8-interleaved planes (rows past M are not stored)
#pragma unroll
      for (int sub = 0; sub < 2; ++sub)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int64_t m = tile * TC_ROWS + wg * 128 + sub * 64 + wi * 16 + g + 8 * h;
          if (m >= M) continue;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int n = j * 8 + 2 * t;
            const float a = fmaxf(acc[sub][4 * j + 2 * h] + __ldg(bias2 + n), 0.f) - __ldg(mu_x3 + n);
            const float b = fmaxf(acc[sub][4 * j + 2 * h + 1] + __ldg(bias2 + n + 1), 0.f) - __ldg(mu_x3 + n + 1);
            *reinterpret_cast<uint32_t*>(x3 + ((size_t)j * out_pitch + m) * 8 + 2 * t) = pack_h2(a, b);
          }
        }
    }
  }
done:
  return;
}

// ------------------------------------------------------------------------------------------------
// k_conv3_wgmma -- c_conv3 (3x3, 128 -> 256, ReLU) + Flatten + the Dense(1) partial sum of each row.
// Rows are (pair, jb, ib) in the x3 planes; the 3x3 tap (a, b) reads row r + a * 24 + b (implicit im2col).
// partial[r][nh] = sum over the 128 channels of half nh of relu(conv + b3eff) * w_dense (0 for the
// rows a valid convolution does not produce).
// Persistent and warp-specialised; a tile is 256 output rows x one half nh of the output channels, and the
// two halves of a row block are consecutive tiles of one CTA (the second finds its x3 rows in L2).  Warp 8 is
// the producer (one lane): the 16 x3 planes of rows [r0, r0 + 306), one 4.9 KB bulk copy per plane (78 KB,
// double-buffered and issued a tile ahead), and W3 half nh in stages of two (tap, 32-channel) slabs (16 KB)
// through a 4-deep ring.  The x3 planes are the no-swizzle K-major layout a descriptor reads (8 rows x 16 B
// core matrices, LBO = plane pitch, SBO = 128 B), so all 9 taps read the same stage from a start address
// shifted by a * 24 + b rows.  Warpgroups 0 and 1 own 128 rows each (2 x m64n128 fp32 accumulators).
// 256 rows per tile because W3 half nh (288 KB) is re-read from L2 for every tile.
// ------------------------------------------------------------------------------------------------
constexpr int C3_AROWS = TC_ROWS + 2 * NB + 2;         // + the reach of the 3x3 window
constexpr uint32_t C3_PLANE = C3_AROWS * 16;           // bytes of one x3 plane in shared memory
constexpr uint32_t C3_SLAB = 4 * 128 * 16;             // W3 slab (tap, 32 channels) x 128 outputs: [4 k8][128 n][8]
constexpr int C3_GROUP = 2;                            // slabs per ring stage
constexpr int C3_NSTAGES = 36 / C3_GROUP;              // ring stages per tile
constexpr int C3_RING = 4;

struct C3Smem {
  __half A[2][16 * C3_PLANE / 2];                      // [buffer][plane c / 8][row][8]
  __half B[C3_RING][C3_GROUP * C3_SLAB / 2];
  MbarRing<C3_RING> w3;
  MbarRing<2> x3;
};
static_assert(sizeof(C3Smem) <= 232448, "k_conv3_wgmma shared memory");
static_assert(offsetof(C3Smem, B) % 16 == 0 && C3_PLANE % 16 == 0, "bulk-copy alignment");

__global__ void __launch_bounds__(TC_THREADS, 1)
k_conv3_wgmma(const __half* __restrict__ X3, int64_t a_pitch, const __half* __restrict__ W3p, const float* __restrict__ bias,
              int64_t M, const float* __restrict__ wd, float* __restrict__ partial, int* __restrict__ err) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  C3Smem& S = *reinterpret_cast<C3Smem*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const Share tiles = work_share(2 * ((M + TC_ROWS - 1) / TC_ROWS), blockIdx.x, gridDim.x);   // 2 * row block + nh
  if (tid == 0) {
    S.w3.init(TC_WG * 4);
    S.x3.init(TC_WG * 4);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == TC_WG * 4) {
    // ===================== producer ==========================================================
    if (lane == 0) {
      const uint32_t nt = (uint32_t)(tiles.end - tiles.begin);
      uint32_t ai = 0, gi = 0;                // tiles whose x3 rows were issued, W3 stages issued
      for (uint32_t ti = 0; ti < nt; ++ti) {
        const int nh = (int)((tiles.begin + ti) & 1);
        for (int st = 0; st < C3_NSTAGES; ++st, ++gi) {
          // x3 rows of this tile (must go now) and of the next one (as soon as its buffer is free, i.e. once
          // the tile before this one is done), so that they load while this tile computes
          while (ai < nt && ai <= ti + 1) {
            if (ai > ti) {
              if (!S.x3.try_acquire(ai, 16 * C3_PLANE)) break;
            } else {
              PIPE_WAIT(S.x3.acquire(ai, 16 * C3_PLANE), kErrConv3X3Producer);
            }
            const int64_t r0 = ((tiles.begin + ai) >> 1) * TC_ROWS;
            for (int pl = 0; pl < 16; ++pl)
              bulk_g2s(S.A[S.x3.slot(ai)] + pl * (C3_PLANE / 2), X3 + ((size_t)pl * a_pitch + r0) * 8, C3_PLANE, S.x3.bar(ai));
            ++ai;
          }
          PIPE_WAIT(S.w3.acquire(gi, C3_GROUP * C3_SLAB), kErrConv3W3Producer);
          bulk_g2s(S.B[S.w3.slot(gi)], W3p + ((size_t)nh * 36 + st * C3_GROUP) * (C3_SLAB / 2), C3_GROUP * C3_SLAB,
                   S.w3.bar(gi));
        }
      }
    }
  } else {
    // ===================== consumers ==========================================================
    const int wg = warp >> 2, wi = warp & 3, g = lane >> 2, t = lane & 3;
    const uint32_t b_base = smem_u32(S.B[0]);
    uint32_t gi = 0;
    bool failed = false;
    for (int64_t tile = tiles.begin; tile < tiles.end; ++tile) {
      const uint32_t ti = (uint32_t)(tile - tiles.begin);
      const int nh = (int)(tile & 1);
      const int64_t r0 = (tile >> 1) * TC_ROWS;
      PIPE_WAIT(S.x3.wait(ti), kErrConv3X3Consumer);
      const uint32_t a_rows = smem_u32(S.A[S.x3.slot(ti)]) + wg * 128 * 16;
      float acc[2][64];                       // [m64 sub-tile][D fragment]
#pragma unroll
      for (int sub = 0; sub < 2; ++sub)
#pragma unroll
        for (int e = 0; e < 64; ++e) acc[sub][e] = 0.f;
#pragma unroll 1
      for (int st = 0; st < C3_NSTAGES; ++st, ++gi) {
        const uint32_t s = S.w3.slot(gi);
        INFLIGHT_WAIT(S.w3.wait(gi), kErrConv3W3Consumer);
        wgmma_fence();
#pragma unroll
        for (int sl = 0; sl < C3_GROUP; ++sl) {
          // slab = tap * 4 + c / 32; the x3 image is stored transposed, tap = a * 3 + b shifts by a * 24 + b rows
          const int slab = st * C3_GROUP + sl, tap = slab >> 2, c32 = slab & 3;
          const uint32_t a_tap = a_rows + ((tap / 3) * NB + tap % 3) * 16;
          const uint32_t slab_addr = b_base + s * (C3_GROUP * C3_SLAB) + sl * C3_SLAB;
#pragma unroll
          for (int kk = 0; kk < 2; ++kk) {    // K16 step = planes 2 c16, 2 c16 + 1 = W3 k8 chunks 2 kk, 2 kk + 1
            const int c16 = c32 * 2 + kk;
            const uint64_t bd = desc_kmajor(slab_addr + kk * 4096, 2048, 128, kNoSwizzle);
#pragma unroll
            for (int sub = 0; sub < 2; ++sub)
              wgmma_m64n128k16_ss(acc[sub], desc_kmajor(a_tap + 2 * c16 * C3_PLANE + sub * 64 * 16, C3_PLANE, 128, kNoSwizzle), bd);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                      // the previous stage's group is done: its slot can be refilled
        if (st > 0) S.w3.release(gi - 1);
      }
      wgmma_wait<0>();
      if (failed) goto done;
      S.w3.release(gi - 1);
      S.x3.release(ti);
#pragma unroll
      for (int sub = 0; sub < 2; ++sub)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int64_t r = r0 + wg * 128 + sub * 64 + wi * 16 + g + 8 * h;
          const int rem = (int)(r % PAIR_ROWS);
          const int yy = rem / NB, xx = rem - yy * NB;
          const bool valid = (r < M) && (yy < NB - 2) && (xx < NB - 2);
          // rows are (pair, jb, ib): yy = jb, xx = ib; Flatten order of the reference is (ib, jb, channel)
          const float* wrow = wd + (size_t)(valid ? (xx * (NB - 2) + yy) : 0) * 256 + nh * 128;
          float sum = 0.f;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int n = j * 8 + 2 * t;
            sum = fmaf(fmaxf(acc[sub][4 * j + 2 * h] + __ldg(bias + nh * 128 + n), 0.f), __ldg(wrow + n), sum);
            sum = fmaf(fmaxf(acc[sub][4 * j + 2 * h + 1] + __ldg(bias + nh * 128 + n + 1), 0.f), __ldg(wrow + n + 1), sum);
          }
          sum += __shfl_xor_sync(0xffffffffu, sum, 1);
          sum += __shfl_xor_sync(0xffffffffu, sum, 2);
          if (t == 0 && r < M) partial[r * 2 + nh] = valid ? sum : 0.f;
        }
    }
  }
done:
  return;
}

// ------------------------------------------------------------------------------------------------
// k_corr_wgmma -- correlation (yaw) head.  G = L R^T (360 x 360, K = 128) from hi / lo fp16 operands
// (G = Lhi Rhi + Llo Rhi + Lhi Rlo: fp32-grade, fp16 alone does not keep the argmax of a flat curve),
// corr[k] = sum_j G[(k + j + 180) mod 360, j]: row i meets column j in bin k = (i - j - 180) mod 360.
// A work unit is one 64-row LEFT tile a of a pair against one 128-row RIGHT third q (m64 x n128, K = 128).
// Persistent and warp-specialised: CTA b serves the third q = b % 3 and walks a contiguous range of the
// n_pairs * 6 (pair, a) units; the CTAs 3c, 3c + 1, 3c + 2 walk the same range at the same pace, so a LEFT
// tile is read from HBM once and served to the other two thirds from L2.  Warp 8 is the producer (one lane):
// the RIGHT third (64 KB, once per CTA in query mode, once per pair in pair mode) and the LEFT tiles (32 KB,
// hi + lo) through a 3-deep ring.  Consumer warpgroups 0 and 1 take alternate units: 24 wgmma.m64n128k16
// (K16 steps in order, each as Lhi Rhi, Llo Rhi, Lhi Rlo), then the 64 x 128 block of G goes to the
// warpgroup's own shared-memory buffer and each of its 191 diagonals is summed in a fixed order into
// corr_part[pair][a][q][k] (the 169 bins the block does not reach are 0), while the other warpgroup
// multiplies.  k_corr_finalize adds the 18 partial curves of a pair in a fixed order: no atomics, results
// are bit-reproducible, and query mode gives the bits of pair mode.
// ------------------------------------------------------------------------------------------------
constexpr int C6_PARTS = C6_LT * C6_RT;                // partial curves per pair
constexpr int C6_WG = 2;
constexpr int C6_THREADS = C6_WG * 128 + 32;
constexpr int C6_RING = 3;
constexpr int C6_GPITCH = 132;                         // fp32 row pitch of a staged G block

struct C6Smem {
  __half R[C6_R_BYTES / 2];
  __half L[C6_RING][C6_L_BYTES / 2];
  float G[C6_WG][C6_LROWS * C6_GPITCH];
  MbarRing<C6_RING> left;
  MbarRing<1> right;
};
static_assert(sizeof(C6Smem) <= 232448, "k_corr_wgmma shared memory");
static_assert(offsetof(C6Smem, L) % 16 == 0, "bulk-copy alignment");

__global__ void __launch_bounds__(C6_THREADS, 1)
k_corr_wgmma(const __half* __restrict__ Lc, const int32_t* __restrict__ l_idx, const __half* __restrict__ Rc,
             int r_per_pair, int n_pairs, float* __restrict__ corr_part, int* __restrict__ err) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  C6Smem& S = *reinterpret_cast<C6Smem*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q = blockIdx.x % C6_RT;
  const Share share = work_share((int64_t)n_pairs * C6_LT, blockIdx.x / C6_RT, gridDim.x / C6_RT);
  const int u_begin = (int)share.begin, u_end = (int)share.end;
  if (tid == 0) {
    S.left.init(4);                           // one warpgroup per unit
    S.right.init(C6_WG * 4);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == C6_WG * 4) {
    // ===================== producer ==========================================================
    if (lane == 0) {
      uint32_t ri = 0, ui = 0;
      int key = -1;                           // pair whose RIGHT third is loaded (0 in query mode)
      for (int u = u_begin; u < u_end; ++u, ++ui) {
        const int p = u / C6_LT, a = u - p * C6_LT;
        if ((r_per_pair ? p : 0) != key) {
          key = r_per_pair ? p : 0;
          PIPE_WAIT(S.right.acquire(ri, C6_R_BYTES), kErrCorrRightProducer);
          bulk_g2s(S.R, Rc + ((size_t)key * C6_RT + q) * (C6_R_BYTES / 2), C6_R_BYTES, S.right.bar(ri));
          ++ri;
        }
        PIPE_WAIT(S.left.acquire(ui, C6_L_BYTES), kErrCorrLeftProducer);
        bulk_g2s(S.L[S.left.slot(ui)], Lc + ((size_t)(l_idx ? l_idx[p] : p) * C6_LT + a) * (C6_L_BYTES / 2), C6_L_BYTES,
                 S.left.bar(ui));
      }
    }
  } else {
    // ===================== consumers ==========================================================
    // A time-out raises the error and skips the later waits, but the warp keeps to the named barriers of its
    // warpgroup (the outputs of the call are poisoned by the flag).
    const int wg = warp >> 2, wi = warp & 3, g = lane >> 2, t = lane & 3, tw = tid & 127;
    float* Gw = S.G[wg];
    const uint32_t r_base = smem_u32(S.R);
    uint32_t ri = 0, ui = 0;
    int key = -1;
    bool failed = false;
    for (int u = u_begin; u < u_end; ++u, ++ui) {
      const int p = u / C6_LT, a = u - p * C6_LT;
      if ((r_per_pair ? p : 0) != key) {      // both warpgroups follow every change of the RIGHT third
        if (key >= 0) S.right.release(ri - 1);
        key = r_per_pair ? p : 0;
        INFLIGHT_WAIT(S.right.wait(ri), kErrCorrRightConsumer);
        ++ri;
      }
      if ((int)(ui & 1) != wg) continue;
      const uint32_t s = S.left.slot(ui);
      INFLIGHT_WAIT(S.left.wait(ui), kErrCorrLeftConsumer);
      const uint32_t l_base = smem_u32(S.L[s]);
      float acc[64];
#pragma unroll
      for (int e = 0; e < 64; ++e) acc[e] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int c16 = 0; c16 < 8; ++c16) {
        // K16 step = planes 2 c16, 2 c16 + 1: LBO = plane pitch, SBO = 8 rows x 16 B
        const uint64_t ah = desc_kmajor(l_base + c16 * 2 * C6_LROWS * 16, C6_LROWS * 16, 128, kNoSwizzle);
        const uint64_t al = desc_kmajor(l_base + C6_L_BYTES / 2 + c16 * 2 * C6_LROWS * 16, C6_LROWS * 16, 128, kNoSwizzle);
        const uint64_t bh = desc_kmajor(r_base + c16 * 2 * C6_RROWS * 16, C6_RROWS * 16, 128, kNoSwizzle);
        const uint64_t bl = desc_kmajor(r_base + C6_R_BYTES / 2 + c16 * 2 * C6_RROWS * 16, C6_RROWS * 16, 128, kNoSwizzle);
        wgmma_m64n128k16_ss(acc, ah, bh);
        wgmma_m64n128k16_ss(acc, al, bh);
        wgmma_m64n128k16_ss(acc, ah, bl);
      }
      wgmma_commit();
      wgmma_wait<0>();
      S.left.release(ui);
      named_bar_sync(1 + wg, 128);           // this warpgroup's previous diagonal sums have read Gw
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float* r0 = Gw + (wi * 16 + g) * C6_GPITCH + j * 8 + 2 * t;
        *reinterpret_cast<float2*>(r0) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(r0 + 8 * C6_GPITCH) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
      named_bar_sync(1 + wg, 128);
      const int i_lim = min(C6_LROWS, WF - a * C6_LROWS), j_lim = min(C6_RROWS, WF - q * C6_RROWS);
      float* out = corr_part + ((size_t)p * C6_PARTS + a * C6_RT + q) * WF;
      for (int d = tw; d < WF; d += 128) {
        // diagonal i - j = d - 127 of the block: d < 191 covers all of them, the other bins get 0
        const int dd = d - (C6_RROWS - 1);
        float sum = 0.f;
        if (d < C6_LROWS + C6_RROWS - 1) {
#pragma unroll 8
          for (int ii = 0; ii < C6_LROWS; ++ii) {
            const int jj = ii - dd;
            if (ii < i_lim && jj >= 0 && jj < j_lim) sum += Gw[ii * C6_GPITCH + jj];
          }
        }
        int k = (a * C6_LROWS - q * C6_RROWS + dd - WF / 2) % WF;
        if (k < 0) k += WF;
        out[k] = sum;
      }
    }
  }
done:
  return;
}

// ------------------------------------------------------------------------------------------------
// k_leg_mma -- one leg layer (2..) on the hi / lo fp16 C8-interleaved activation planes:
//   out[y, px, n] = relu(bias[n] + sum_{dh, dw, c} x[y * sh + dh, px + dw, c] W[dh, dw, c, n]),
//   x * w ~= xh wh + xl wh + xh wl  (three MMAs per K16 step, fp32-grade).
// EPI 4: output as the next layer's hi / lo planes; EPI 3 (last layer): fp32 feature volume; EPI 5: the fp32
// sum over K slice `slice` of the layer (no bias), combined by k_leg_splitk_reduce.
// K is walked as (tap = dh * kw + dw, c8) in that order; slice s of n_split takes the iterations
// [it * s / n_split, it * (s + 1) / n_split) of that walk.
// grid = (n_img * h_out, ceil(M / 64), n_split * cout / 64), blockIdx.z = slice * nz + z
// ------------------------------------------------------------------------------------------------
template <int EPI>
__global__ void __launch_bounds__(MMA_THREADS)
k_leg_mma(LegArgs g) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const int64_t px0 = (int64_t)blockIdx.y * MMA_ROWS + warp * 16;
  if (px0 >= g.M) return;
  const int nz = (g.n_valid + 63) / 64;
  const int y = blockIdx.x, z = blockIdx.z % nz, slice = blockIdx.z / nz;
  const int64_t in_base = (int64_t)(y / g.runs_per_img) * g.in_img_planes + (int64_t)(y % g.runs_per_img) * g.in_run_planes;
  const int64_t pa = px0 + gq < g.M ? px0 + gq : g.M - 1, pb = px0 + gq + 8 < g.M ? px0 + gq + 8 : g.M - 1;
  const int n_slabs = g.kh * g.kw * 3;
  const size_t plane = (size_t)g.a_pitch * 8;
  const int per_tap = g.c8in / 2, n_it = g.kh * g.kw * per_tap;
  const int it0 = n_it * slice / g.n_split, it1 = n_it * (slice + 1) / g.n_split;
  float acc[8][4] = {};
#pragma unroll 1
  for (int it = it0; it < it1;) {
    const int tap = it / per_tap, dh = tap / g.kw, dw = tap - dh * g.kw;
    const int c8_end = (tap + 1) * per_tap < it1 ? g.c8in : (it1 - tap * per_tap) * 2;
    {
      const __half* Ah = g.A + (size_t)(in_base + (int64_t)dh * 2 * g.c8in) * plane + (size_t)dw * 8 + 2 * t;
      const __half* Al = Ah + (size_t)g.c8in * plane;
      // [z][slab = (dh * kw + dw) * 3 + term][c8][64][8]; term 0 = hi, term 2 = lo
      const __half* Bh = g.Bp + ((size_t)(z * n_slabs + (dh * g.kw + dw) * 3) * g.c8in * 64 + gq) * 8 + 2 * t;
      const __half* Bl = Bh + (size_t)2 * g.c8in * 64 * 8;
#pragma unroll 1
      for (int c8 = (it - tap * per_tap) * 2; c8 < c8_end; c8 += 2) {
        const size_t o0 = (size_t)c8 * plane, o1 = o0 + plane;
        const uint32_t h0 = ld_h2(Ah + o0 + pa * 8), h1 = ld_h2(Ah + o0 + pb * 8), h2 = ld_h2(Ah + o1 + pa * 8), h3 = ld_h2(Ah + o1 + pb * 8);
        const uint32_t l0 = ld_h2(Al + o0 + pa * 8), l1 = ld_h2(Al + o0 + pb * 8), l2 = ld_h2(Al + o1 + pa * 8), l3 = ld_h2(Al + o1 + pb * 8);
        const size_t bo = (size_t)c8 * 64 * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint32_t wh0 = ld_h2(Bh + bo + j * 64), wh1 = ld_h2(Bh + bo + 64 * 8 + j * 64);
          const uint32_t wl0 = ld_h2(Bl + bo + j * 64), wl1 = ld_h2(Bl + bo + 64 * 8 + j * 64);
          mma16816(acc[j], h0, h1, h2, h3, wh0, wh1);
          mma16816(acc[j], l0, l1, l2, l3, wh0, wh1);
          mma16816(acc[j], h0, h1, h2, h3, wl0, wl1);
        }
      }
    }
    it = tap * per_tap + c8_end / 2;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t px = px0 + gq + 8 * h;
    if (px >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = z * 64 + j * 8 + 2 * t;
      if (n >= g.n_valid) continue;
      if (EPI == 5) {         // [slice][y][px][n_valid]
        *reinterpret_cast<float2*>(g.part + (((size_t)slice * gridDim.x + y) * g.M + px) * g.n_valid + n) =
            make_float2(acc[j][2 * h], acc[j][2 * h + 1]);
        continue;
      }
      const float pre_a = acc[j][2 * h] + __ldg(g.bias + n), pre_b = acc[j][2 * h + 1] + __ldg(g.bias + n + 1);
      const float a = fmaxf(pre_a, 0.f), b = fmaxf(pre_b, 0.f);
      if (EPI == 4) {
        if (leg_act_unstorable(pre_a) || leg_act_unstorable(pre_b)) atomicCAS(g.err, 0, kErrNonFiniteOperand);
        const __half2 hi = __floats2half2_rn(a, b);
        const float2 hf = __half22float2(hi);
        const int64_t pl = (int64_t)y * g.out_run_planes + (n >> 3);
        *reinterpret_cast<__half2*>(g.out_planes + ((size_t)pl * g.out_pitch + px) * 8 + (n & 7)) = hi;
        *reinterpret_cast<uint32_t*>(g.out_planes + ((size_t)(pl + g.out_run_planes / 2) * g.out_pitch + px) * 8 + (n & 7)) =
            pack_h2(a - hf.x, b - hf.y);
      } else {
        *reinterpret_cast<float2*>(g.out_f32 + ((size_t)y * g.M + px) * g.n_valid + n) = make_float2(a, b);
      }
    }
  }
}

// Single-scan leg: adds the n_split fp32 K-slice sums of k_leg_mma<5> in slice order, then bias, ReLU and the
// output of EPI (4: hi / lo planes, 3: fp32 volume).  One thread per (row y, pixel, 8 channels).
template <int EPI>
__global__ void __launch_bounds__(256)
k_leg_splitk_reduce(LegArgs g, int rows) {
  const int c8n = g.n_valid / 8;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)rows * g.M * c8n) return;
  const int c8 = (int)(i % c8n);
  const int64_t px = (i / c8n) % g.M, y = i / c8n / g.M;
  const int64_t slice_stride = (int64_t)rows * g.M * g.n_valid;
  const float* src = g.part + (y * g.M + px) * g.n_valid + c8 * 8;
  float v[8] = {};
  for (int sl = 0; sl < g.n_split; ++sl) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(src + sl * slice_stride));
    const float4 b = __ldg(reinterpret_cast<const float4*>(src + sl * slice_stride + 4));
    v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
  }
  bool bad = false;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    v[e] += __ldg(g.bias + c8 * 8 + e);
    bad |= leg_act_unstorable(v[e]);
    v[e] = fmaxf(v[e], 0.f);
  }
  if (EPI == 4) {
    if (bad) atomicCAS(g.err, 0, kErrNonFiniteOperand);
    __half hi[8], lo[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      hi[e] = __float2half_rn(v[e]);
      lo[e] = __float2half_rn(v[e] - __half2float(hi[e]));
    }
    const int64_t pl = y * g.out_run_planes + c8;
    *reinterpret_cast<uint4*>(g.out_planes + ((size_t)pl * g.out_pitch + px) * 8) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(g.out_planes + ((size_t)(pl + g.out_run_planes / 2) * g.out_pitch + px) * 8) =
        *reinterpret_cast<const uint4*>(lo);
  } else {
    float* dst = g.out_f32 + (y * g.M + px) * g.n_valid + c8 * 8;
    *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(dst + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
}

__global__ void __launch_bounds__(384)
k_corr_finalize(const float* __restrict__ part, float* __restrict__ corr_out, int32_t* __restrict__ yaw,
                const int* __restrict__ err) {
  __shared__ float s_corr[WF];
  const int p = blockIdx.x;
  for (int k = threadIdx.x; k < WF; k += blockDim.x) {
    float c = 0.f;
    for (int b = 0; b < C6_PARTS; ++b) c += part[((size_t)p * C6_PARTS + b) * WF + k];
    s_corr[k] = c;
    if (corr_out) corr_out[(size_t)p * WF + k] = c;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int best = 0;
    float bv = s_corr[0];
    for (int k = 1; k < WF; ++k)
      if (s_corr[k] > bv) { bv = s_corr[k]; best = k; }
    // a raised error flag (pipeline failure, bad index) poisons the result: garbage never looks valid
    yaw[p] = (*err != 0) ? INT32_MIN : 180 - best;   // infer.py:158, as k_corr_readout
  }
}

// ---- calibration of the o1 / x3 centres (runs once per handle, on the first pairs it scores) --------
// per-channel mean of o1 over rows [0, M): o1 tiles [m/128][15 di][128][64 swizzled]; one block, fixed order
__global__ void __launch_bounds__(1024)
k_o1_channel_mean(const __half* __restrict__ o1, int64_t M, float* __restrict__ mu) {
  __shared__ float part[16][64];
  const int o = threadIdx.x & 63, g = threadIdx.x >> 6;            // 16 row groups
  float acc = 0.f;
  for (int64_t m = g; m < M; m += 16)
    for (int di = 0; di < S15; ++di) acc += __half2float(o1[o1_chunk_offset(m, di, o >> 3) + (o & 7)]);
  part[g][o] = acc;
  __syncthreads();
  if (g == 0) {
    float t = 0.f;
    for (int k = 0; k < 16; ++k) t += part[k][o];
    mu[o] = __half2float(__float2half_rn(t / (float)(M * S15)));   // fp16: k_delta_conv1_wgmma starts its accumulators at -mu_o1
  }
}

// per-channel mean of x3 over rows [0, M): planes [16][pitch][8]
__global__ void __launch_bounds__(1024)
k_x3_channel_mean(const __half* __restrict__ x3, int64_t pitch, int64_t M, float* __restrict__ mu) {
  __shared__ float part[8][128];
  const int n = threadIdx.x & 127, g = threadIdx.x >> 7;
  float acc = 0.f;
  for (int64_t m = g; m < M; m += 8) acc += __half2float(x3[((size_t)(n >> 3) * pitch + m) * 8 + (n & 7)]);
  part[g][n] = acc;
  __syncthreads();
  if (g == 0) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += part[k][n];
    mu[n] = t / (float)M;
  }
}

// b2eff[n] = b2base[n] + sum_{di,o} mu_o1[o] W2[di][o][n]      (c_conv2 is linear: generateNet.py:102-106)
__global__ void __launch_bounds__(128)
k_fold_bias2(const float* __restrict__ b2base, const float* __restrict__ mu_o1, const float* __restrict__ W2,
             float* __restrict__ b2eff) {
  const int n = threadIdx.x;
  float acc = b2base[n];
  for (int di = 0; di < S15; ++di)
    for (int o = 0; o < 64; ++o) acc = fmaf(mu_o1[o], W2[((size_t)di * 64 + o) * 128 + n], acc);
  b2eff[n] = acc;
}

// b3eff[m] = b3[m] + sum_{tap,n} mu_x3[n] W3[tap][n][m] with the EXACT fp32 weights: the tensor path then
// computes  sum (x3 - mu) W3_f16 + sum mu W3_f32 = sum x3 W3_f32 - sum (x3 - mu) dW3,  i.e. the fp16
// rounding of W3 only acts on the centred fluctuation of x3.  Without this its effect was a nearly
// pair-independent logit offset (a static perturbation times a non-negative input of stable mean):
// the largest single term of the error budget on the Infer parity test (float64 emulation, tools/precision_study.py).
__global__ void __launch_bounds__(256)
k_fold_bias3(const float* __restrict__ b3, const float* __restrict__ mu_x3, const float* __restrict__ W3,
             float* __restrict__ b3eff) {
  const int m = threadIdx.x;
  float acc = b3[m];
  for (int tap = 0; tap < 9; ++tap)
    for (int n = 0; n < 128; ++n)
      acc = fmaf(mu_x3[n], W3[((size_t)tap * 128 + n) * 256 + m], acc);
  b3eff[m] = acc;
}

// Dense bias + sigmoid: fixed-order reduction of the per-row partial sums of one pair
__global__ void __launch_bounds__(256)
k_dense_finalize(const float* __restrict__ partial, const float* __restrict__ bd, int rows_per_pair,
                 float* __restrict__ overlap, const int* __restrict__ err) {
  __shared__ float red[256];
  const int p = blockIdx.x;
  const float* x = partial + (size_t)p * rows_per_pair * 2;
  float acc = 0.f;
  for (int i = threadIdx.x; i < rows_per_pair * 2; i += 256) acc += x[i];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) overlap[p] = (*err != 0) ? __int_as_float(0x7fc00000) : 1.0f / (1.0f + expf(-(red[0] + bd[0])));
}

constexpr size_t L1_DIRECT_SMEM = 48 * 1024;           // k_leg_layer1_direct: one kernel row of the weights
constexpr size_t L1_SMALL_SMEM = 200 * 1024;           // k_leg_layer1_small: all of them

// Leg layer 1 (5x15 stride (2,2), C_in = 4..25 -> 16, ReLU) straight from the fp32 NHWC input
// image to the hi/lo fp16 planes layer 2 reads.  K = kh*kw*C_in is only 300 for the geometric cues
// and N = 16: as a 64x64-tiled SIMT GEMM this took 61 us of a 245 us single-scan leg.  One thread
// per TWO adjacent output pixels x all 16 output channels: the 16 weights of a (tap, channel) are read
// once from shared memory (4 broadcast LDS.128) and feed 32 FFMAs -- the first version (one pixel x 8
// channels per thread: 8 LDS per 32 FFMA) was bound by the load/store unit.
template <bool CIN4>
__global__ void __launch_bounds__(512, CIN4 ? 0 : 2)      // generic C_in: two blocks per SM (64 registers); C_in = 4: no minimum
k_leg_layer1_direct(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                    int n, int H_in, int W_in, int cin, int kh, int kw, int sh, int sw, int H_out, int W_out,
                    int relu, __half* __restrict__ out, int* __restrict__ err) {
  constexpr int CO = 16;                                     // generateNet.py:161-164
  extern __shared__ __align__(16) float w_s[];              // [kw*cin][16]: the taps of ONE kernel row at a time
  const int pairs = (W_out + 1) / 2;                        //   (C_in = 25: 24 KB instead of 120 KB -> 4x the occupancy)
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;            // (img, y, pixel pair)
  const bool active = idx < (int64_t)n * H_out * pairs;
  if (!active) idx = 0;                                     // idle threads still take part in the barriers
  const int xo = 2 * (int)(idx % pairs);
  const int64_t r = idx / pairs;                                          // img*H_out + y
  const int y = (int)(r % H_out);
  const int64_t img = r / H_out;
  const bool has1 = xo + 1 < W_out;
  float acc0[CO], acc1[CO];
#pragma unroll
  for (int e = 0; e < CO; ++e) acc0[e] = acc1[e] = bias[e];
  const float* base0 = x + ((img * H_in + (int64_t)y * sh) * W_in + (int64_t)xo * sw) * cin;
  const float* base1 = has1 ? base0 + (int64_t)sw * cin : base0;         // a lone last pixel is computed twice
  for (int dh = 0; dh < kh; ++dh) {
    __syncthreads();
    for (int i = threadIdx.x; i < kw * cin * CO; i += blockDim.x) w_s[i] = w[(size_t)dh * kw * cin * CO + i];
    __syncthreads();
    for (int dw = 0; dw < kw; ++dw) {
      const int64_t off = ((int64_t)dh * W_in + dw) * cin;
      const float* pw = w_s + (size_t)(dw * cin) * CO;
      if (CIN4) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(base0 + off));
        const float4 b = __ldg(reinterpret_cast<const float4*>(base1 + off));
        const float va[4] = {a.x, a.y, a.z, a.w}, vb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
#pragma unroll
          for (int q4 = 0; q4 < 4; ++q4) {
            const float4 wv = *reinterpret_cast<const float4*>(pw + c * CO + q4 * 4);
            acc0[q4 * 4 + 0] = fmaf(va[c], wv.x, acc0[q4 * 4 + 0]); acc1[q4 * 4 + 0] = fmaf(vb[c], wv.x, acc1[q4 * 4 + 0]);
            acc0[q4 * 4 + 1] = fmaf(va[c], wv.y, acc0[q4 * 4 + 1]); acc1[q4 * 4 + 1] = fmaf(vb[c], wv.y, acc1[q4 * 4 + 1]);
            acc0[q4 * 4 + 2] = fmaf(va[c], wv.z, acc0[q4 * 4 + 2]); acc1[q4 * 4 + 2] = fmaf(vb[c], wv.z, acc1[q4 * 4 + 2]);
            acc0[q4 * 4 + 3] = fmaf(va[c], wv.w, acc0[q4 * 4 + 3]); acc1[q4 * 4 + 3] = fmaf(vb[c], wv.w, acc1[q4 * 4 + 3]);
          }
        }
      } else {
        for (int c = 0; c < cin; ++c) {
          const float va = __ldg(base0 + off + c), vb = __ldg(base1 + off + c);
#pragma unroll
          for (int q4 = 0; q4 < 4; ++q4) {
            const float4 wv = *reinterpret_cast<const float4*>(pw + c * CO + q4 * 4);
            acc0[q4 * 4 + 0] = fmaf(va, wv.x, acc0[q4 * 4 + 0]); acc1[q4 * 4 + 0] = fmaf(vb, wv.x, acc1[q4 * 4 + 0]);
            acc0[q4 * 4 + 1] = fmaf(va, wv.y, acc0[q4 * 4 + 1]); acc1[q4 * 4 + 1] = fmaf(vb, wv.y, acc1[q4 * 4 + 1]);
            acc0[q4 * 4 + 2] = fmaf(va, wv.z, acc0[q4 * 4 + 2]); acc1[q4 * 4 + 2] = fmaf(vb, wv.z, acc1[q4 * 4 + 2]);
            acc0[q4 * 4 + 3] = fmaf(va, wv.w, acc0[q4 * 4 + 3]); acc1[q4 * 4 + 3] = fmaf(vb, wv.w, acc1[q4 * 4 + 3]);
          }
        }
      }
    }
  }
  if (!active) return;
  // [img][y][hi,lo][c8 = 2][x][8]
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    if (p == 1 && !has1) break;
    const float* acc = p ? acc1 : acc0;
#pragma unroll
    for (int g = 0; g < 2; ++g) {
      __half hi[8], lo[8];
      bool bad = false;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float v = relu ? fmaxf(acc[g * 8 + e], 0.f) : acc[g * 8 + e];
        bad |= leg_act_unstorable(relu ? acc[g * 8 + e] : fabsf(acc[g * 8 + e]));
        hi[e] = __float2half_rn(v);
        lo[e] = __float2half_rn(v - __half2float(hi[e]));
      }
      if (bad) atomicCAS(err, 0, kErrNonFiniteOperand);
      const int64_t plane_hi = r * 4 + g;
      *reinterpret_cast<uint4*>(out + ((size_t)plane_hi * W_out + xo + p) * 8) = *reinterpret_cast<const uint4*>(hi);
      *reinterpret_cast<uint4*>(out + ((size_t)(plane_hi + 2) * W_out + xo + p) * 8) = *reinterpret_cast<const uint4*>(lo);
    }
  }
}

template <bool CIN4>
__global__ void __launch_bounds__(256)
k_leg_layer1_small(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                    int n, int H_in, int W_in, int cin, int kh, int kw, int sh, int sw, int H_out, int W_out, int cout,
                    int relu, __half* __restrict__ out, int* __restrict__ err) {
  // latency-mode variant (1-2 scans): one thread per (pixel, 8 output channels) -- four times the threads of
  // k_leg_layer1_direct, which matters when a single scan has to fill every SM
  extern __shared__ __align__(16) float w_s[];              // [kh*kw*cin][cout]
  for (int i = threadIdx.x; i < kh * kw * cin * cout; i += blockDim.x) w_s[i] = w[i];
  __syncthreads();
  const int C8 = cout / 8;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // (img, y, c8, x)
  if (idx >= (int64_t)n * H_out * C8 * W_out) return;
  const int xo = (int)(idx % W_out);
  int64_t r = idx / W_out;
  const int g = (int)(r % C8); r /= C8;                                   // r = img*H_out + y
  const int y = (int)(r % H_out);
  const int64_t img = r / H_out;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = bias[g * 8 + e];
  const float* base = x + ((img * H_in + (int64_t)y * sh) * W_in + (int64_t)xo * sw) * cin;
  for (int dh = 0; dh < kh; ++dh) {
    for (int dw = 0; dw < kw; ++dw) {
      const float* px = base + ((int64_t)dh * W_in + dw) * cin;
      const float* pw = w_s + (size_t)((dh * kw + dw) * cin) * cout + g * 8;
      if (CIN4) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(px));
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float4 w0 = *reinterpret_cast<const float4*>(pw + c * cout);
          const float4 w1 = *reinterpret_cast<const float4*>(pw + c * cout + 4);
          acc[0] = fmaf(vv[c], w0.x, acc[0]); acc[1] = fmaf(vv[c], w0.y, acc[1]);
          acc[2] = fmaf(vv[c], w0.z, acc[2]); acc[3] = fmaf(vv[c], w0.w, acc[3]);
          acc[4] = fmaf(vv[c], w1.x, acc[4]); acc[5] = fmaf(vv[c], w1.y, acc[5]);
          acc[6] = fmaf(vv[c], w1.z, acc[6]); acc[7] = fmaf(vv[c], w1.w, acc[7]);
        }
      } else {
        for (int c = 0; c < cin; ++c) {
          const float vc = __ldg(px + c);
          const float4 w0 = *reinterpret_cast<const float4*>(pw + c * cout);
          const float4 w1 = *reinterpret_cast<const float4*>(pw + c * cout + 4);
          acc[0] = fmaf(vc, w0.x, acc[0]); acc[1] = fmaf(vc, w0.y, acc[1]);
          acc[2] = fmaf(vc, w0.z, acc[2]); acc[3] = fmaf(vc, w0.w, acc[3]);
          acc[4] = fmaf(vc, w1.x, acc[4]); acc[5] = fmaf(vc, w1.y, acc[5]);
          acc[6] = fmaf(vc, w1.z, acc[6]); acc[7] = fmaf(vc, w1.w, acc[7]);
        }
      }
    }
  }
  __half hi[8], lo[8];
  bool bad = false;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float v = relu ? fmaxf(acc[e], 0.f) : acc[e];
    bad |= leg_act_unstorable(relu ? acc[e] : fabsf(acc[e]));
    hi[e] = __float2half_rn(v);
    lo[e] = __float2half_rn(v - __half2float(hi[e]));
  }
  if (bad) atomicCAS(err, 0, kErrNonFiniteOperand);
  const int64_t plane_hi = r * (2 * C8) + g;                               // [img][y][hi,lo][c8][x][8]
  *reinterpret_cast<uint4*>(out + ((size_t)plane_hi * W_out + xo) * 8) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(out + ((size_t)(plane_hi + C8) * W_out + xo) * 8) = *reinterpret_cast<const uint4*>(lo);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int tc_supported(const ovn_handle* h) {
  return h->net_ok && h->cfg.leg_output_width == WF && h->cfg.conv1size == S15;
}

// K slices of a leg layer (2..) for n scans.  A single scan gives layers 3.. only 14-42 output tiles of 64 pixels
// x 64 channels for 132 SMs, each a chain of up to 144 K iterations whose loads miss a cold L2; n <= 2 (the
// threshold of k_leg_layer1_small) splits K into slices of >= 4 iterations, up to about 4 CTAs per SM.
// Batches fill the GPU with tiles and keep one slice (no partial round trip).
static int leg_split(const ovn_handle* h, const ConvSpec& L, int n) {
  if (n > 2) return 1;
  const int64_t tiles = (int64_t)n * L.h_out * ((L.w_out + MMA_ROWS - 1) / MMA_ROWS) * ((L.cout + 63) / 64);
  const int64_t n_it = (int64_t)L.kh * L.kw * (L.cin / 16);
  int64_t sp = (4 * h->sm_count + tiles - 1) / tiles;
  if (sp > n_it / 4) sp = n_it / 4;
  return sp < 1 ? 1 : (int)sp;
}

int tc_pack_weights(ovn_handle* h) {
  if (!tc_supported(h))
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "precision f16_tc supports leg_output_width=360, conv1size=15 only");
  const ConvSpec& L1 = h->leg[0];              // leg_forward_tc runs layer 1 on k_leg_layer1_small or _direct only
  const size_t l1_row_bytes = (size_t)L1.kw * L1.cin * L1.cout * sizeof(float);
  if (L1.cout != 16 || l1_row_bytes > L1_DIRECT_SMEM || l1_row_bytes * L1.kh > L1_SMALL_SMEM)
    OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "tensor-core leg: layer %s does not fit k_leg_layer1_direct / _small", L1.name);
  // h->tc, complete or not at all: a failed re-pack leaves no half-built state for the heads to read.  The old
  // state is freed first, so that the new one can use its memory.
  h->tc.reset();
  std::unique_ptr<TcState, TcStateDelete> t(new TcState());
  const LayerWeights& w1 = h->host_w["c_conv1"];   // (1,15,128,64)
  const LayerWeights& w2 = h->host_w["c_conv2"];   // (15,1,64,128)
  const LayerWeights& w3 = h->host_w["c_conv3"];   // (3,3,128,256)
  // W1p[st = cc*15 + dj][k8][o][e] = W1[dj][c = cc*32 + k8*8 + e][o]
  std::vector<__half> p1((size_t)K4_STEPS * 4 * 64 * 8);
  for (int cc = 0; cc < 4; ++cc)
    for (int dj = 0; dj < S15; ++dj)
      for (int k8 = 0; k8 < 4; ++k8)
        for (int o = 0; o < 64; ++o)
          for (int e = 0; e < 8; ++e) {
            const int c = cc * 32 + k8 * 8 + e;
            p1[((((size_t)(cc * S15 + dj) * 4 + k8) * 64 + o) * 8) + e] =
                __float2half(w1.kernel[((size_t)dj * CF + c) * 64 + o]);
          }
  // c_conv2: two SWIZZLE_128B tiles (hi, lo) per di: W2s[di][part][n][chunk (o/8) ^ (n & 7)][o % 8], W2[di][o][n] = hi + lo
  std::vector<__half> p2((size_t)S15 * 2 * 128 * 64);
  for (int di = 0; di < S15; ++di)
    for (int n = 0; n < 128; ++n)
      for (int o = 0; o < 64; ++o) {
        const float wf = w2.kernel[((size_t)di * 64 + o) * 128 + n];
        const __half wh = __float2half(wf);
        const __half wl = __float2half(wf - __half2float(wh));
        const size_t off = (size_t)n * 64 + (((o >> 3) ^ (n & 7)) << 3) + (o & 7);
        p2[((size_t)di * 2 + 0) * 128 * 64 + off] = wh;
        p2[((size_t)di * 2 + 1) * 128 * 64 + off] = wl;
      }
  // c_conv3: slab = (tap, channel group g of 32); planes c8 = g*4..g*4+3 of X3.  The x3 image is
  // stored transposed (row = jb*24 + ib), so the slab applied at row shift a*24 + b holds the kernel
  // tap (dy = b, dx = a) of the reference's (ib, jb) image.
  std::vector<__half> p3((size_t)2 * 36 * 4 * 128 * 8);
  for (int dy = 0; dy < 3; ++dy)
    for (int dx = 0; dx < 3; ++dx)
      for (int gq = 0; gq < 4; ++gq) {
        const int sl = (dy * 3 + dx) * 4 + gq;
        for (int nh = 0; nh < 2; ++nh)
          for (int j = 0; j < 4; ++j)
            for (int n = 0; n < 128; ++n)
              for (int e = 0; e < 8; ++e) {
                const int c = (gq * 4 + j) * 8 + e;
                p3[((((size_t)nh * 36 + sl) * 4 + j) * 128 + n) * 8 + e] =
                    __float2half(w3.kernel[(((size_t)dx * 3 + dy) * 128 + c) * 256 + nh * 128 + n]);
              }
      }
  // k_delta_conv1_wgmma stores o1 without the c_conv1 bias; its image under c_conv2 is a constant per channel
  std::vector<float> b2e(128);
  {
    const LayerWeights& wb1 = h->host_w["c_conv1"];
    for (int n = 0; n < 128; ++n) {
      double acc = w2.bias[n];
      for (int di = 0; di < S15; ++di)
        for (int o = 0; o < 64; ++o) acc += (double)wb1.bias[o] * (double)w2.kernel[((size_t)di * 64 + o) * 128 + n];
      b2e[n] = (float)acc;
    }
  }
  int rc;
  if ((rc = upload_vec(h, t->b2eff, b2e)) != OVN_OK) return rc;
  if ((rc = upload_vec(h, t->b2base, b2e)) != OVN_OK) return rc;
  if ((rc = upload_vec(h, t->b3eff, w3.bias)) != OVN_OK) return rc;
  if ((rc = t->mu_o1.ensure(h, 64 * sizeof(float))) != OVN_OK) return rc;
  OVN_CUDA(h, cudaMemset(t->mu_o1, 0, 64 * sizeof(float)));
  if ((rc = t->mu_x3.ensure(h, 128 * sizeof(float))) != OVN_OK) return rc;
  OVN_CUDA(h, cudaMemset(t->mu_x3, 0, 128 * sizeof(float)));
  if ((rc = upload_vec(h, t->w1p, p1)) != OVN_OK) return rc;
  if ((rc = upload_vec(h, t->w2p, p2)) != OVN_OK) return rc;
  if ((rc = upload_vec(h, t->w3p, p3)) != OVN_OK) return rc;
  // ---- leg layers 2.. : weights as (tap, term) slabs.  Three-term split product
  // x*w ~= xh*wh + xl*wh + xh*wl  (x = xh + xl, w = wh + wl in fp16): slab = (dh, dw, term)
  size_t max_planes_bytes = 0;
  for (int l = 0; l < h->n_leg; ++l) {
    const ConvSpec& L = h->leg[l];
    const size_t out_bytes = (size_t)L.h_out * 2 * (L.cout / 8) * L.w_out * 16;   // hi + lo planes
    if (out_bytes > max_planes_bytes) max_planes_bytes = out_bytes;
    if (l == 0) continue;
    if (L.cin % 16 != 0 || L.cout % 8 != 0 || L.sw != 1)
      OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "tensor-core leg: layer %s shape not supported", L.name);
    const LayerWeights& w = h->host_w[L.name];
    const int c8in = L.cin / 8;
    const int nz = (L.cout + 63) / 64;
    int rc2;
    {
      // slab = (dh, dw, term), rows = all C_in/8 chunks, 64 output channels
      const int nsl = L.kh * L.kw * 3;
      std::vector<__half> br((size_t)nz * nsl * c8in * 64 * 8, __float2half(0.f));
      for (int z = 0; z < nz; ++z)
        for (int dh = 0; dh < L.kh; ++dh)
          for (int dw = 0; dw < L.kw; ++dw)
            for (int term = 0; term < 3; ++term) {
              const int sl = (dh * L.kw + dw) * 3 + term;
              for (int c8 = 0; c8 < c8in; ++c8)
                for (int n = 0; n < 64 && z * 64 + n < L.cout; ++n)
                  for (int k = 0; k < 8; ++k) {
                    const float wf = w.kernel[(((size_t)dh * L.kw + dw) * L.cin + c8 * 8 + k) * L.cout + z * 64 + n];
                    const __half wh = __float2half(wf);
                    const __half wl = __float2half(wf - __half2float(wh));
                    br[((((size_t)z * nsl + sl) * c8in + c8) * 64 + n) * 8 + k] = (term == 2) ? wl : wh;
                  }
            }
      if ((rc2 = upload_vec(h, t->wres[l], br)) != OVN_OK) return rc2;
    }
  }
  size_t part_bytes = 0;
  for (int l = 1; l < h->n_leg; ++l)
    for (int n = 1; n <= 2 && n <= h->cfg.max_batch_scans; ++n) {
      const ConvSpec& L = h->leg[l];
      const int sp = leg_split(h, L, n);
      const size_t b = sp > 1 ? (size_t)sp * n * L.h_out * L.w_out * L.cout * sizeof(float) : 0;
      if (b > part_bytes) part_bytes = b;
    }
  if ((rc = t->leg_part.ensure(h, part_bytes)) != OVN_OK) return rc;
  for (int b = 0; b < 2; ++b) {
    const size_t bytes = max_planes_bytes * h->cfg.max_batch_scans + 32768;   // + tile overrun slack
    if ((rc = t->actp[b].ensure(h, bytes)) != OVN_OK) return rc;
    OVN_CUDA(h, cudaMemset(t->actp[b], 0, bytes));
  }
  const int64_t maxp = h->cfg.max_batch_pairs;
  // + slack for the last 256-row tile of c_conv2 / c_conv3 (255 rows) and c_conv3's window (50 rows); whole tiles
  t->rows_pad = ((maxp * PAIR_ROWS + 1024 + 255) / 256) * 256;
  if ((rc = t->l16.ensure(h, (size_t)maxp * WF * K4_PITCH * sizeof(__half))) != OVN_OK) return rc;
  if ((rc = t->r16.ensure(h, (size_t)maxp * WF * K4_PITCH * sizeof(__half))) != OVN_OK) return rc;
  OVN_CUDA(h, cudaMemset(t->l16, 0, (size_t)maxp * WF * K4_PITCH * sizeof(__half)));
  OVN_CUDA(h, cudaMemset(t->r16, 0, (size_t)maxp * WF * K4_PITCH * sizeof(__half)));
  if ((rc = t->o1.ensure(h, (size_t)120 * t->rows_pad * 8 * sizeof(__half))) != OVN_OK) return rc;
  if ((rc = t->x3.ensure(h, (size_t)16 * t->rows_pad * 8 * sizeof(__half))) != OVN_OK) return rc;
  if ((rc = t->partial.ensure(h, (size_t)t->rows_pad * 2 * sizeof(float))) != OVN_OK) return rc;
  if ((rc = t->lc.ensure(h, (size_t)maxp * C6_VOL_L_BYTES)) != OVN_OK) return rc;
  if ((rc = t->rc.ensure(h, (size_t)maxp * C6_VOL_R_BYTES)) != OVN_OK) return rc;
  if ((rc = t->corr_part.ensure(h, (size_t)maxp * C6_PARTS * WF * sizeof(float))) != OVN_OK) return rc;
  OVN_CUDA(h, cudaFuncSetAttribute(k_delta_conv1_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(K4Smem)));
  OVN_CUDA(h, cudaFuncSetAttribute(k_conv2_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C2_SMEM));
  OVN_CUDA(h, cudaFuncSetAttribute(k_conv3_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(C3Smem)));
  OVN_CUDA(h, cudaFuncSetAttribute(k_corr_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(C6Smem)));
  if ((rc = t->mu.ensure(h, CF * sizeof(float))) != OVN_OK) return rc;
  OVN_CUDA(h, cudaMemset(t->mu, 0, CF * sizeof(float)));
  OVN_CUDA(h, cudaMemset(t->o1, 0, (size_t)120 * t->rows_pad * 8 * sizeof(__half)));
  OVN_CUDA(h, cudaMemset(t->x3, 0, (size_t)16 * t->rows_pad * 8 * sizeof(__half)));
  OVN_CUDA(h, cudaFuncSetAttribute(k_leg_layer1_small<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L1_SMALL_SMEM));
  OVN_CUDA(h, cudaFuncSetAttribute(k_leg_layer1_small<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L1_SMALL_SMEM));
  h->tc = std::move(t);
  return OVN_OK;
}

int leg_forward_tc(ovn_handle* h, const float* d_input, int n, float* d_fv, cudaStream_t s, int stop_layer) {
  // Leg layers 0 .. stop_layer (the whole leg by default); layer l leaves its planes in actp[l & 1].
  // layer 1 (C_in = 4..25, stride (2,2), N = 16: K = 16 per MMA would be mostly padding) runs on the
  // direct SIMT kernels and writes hi/lo fp16 C8-interleaved planes; layers 2.. run on k_leg_mma.
  TcState* t = h->tc.get();
  if (!t) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "tensor-core weights not packed");
  prof_mark(h, PROF_LEG, s);
  {
    const ConvSpec& L = h->leg[0];                 // tc_pack_weights checked that both kernels take its shape
    const size_t w_bytes = (size_t)L.kw * L.cin * L.cout * sizeof(float);        // one kernel row of taps
    const size_t w_all = w_bytes * L.kh;
    if (n <= 2) {
      const unsigned grid = (unsigned)(((int64_t)n * L.h_out * (L.cout / 8) * L.w_out + 255) / 256);
      if (L.cin == 4)
        k_leg_layer1_small<true><<<grid, 256, w_all, s>>>(d_input, h->d_w[0], h->d_b[0], n, L.h_in, L.w_in, L.cin, L.kh, L.kw,
                                                         L.sh, L.sw, L.h_out, L.w_out, L.cout, L.relu, t->actp[0], h->d_err);
      else
        k_leg_layer1_small<false><<<grid, 256, w_all, s>>>(d_input, h->d_w[0], h->d_b[0], n, L.h_in, L.w_in, L.cin, L.kh, L.kw,
                                                          L.sh, L.sw, L.h_out, L.w_out, L.cout, L.relu, t->actp[0], h->d_err);
    } else {
      const int64_t work = (int64_t)n * L.h_out * ((L.w_out + 1) / 2);          // one thread per pixel pair
      const unsigned grid = (unsigned)((work + 511) / 512);
      if (L.cin == 4)
        k_leg_layer1_direct<true><<<grid, 512, w_bytes, s>>>(d_input, h->d_w[0], h->d_b[0], n, L.h_in, L.w_in, L.cin, L.kh, L.kw,
                                                            L.sh, L.sw, L.h_out, L.w_out, L.relu, t->actp[0], h->d_err);
      else
        k_leg_layer1_direct<false><<<grid, 512, w_bytes, s>>>(d_input, h->d_w[0], h->d_b[0], n, L.h_in, L.w_in, L.cin, L.kh, L.kw,
                                                             L.sh, L.sw, L.h_out, L.w_out, L.relu, t->actp[0], h->d_err);
    }
    OVN_LAUNCH_CHECK(h);
  }
  int cur = 0;
  for (int l = 1; l < h->n_leg && l <= stop_layer; ++l) {
    const ConvSpec& L = h->leg[l];
    const bool last = (l == h->n_leg - 1);
    const int nz = (L.cout + 63) / 64;
    if (last && (L.cout != 128 || L.h_out != 1)) OVN_SET_ERR(h, OVN_ERR_BAD_CONFIG, "tensor-core leg: unexpected last layer");
    LegArgs la = {};
    la.A = t->actp[cur]; la.a_pitch = L.w_in; la.runs_per_img = L.h_out; la.in_img_planes = L.h_in * 2 * (L.cin / 8);
    la.in_run_planes = L.sh * 2 * (L.cin / 8); la.kh = L.kh; la.kw = L.kw; la.c8in = L.cin / 8; la.Bp = t->wres[l];
    la.bias = h->d_b[l]; la.n_valid = L.cout; la.M = L.w_out; la.out_planes = t->actp[cur ^ 1]; la.out_pitch = L.w_out;
    la.out_run_planes = 2 * (L.cout / 8); la.out_f32 = d_fv;
    la.n_split = leg_split(h, L, n); la.part = t->leg_part; la.err = h->d_err;
    const dim3 grid((unsigned)(n * L.h_out), (unsigned)((L.w_out + MMA_ROWS - 1) / MMA_ROWS), (unsigned)(nz * la.n_split));
    if (la.n_split > 1) {
      k_leg_mma<5><<<grid, MMA_THREADS, 0, s>>>(la);
      OVN_LAUNCH_CHECK(h);
      const int64_t work = (int64_t)n * L.h_out * L.w_out * (L.cout / 8);
      if (last) k_leg_splitk_reduce<3><<<(unsigned)((work + 255) / 256), 256, 0, s>>>(la, n * L.h_out);
      else k_leg_splitk_reduce<4><<<(unsigned)((work + 255) / 256), 256, 0, s>>>(la, n * L.h_out);
    } else if (last) {
      k_leg_mma<3><<<grid, MMA_THREADS, 0, s>>>(la);
    } else {
      k_leg_mma<4><<<grid, MMA_THREADS, 0, s>>>(la);
    }
    OVN_LAUNCH_CHECK(h);
    cur ^= 1;
  }
  prof_mark(h, PROF_LEG, s);
  return OVN_OK;
}

static int calibrate_all(ovn_handle* h, const float* d_vols, const int32_t* d_idx, bool keep_mu, cudaStream_t s);

int tc_bank_release(ovn_handle* h, const float* d_bank) {
  TcState* t = h->tc.get();
  if (!t || (d_bank && t->pb_key != d_bank)) return OVN_OK;
  OVN_CUDA(h, cudaDeviceSynchronize());
  t->pb_l16 = {};
  t->pb_lc = {};
  t->pb_bad = {};
  t->pb_key = nullptr;
  t->pb_rows = 0;
  return OVN_OK;
}

int tc_bank_prepare(ovn_handle* h, const float* d_bank, int64_t capacity, int64_t first, int64_t count, cudaStream_t s) {
  TcState* t = h->tc.get();
  if (!t) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "tensor-core weights not packed");
  const size_t l16_bytes = (size_t)capacity * WF * K4_PITCH * sizeof(__half);
  if (t->pb_key != d_bank || l16_bytes > t->pb_l16.bytes()) {      // a new bank, allocated to its capacity
    int rc = OVN_OK;
    if (t->pb_key != nullptr || t->pb_l16) rc = tc_bank_release(h, nullptr);
    if (rc == OVN_OK) rc = t->pb_l16.ensure(h, l16_bytes);
    if (rc == OVN_OK) rc = t->pb_lc.ensure(h, (size_t)capacity * C6_VOL_L_BYTES);
    if (rc == OVN_OK) rc = t->pb_bad.ensure(h, (size_t)capacity * sizeof(int32_t));
    if (rc != OVN_OK) return rc;
    OVN_CUDA(h, cudaMemsetAsync(t->pb_l16, 0, l16_bytes, s));
    t->pb_key = d_bank;
    t->pb_rows = 0;
    if (first != 0) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_bank_prepare: a new bank must be prepared from row 0");
  }
  if (first > t->pb_rows) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_bank_prepare: rows [%lld, %lld) were never prepared",
                                      (long long)t->pb_rows, (long long)first);
  const int64_t per = (int64_t)WF * CF / 4, perL = 16 * C6_LT * C6_LROWS;
  const float* src = d_bank + (size_t)first * WF * CF;
  if (!t->mu_set) {                     // first bank row seen by this handle: calibrate the centres on it
    int rc = calibrate_all(h, src, nullptr, false, s);
    if (rc != OVN_OK) return rc;
  }
  // the rows' non-finite marks start clear and are set by the two conversions; heads calls check them through lidx
  OVN_CUDA(h, cudaMemsetAsync(t->pb_bad + first, 0, (size_t)count * sizeof(int32_t), s));
  k_gather_rows_f16<<<(unsigned)((count * per + 255) / 256), 256, 0, s>>>(src, nullptr, (int)count, t->mu, 0,
                                                                         t->pb_l16 + (size_t)first * WF * K4_PITCH, h->d_err,
                                                                         t->pb_bad + first);
  OVN_LAUNCH_CHECK(h);
  k_pack_corr<C6_LROWS, C6_LT><<<(unsigned)((count * perL + 255) / 256), 256, 0, s>>>(src, nullptr, (int)count,
                                                                      t->pb_lc + (size_t)first * (C6_VOL_L_BYTES / 2), h->d_err,
                                                                      t->pb_bad + first);
  OVN_LAUNCH_CHECK(h);
  if (first + count > t->pb_rows) t->pb_rows = first + count;
  return OVN_OK;
}

// ---- calibration of the three centres ----------------------------------------------------------------
// Everything is derived from ONE volume V0 (the first one the handle sees: first bank row prepared, else the
// first RIGHT volume scored, or the one given to ovn_calibrate): mu = channel means of V0; the o1 / x3
// centres are the channel means over the canonical pair (LEFT = V0, RIGHT = V0 rolled by half a turn) --
// c_conv1 with centre 0 -> mean of o1 -> fold into b2eff; c_conv1 again (centred) + c_conv2 with centre 0
// -> mean of x3 -> fold into b3eff.  All on the stream, fixed summation orders: two handles calibrated on
// the same volume (e.g. every rank of a sharded bank) give bit-identical results.
static int calibrate_all(ovn_handle* h, const float* d_vols, const int32_t* d_idx, bool keep_mu, cudaStream_t s) {
  TcState* t = h->tc.get();
  const int base = kMaxLegLayers;
  const int64_t per = (int64_t)WF * CF / 4;
  if (!keep_mu) {
    k_channel_mean<<<1, 1024, 0, s>>>(d_vols, d_idx, 1, t->mu);
    OVN_LAUNCH_CHECK(h);
  }
  OVN_CUDA(h, cudaMemsetAsync(t->mu_o1, 0, 64 * sizeof(float), s));
  OVN_CUDA(h, cudaMemsetAsync(t->mu_x3, 0, 128 * sizeof(float), s));
  k_gather_rows_f16<<<(unsigned)((per + 255) / 256), 256, 0, s>>>(d_vols, d_idx, 1, t->mu, 0, t->l16, h->d_err, nullptr);
  OVN_LAUNCH_CHECK(h);
  k_gather_rows_f16<<<(unsigned)((per + 255) / 256), 256, 0, s>>>(d_vols, d_idx, 1, t->mu, WF / 2, t->r16, h->d_err, nullptr);
  OVN_LAUNCH_CHECK(h);
  t->last_n = 0;                        // o1 and x3 now hold the calibration pair
  const int64_t Mc = PAIR_ROWS;
  const int g4c = NB < h->sm_count ? NB : h->sm_count;
  const int64_t tiles_c = (Mc + TC_ROWS - 1) / TC_ROWS;
  k_delta_conv1_wgmma<<<g4c, K4_THREADS, sizeof(K4Smem), s>>>(t->l16, nullptr, t->r16, 0, t->w1p, t->mu_o1, t->o1, 1, h->d_err);
  OVN_LAUNCH_CHECK(h);
  k_o1_channel_mean<<<1, 1024, 0, s>>>(t->o1, Mc, t->mu_o1);
  OVN_LAUNCH_CHECK(h);
  k_fold_bias2<<<1, 128, 0, s>>>(t->b2base, t->mu_o1, h->d_w[base + 1], t->b2eff);
  OVN_LAUNCH_CHECK(h);
  k_delta_conv1_wgmma<<<g4c, K4_THREADS, sizeof(K4Smem), s>>>(t->l16, nullptr, t->r16, 0, t->w1p, t->mu_o1, t->o1, 1, h->d_err);
  OVN_LAUNCH_CHECK(h);
  k_conv2_wgmma<<<(unsigned)tiles_c, TC_THREADS, C2_SMEM, s>>>(t->o1, t->w2p, t->b2eff, t->mu_x3, t->x3, t->rows_pad, Mc, 0,
                                                              h->d_err);
  OVN_LAUNCH_CHECK(h);
  k_x3_channel_mean<<<1, 1024, 0, s>>>(t->x3, t->rows_pad, Mc, t->mu_x3);
  OVN_LAUNCH_CHECK(h);
  k_fold_bias3<<<1, 256, 0, s>>>(h->d_b[base + 2], t->mu_x3, h->d_w[base + 2], t->b3eff);
  OVN_LAUNCH_CHECK(h);
  t->mu_set = true;
  t->act_set = true;
  return OVN_OK;
}

int tc_calibrate(ovn_handle* h, const float* d_volume, cudaStream_t s) {
  TcState* t = h->tc.get();
  if (!t) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "tensor-core weights not packed");
  if (t->pb_key != nullptr)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_calibrate: release the resident bank first (its operand copies were built "
                "with the previous centre)");
  return calibrate_all(h, d_volume, nullptr, false, s);
}

int tc_set_center(ovn_handle* h, const float* h_mu) {
  TcState* t = h->tc.get();
  if (!t) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "tensor-core weights not packed");
  if (t->pb_key != nullptr)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_set_feature_center: release the resident bank first (its operand copies "
                "were built with the previous centre)");
  OVN_CUDA(h, cudaDeviceSynchronize());
  t->act_set = false;                // the o1 / x3 centres are re-calibrated with the new operands
  OVN_CUDA(h, cudaMemset(t->mu_o1, 0, 64 * sizeof(float)));
  OVN_CUDA(h, cudaMemset(t->mu_x3, 0, 128 * sizeof(float)));
  if (!h_mu) {                       // back to "calibrate at first use"
    t->mu_set = false;
    OVN_CUDA(h, cudaMemset(t->mu, 0, CF * sizeof(float)));
    return OVN_OK;
  }
  float m[CF];
  for (int c = 0; c < CF; ++c) m[c] = __half2float(__float2half(h_mu[c]));
  OVN_CUDA(h, cudaMemcpy(t->mu, m, sizeof(m), cudaMemcpyHostToDevice));
  t->mu_set = true;
  return OVN_OK;
}

int tc_get_center(ovn_handle* h, float* h_mu, int32_t* is_set) {
  TcState* t = h->tc.get();
  if (!t) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "tensor-core weights not packed");
  OVN_CUDA(h, cudaDeviceSynchronize());
  OVN_CUDA(h, cudaMemcpy(h_mu, t->mu, CF * sizeof(float), cudaMemcpyDeviceToHost));
  *is_set = t->mu_set ? 1 : 0;
  return OVN_OK;
}

int heads_forward_tc(ovn_handle* h, const float* d_bank, const float* d_query, const int32_t* d_left,
                     const int32_t* d_right, int n, float* d_overlap, int32_t* d_yaw, float* d_corr,
                     cudaStream_t s) {
  TcState* t = h->tc.get();
  if (!t) OVN_SET_ERR(h, OVN_ERR_WEIGHTS, "tensor-core weights not packed");
  const int maxp = h->cfg.max_batch_pairs;
  const int base = kMaxLegLayers;
  const int64_t per = (int64_t)WF * CF / 4;
  t->last_n = 0;                                  // o1 / x3 / partial are overwritten from here on
  if ((!t->mu_set || !t->act_set) && n > 0) {     // first pairs seen by this handle: calibrate on the first RIGHT volume
    int rc = d_query ? calibrate_all(h, d_query, nullptr, t->mu_set, s) : calibrate_all(h, d_bank, d_right, t->mu_set, s);
    if (rc != OVN_OK) return rc;
  }
  // resident bank: the LEFT operand copies already exist, the kernels index them through `lidx`
  // (indices arrive bounds-checked against bank_size; rows past the prepared range raise kErrRowNotPrepared)
  const bool resident = (t->pb_key == d_bank) && t->pb_rows > 0;
  const __half* l16 = resident ? t->pb_l16 : t->l16;
  const __half* lc = resident ? t->pb_lc : t->lc;
  int32_t* lidx = nullptr;
  if (resident) {
    lidx = h->d_idx_san + 2 * (size_t)maxp;
    int rc = sanitize_indices(h, d_left, n, t->pb_rows, kErrRowNotPrepared, lidx, s, t->pb_bad);
    if (rc != OVN_OK) return rc;
  } else {
    k_gather_rows_f16<<<(unsigned)((n * per + 255) / 256), 256, 0, s>>>(d_bank, d_left, n, t->mu, 0, t->l16, h->d_err, nullptr);
    OVN_LAUNCH_CHECK(h);
  }
  if (d_query)
    k_gather_rows_f16<<<(unsigned)((per + 255) / 256), 256, 0, s>>>(d_query, nullptr, 1, t->mu, 0, t->r16, h->d_err, nullptr);
  else
    k_gather_rows_f16<<<(unsigned)((n * per + 255) / 256), 256, 0, s>>>(d_bank, d_right, n, t->mu, 0, t->r16, h->d_err, nullptr);
  OVN_LAUNCH_CHECK(h);
  const int64_t M = (int64_t)n * PAIR_ROWS;
  const int64_t tiles = (M + TC_ROWS - 1) / TC_ROWS;                 // 256-row tiles of c_conv2 / c_conv3
  const int grid2 = tiles < h->sm_count ? (int)tiles : h->sm_count;
  const int grid3 = 2 * tiles < h->sm_count ? (int)(2 * tiles) : h->sm_count;
  prof_mark(h, PROF_DELTA, s);
  const int64_t units = (int64_t)k4_blocks(n, d_query ? 0 : 1) * NB;
  const int grid4 = units < h->sm_count ? (int)units : h->sm_count;
  k_delta_conv1_wgmma<<<grid4, K4_THREADS, sizeof(K4Smem), s>>>(l16, lidx, t->r16, d_query ? 0 : 1, t->w1p, t->mu_o1, t->o1,
                                                               n, h->d_err);
  prof_mark(h, PROF_DELTA, s);
  OVN_LAUNCH_CHECK(h);
  const bool inject_fault = getenv("OVN_DEBUG_FAULT") != nullptr;            // error-path test hook
  prof_mark(h, PROF_CONV2, s);
  k_conv2_wgmma<<<grid2, TC_THREADS, C2_SMEM, s>>>(t->o1, t->w2p, t->b2eff, t->mu_x3, t->x3, t->rows_pad, M,
                                                   inject_fault ? 1 : 0, h->d_err);
  prof_mark(h, PROF_CONV2, s);
  OVN_LAUNCH_CHECK(h);
  prof_mark(h, PROF_CONV3, s);
  k_conv3_wgmma<<<grid3, TC_THREADS, sizeof(C3Smem), s>>>(t->x3, t->rows_pad, t->w3p, t->b3eff, M, h->d_w[base + 3],
                                                          t->partial, h->d_err);
  prof_mark(h, PROF_CONV3, s);
  OVN_LAUNCH_CHECK(h);
  k_dense_finalize<<<n, 256, 0, s>>>(t->partial, h->d_b[base + 3], PAIR_ROWS, d_overlap, h->d_err);
  OVN_LAUNCH_CHECK(h);
  // correlation head (tensor cores, hi/lo split operands)
  const int64_t perL = 16 * C6_LT * C6_LROWS, perR = 16 * C6_RT * C6_RROWS;
  if (!resident) {
    k_pack_corr<C6_LROWS, C6_LT><<<(unsigned)((n * perL + 255) / 256), 256, 0, s>>>(d_bank, d_left, n, t->lc, h->d_err, nullptr);
    OVN_LAUNCH_CHECK(h);
  }
  if (d_query)
    k_pack_corr<C6_RROWS, C6_RT><<<(unsigned)((perR + 255) / 256), 256, 0, s>>>(d_query, nullptr, 1, t->rc, h->d_err, nullptr);
  else
    k_pack_corr<C6_RROWS, C6_RT><<<(unsigned)((n * perR + 255) / 256), 256, 0, s>>>(d_bank, d_right, n, t->rc, h->d_err, nullptr);
  OVN_LAUNCH_CHECK(h);
  prof_mark(h, PROF_CORR, s);
  const int nc = (int64_t)n * C6_LT < h->sm_count / C6_RT ? n * C6_LT : h->sm_count / C6_RT;
  k_corr_wgmma<<<nc * C6_RT, C6_THREADS, sizeof(C6Smem), s>>>(lc, lidx, t->rc, d_query ? 0 : 1, n, t->corr_part, h->d_err);
  prof_mark(h, PROF_CORR, s);
  OVN_LAUNCH_CHECK(h);
  k_corr_finalize<<<n, 384, 0, s>>>(t->corr_part, d_corr, d_yaw, h->d_err);
  OVN_LAUNCH_CHECK(h);
  t->last_n = n;
  static const bool debug_sync = getenv("OVN_DEBUG_SYNC") != nullptr;
  if (debug_sync) return check_device_error(h, s);
  return OVN_OK;
}

// ovn_copy_heads_stage: the stored o1 / x3 / partial of pairs [first, first + n) as float32, in the reference's
// orientation; a copy and a conversion only.  One thread per output element.
//   O1 [n][360][24][64] (i, jb, o) from the o1 tiles, X3 [n][24][24][128] (ib, jb, c) from the C8 planes,
//   DENSE [n][24][24][2] (ib, jb, half) from partial; row m = pair * 576 + jb * 24 + ib in all three.
__global__ void __launch_bounds__(256)
k_copy_heads_stage(int stage, const __half* __restrict__ o1, const __half* __restrict__ x3, int64_t x3_pitch,
                   const float* __restrict__ partial, int64_t first, int64_t total, float* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  out += e;
  if (stage == OVN_STAGE_O1) {
    const int o = (int)(e % 64), jb = (int)(e / 64 % NB), i = (int)(e / (64 * NB) % WF);
    const int64_t p = first + e / (64 * NB * WF);
    const int64_t m = p * PAIR_ROWS + jb * NB + i / S15;
    *out = __half2float(o1[o1_chunk_offset(m, i % S15, o >> 3) + (o & 7)]);
  } else if (stage == OVN_STAGE_X3) {
    const int c = (int)(e % 128), jb = (int)(e / 128 % NB), ib = (int)(e / (128 * NB) % NB);
    const int64_t m = (first + e / (128 * PAIR_ROWS)) * PAIR_ROWS + jb * NB + ib;
    *out = __half2float(x3[((size_t)(c >> 3) * x3_pitch + m) * 8 + (c & 7)]);
  } else {
    const int half = (int)(e % 2), jb = (int)(e / 2 % NB), ib = (int)(e / (2 * NB) % NB);
    const int64_t m = (first + e / (2 * PAIR_ROWS)) * PAIR_ROWS + jb * NB + ib;
    *out = partial[m * 2 + half];
  }
}

int64_t tc_heads_stage_pairs(const ovn_handle* h) {
  const TcState* t = h->tc.get();
  return t ? t->last_n : 0;
}

int tc_copy_heads_stage(ovn_handle* h, int stage, int64_t first, int64_t count, float* d_out, cudaStream_t s) {
  TcState* t = h->tc.get();
  if (!t || t->last_n == 0)
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_copy_heads_stage: no stored stages (no complete heads call since the "
                "weights were packed or the centres calibrated)");
  if (!d_out) OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_copy_heads_stage: NULL pointer");
  if (stage != OVN_STAGE_CENTRES && (first < 0 || count < 1 || first + count > t->last_n))
    OVN_SET_ERR(h, OVN_ERR_INVALID_ARG, "ovn_copy_heads_stage: pairs [%lld, %lld) outside the %lld stored",
                (long long)first, (long long)(first + count), (long long)t->last_n);
  if (stage == OVN_STAGE_CENTRES) {
    const Buffer<float>* parts[4] = {&t->mu_o1, &t->mu_x3, &t->b2eff, &t->b3eff};
    const size_t len[4] = {64, 128, 128, 256};
    for (int k = 0; k < 4; ++k) {
      OVN_CUDA(h, cudaMemcpyAsync(d_out, *parts[k], len[k] * sizeof(float), cudaMemcpyDeviceToDevice, s));
      d_out += len[k];
    }
    return OVN_OK;
  }
  const int64_t per = stage == OVN_STAGE_O1 ? (int64_t)WF * NB * 64 : stage == OVN_STAGE_X3 ? PAIR_ROWS * 128 : PAIR_ROWS * 2;
  const int64_t total = count * per;
  k_copy_heads_stage<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(stage, t->o1, t->x3, t->rows_pad, t->partial, first,
                                                                       total, d_out);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

// ovn_leg_stage: the hi / lo planes of one leg layer ([img][y][hi, lo][c8][x][8] fp16, leg_forward_tc) as two NHWC
// float32 arrays [n][h_out][w_out][cout]; a copy and a conversion only.  One thread per output element.
__global__ void __launch_bounds__(256)
k_copy_leg_stage(const __half* __restrict__ planes, int w_out, int cout, int64_t total, float* __restrict__ hi,
                 float* __restrict__ lo) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int c = (int)(e % cout), x = (int)(e / cout % w_out);
  const int64_t row = e / cout / w_out;                                  // img * h_out + y
  const int c8n = cout / 8;
  const __half* p = planes + ((size_t)(row * 2 * c8n + (c >> 3)) * w_out + x) * 8 + (c & 7);
  hi[e] = __half2float(p[0]);
  lo[e] = __half2float(p[(size_t)c8n * w_out * 8]);
}

int tc_leg_stage(ovn_handle* h, const float* d_input, int n, int layer, float* d_hi, float* d_lo, cudaStream_t s) {
  const int rc = leg_forward_tc(h, d_input, n, nullptr, s, layer);
  if (rc != OVN_OK) return rc;
  const ConvSpec& L = h->leg[layer];
  const int64_t total = (int64_t)n * L.h_out * L.w_out * L.cout;
  k_copy_leg_stage<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(h->tc->actp[layer & 1], L.w_out, L.cout, total, d_hi, d_lo);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

}  // namespace ovn
