// network_fp32.cu -- fp32 SIMT verification path for the leg and the two heads.
//
// One tiled implicit-GEMM kernel (64x64x16 tiles, 4x4 register blocking) serves every layer; the
// A operand is produced on the fly by an "operand functor" (im2col of a valid-padded NHWC conv,
// or the |L - R| delta operand), so neither the im2col matrix nor the 66 MB delta tensor of the
// reference (generateNet.py:45-59) is ever materialised.  This path exists to (a) give a
// bit-for-bit reproducible fp32 result that the tensor-core path is validated against on the
// device and (b) serve precision=OVN_PREC_FP32.  The performance path is network_tc.cu.
//
// Replaces: generate360OutputkLegs (generateNet.py:161-217), DeltaLayer (:15-61),
// generateDeltaLayerConv1NetworkHead (:64-116), RangePadding2D.call (RangePadding2D.py:31-38),
// NormalizedCorrelation2D.call (NormalizedCorrelation2D.py:43-109), readout (infer.py:157-158).
#include "common.cuh"

namespace ovn {

constexpr int BM = 64, BN = 64, BK = 16;

// ---- operand functors ------------------------------------------------------------------------
// NHWC valid conv:  A[m, k] = X[img, ho*sh + dh, wo*sw + dw, c],  m = (img, ho, wo), k = (dh, dw, c)
struct ConvOperand {
  const float* X;
  int H, W, C, kw, sh, sw, Ho, Wo;
  __device__ __forceinline__ int64_t row_base(int m, int /*z*/) const {
    const int wo = m % Wo;
    const int t = m / Wo;
    const int ho = t % Ho;
    const int img = t / Ho;
    return (((int64_t)img * H + (int64_t)ho * sh) * W + (int64_t)wo * sw) * C;
  }
  __device__ __forceinline__ int col_off(int k) const {
    const int rowlen = kw * C;
    const int dh = k / rowlen;
    return dh * W * C + (k - dh * rowlen);
  }
  __device__ __forceinline__ float load(int64_t rb, int co, int64_t, int) const { return __ldg(X + rb + co); }
  __device__ __forceinline__ int64_t row_base2(int, int) const { return 0; }
  __device__ __forceinline__ int col_off2(int) const { return 0; }
};

// c_conv1 on the delta image (generateNet.py:45-59,96-100):
//   A[m, k] = | L[i, c] - R[s*jb + dj, c] |,  m = (pair, i, jb),  k = (dj, c)
struct DeltaOperand {
  const float* bank;          // [n][Wf][128]
  const float* query;         // non-null: RIGHT is this single volume for every pair
  const int32_t* left;        // [n_pairs] bank rows
  const int32_t* right;       // [n_pairs] bank rows (ignored when query != null)
  int Wf, Cf, s, nb;          // 360, 128, 15, 24
  __device__ __forceinline__ int64_t row_base(int m, int) const {          // into LEFT
    const int jb = m % nb;
    const int t = m / nb;
    const int i = t % Wf;
    const int p = t / Wf;
    (void)jb;
    return ((int64_t)left[p] * Wf + i) * Cf;
  }
  __device__ __forceinline__ int64_t row_base2(int m, int) const {         // into RIGHT
    const int jb = m % nb;
    const int p = m / (nb * Wf);
    const int64_t vol = query ? 0 : (int64_t)right[p] * Wf * Cf;
    return vol + (int64_t)(s * jb) * Cf;
  }
  __device__ __forceinline__ int col_off(int k) const { return k % Cf; }
  __device__ __forceinline__ int col_off2(int k) const { return k; }
  __device__ __forceinline__ float load(int64_t rb, int co, int64_t rb2, int co2) const {
    const float* R = query ? query : bank;
    return fabsf(__ldg(bank + rb + co) - __ldg(R + rb2 + co2));
  }
};

// correlation Gram matrix: A = LEFT volume rows (z = pair); B comes from the RIGHT volume
struct GramOperand {
  const float* bank;
  const int32_t* left;
  int Wf, Cf;
  __device__ __forceinline__ int64_t row_base(int m, int z) const { return ((int64_t)left[z] * Wf + m) * Cf; }
  __device__ __forceinline__ int col_off(int k) const { return k; }
  __device__ __forceinline__ float load(int64_t rb, int co, int64_t, int) const { return __ldg(bank + rb + co); }
  __device__ __forceinline__ int64_t row_base2(int, int) const { return 0; }
  __device__ __forceinline__ int col_off2(int) const { return 0; }
};

// ---- operands of the overlap-head backward (training) ----
// Weight gradient of a valid NHWC conv, as the transposed im2col:  A[k, m] = X[img, ho*sh + dh, wo*sw + dw, c],
// k = (dh, dw, c) < Kc, m = (img, ho, wo).  Row k = Kc is all ones, so that the same product also yields
// the bias gradient (the column sums of dY) as row Kc of the [Kc + 1][N] result.
struct ConvWgradOperand {
  const float* X;
  int H, W, C, kw, sh, sw, Ho, Wo, Kc;
  __device__ __forceinline__ int64_t row_base(int k, int) const {           // offset of tap (dh, dw, c)
    if (k >= Kc) return 0;
    const int rowlen = kw * C;
    const int dh = k / rowlen;
    return (int64_t)dh * W * C + (k - dh * rowlen);
  }
  __device__ __forceinline__ int64_t row_base2(int k, int) const { return k >= Kc; }   // 1: the ones row
  __device__ __forceinline__ int col_off(int m) const { return m; }
  __device__ __forceinline__ int col_off2(int) const { return 0; }
  __device__ __forceinline__ float load(int64_t rb, int m, int64_t ones, int) const {
    if (ones) return 1.f;
    const int wo = m % Wo;
    const int t = m / Wo;
    const int ho = t % Ho;
    const int img = t / Ho;
    return __ldg(X + (((int64_t)img * H + (int64_t)ho * sh) * W + (int64_t)wo * sw) * C + rb);
  }
};

// Weight gradient of c_conv1, with the |l - r| operand synthesised like DeltaOperand (never materialised):
//   A[k, m] = | L[s*ho + dh, c] - R[s*jb + dj, c] |,  k = (dj, c) < Kc,  m = (((p*nho + ho)*nb + jb)*s + dh)
// m runs over the rows of the c_conv1 output in the order in which the c_conv2 input gradient is stored
// ([p][ho][jb][dh][o], see head_gradients_fp32).  Row Kc is all ones (bias gradient).
struct DeltaWgradOperand {
  const float* bank;
  const int32_t* left;
  const int32_t* right;
  int Wf, Cf, s, nb, nho, Kc;
  __device__ __forceinline__ int64_t row_base(int k, int) const { return k < Kc ? k % Cf : 0; }       // c
  __device__ __forceinline__ int64_t row_base2(int k, int) const { return k < Kc ? k / Cf : -1; }     // dj, -1: ones
  __device__ __forceinline__ int col_off(int m) const { return m; }
  __device__ __forceinline__ int col_off2(int) const { return 0; }
  __device__ __forceinline__ float load(int64_t c, int m, int64_t dj, int) const {
    if (dj < 0) return 1.f;
    const int dh = m % s;
    int t = m / s;
    const int jb = t % nb;
    t /= nb;
    const int ho = t % nho;
    const int p = t / nho;
    const float l = __ldg(bank + ((int64_t)left[p] * Wf + ho * s + dh) * Cf + c);
    const float r = __ldg(bank + ((int64_t)right[p] * Wf + s * jb + dj) * Cf + c);
    return fabsf(l - r);
  }
};

// Input gradient of a stride-1 valid conv (the transposed conv):  A[m, k] = dY[img, h - dh, w - dw, n],
// zero outside dY;  m = (img, h, w) over the [H][W] input, k = (dh, dw, n).  B = the kernel with its
// in / out axes swapped, [(dh, dw, n)][c].
struct ConvDgradOperand {
  const float* dY;            // [img][Ho][Wo][Cout]
  int Ho, Wo, Cout, kw, H, W;
  __device__ __forceinline__ int64_t row_base(int m, int) const {
    const int w = m % W;
    const int t = m / W;
    const int hh = t % H;
    const int img = t / H;
    return (((int64_t)img * Ho + hh) * Wo + w) * Cout;
  }
  __device__ __forceinline__ int64_t row_base2(int m, int) const {
    const int t = m / W;
    return ((int64_t)(t % H) << 16) | (m % W);
  }
  __device__ __forceinline__ int col_off(int k) const {
    const int rowlen = kw * Cout;
    const int dh = k / rowlen;
    const int r = k - dh * rowlen;
    const int dw = r / Cout;
    return -(dh * Wo + dw) * Cout + (r - dw * Cout);
  }
  __device__ __forceinline__ int col_off2(int k) const {
    const int rowlen = kw * Cout;
    const int dh = k / rowlen;
    return (dh << 16) | ((k - dh * rowlen) / Cout);
  }
  __device__ __forceinline__ float load(int64_t rb, int co, int64_t hw, int tap) const {
    const int y = (int)(hw >> 16) - (tap >> 16);
    const int x = (int)(hw & 0xffff) - (tap & 0xffff);
    if (y < 0 || y >= Ho || x < 0 || x >= Wo) return 0.f;
    return __ldg(dY + rb + co);
  }
};

// Input gradient of a strided valid conv:  A[m, k] = dY[img, (h - dh) / sh, (w - dw) / sw, n] where both
// divisions are exact and land inside dY, else 0.  m = (img, h, w), k = (dh, dw, n), B as in ConvDgradOperand.
// An input row that no output reads (row H - 1 of an even-height input under a stride-2, 3-row kernel) gets 0.
struct ConvDgradStridedOperand {
  const float* dY;
  int Ho, Wo, Cout, kw, H, W, sh, sw;
  __device__ __forceinline__ int64_t row_base(int m, int) const { return (int64_t)(m / (H * W)) * Ho * Wo * Cout; }
  __device__ __forceinline__ int64_t row_base2(int m, int) const {
    const int t = m / W;
    return ((int64_t)(t % H) << 16) | (m % W);
  }
  __device__ __forceinline__ int col_off(int k) const { return k % Cout; }
  __device__ __forceinline__ int col_off2(int k) const {
    const int rowlen = kw * Cout;
    const int dh = k / rowlen;
    return (dh << 16) | ((k - dh * rowlen) / Cout);
  }
  __device__ __forceinline__ float load(int64_t rb, int n, int64_t hw, int tap) const {
    int y = (int)(hw >> 16) - (tap >> 16);
    int x = (int)(hw & 0xffff) - (tap & 0xffff);
    if (y < 0 || x < 0 || y % sh || x % sw) return 0.f;
    y /= sh;
    x /= sw;
    if (y >= Ho || x >= Wo) return 0.f;
    return __ldg(dY + rb + ((int64_t)y * Wo + x) * Cout + n);
  }
};

struct BOperand {
  const float* B;             // weights [K][N] (b_nk = 0) or per-batch [N][K] (b_nk = 1)
  const float* query;         // b_nk: RIGHT volume = query for every z when non-null
  const int32_t* right;       // b_nk: bank row of the RIGHT volume of pair z
  int64_t vol_stride;
  int b_nk;
};

// ---- the staging k_simt_gemm and k_tc_gemm share ----
// A CTA of either kernel: the 64 x 64 output tile at (m0, n0) of batch / split index z, its K slice [kbeg, kend)
// and its B operand Bz.  gemm_tile also writes the row bases of the tile's BM rows to s_rb / s_rb2 (-1: past M);
// the caller synchronises before gemm_fetch reads them.
struct GemmTile {
  int m0, n0, z, kbeg, kend;
  const float* Bz;
};

template <class AOp>
__device__ __forceinline__ GemmTile gemm_tile(const AOp& a, const BOperand& bop, int M, int K, int kchunk,
                                              int64_t* s_rb, int64_t* s_rb2) {
  GemmTile t;
  t.m0 = blockIdx.y * BM;
  t.n0 = blockIdx.x * BN;
  t.z = blockIdx.z;
  const int zb = kchunk ? 0 : t.z;
  t.kbeg = kchunk ? t.z * kchunk : 0;
  t.kend = kchunk ? min(K, t.kbeg + kchunk) : K;
  if (threadIdx.x < BM) {
    const int m = t.m0 + threadIdx.x;
    s_rb[threadIdx.x] = m < M ? a.row_base(m, zb) : -1;
    s_rb2[threadIdx.x] = m < M ? a.row_base2(m, zb) : 0;
  }
  t.Bz = bop.B;
  if (bop.b_nk) t.Bz = bop.query ? bop.query : bop.B + (int64_t)bop.right[zb] * bop.vol_stride;
  return t;
}

// The place (kk, mm) in the A tile of element e = tid + 256 i of a K16 tile: consecutive threads take consecutive
// k, contiguous in memory.  Its place (kk, nn) in the B tile: for b_nk = 0 consecutive threads take consecutive n.
__device__ __forceinline__ int2 a_place(int e) { return make_int2(e % BK, e / BK); }
__device__ __forceinline__ int2 b_place(int b_nk, int e) {
  return b_nk ? make_int2(e % BK, e / BK) : make_int2(e / BN, e % BN);
}

// A thread's four A and four B elements of the K16 tile at k0, zero outside [k0, kend), past M and past N:
// put_a(kk, mm, v) and put_b(kk, nn, v) take them at their places.
template <class AOp, class PutA, class PutB>
__device__ __forceinline__ void gemm_fetch(const AOp& a, const BOperand& bop, const GemmTile& t, int k0, int N, int K,
                                           const int64_t* s_rb, const int64_t* s_rb2, PutA put_a, PutB put_b) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int2 q = a_place(tid + i * 256);
    const int k = k0 + q.x, mm = q.y;
    float v = 0.f;
    if (k < t.kend && s_rb[mm] >= 0) v = a.load(s_rb[mm], a.col_off(k), s_rb2[mm], a.col_off2(k));
    put_a(i, q.x, mm, v);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float v = 0.f;
    if (!bop.b_nk) {
      const int2 q = b_place(0, tid + i * 256);
      if (k0 + q.x < t.kend && t.n0 + q.y < N) v = __ldg(t.Bz + (int64_t)(k0 + q.x) * N + t.n0 + q.y);
      put_b(i, q.x, q.y, v);
    } else {
      const int2 q = b_place(1, tid + i * 256);
      if (k0 + q.x < t.kend && t.n0 + q.y < N) v = __ldg(t.Bz + (int64_t)(t.n0 + q.y) * K + k0 + q.x);
      put_b(i, q.x, q.y, v);
    }
  }
}

// The epilogue of output element (m, n) of the tile: C[z][m][n] = act(acc + bias[n]) inside M x N
__device__ __forceinline__ void gemm_store(const GemmTile& t, float acc, int m, int n, const float* bias, int relu,
                                           float* C, int M, int N) {
  if (m >= M || n >= N) return;
  float v = acc + (bias ? __ldg(bias + n) : 0.f);
  if (relu) v = fmaxf(v, 0.f);
  C[((int64_t)t.z * M + m) * N + n] = v;
}

// C[m, n] = act(sum_k A[m,k] * B[k,n] + bias[n]);  C row-major [z][M][N].
// kchunk == 0: z = blockIdx.z is the batch index of the operands.  kchunk > 0 (split-K): every z works on
// the same product and sums only k in [z*kchunk, (z+1)*kchunk); C[z] is that slice's partial, which
// k_splitk_reduce adds up in a fixed order (no atomics, so results are bit-reproducible).
template <class AOp>
__global__ void __launch_bounds__(256)
k_simt_gemm(AOp a, BOperand bop, const float* __restrict__ bias, float* __restrict__ C, int M, int N, int K,
            int relu, int kchunk) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  __shared__ int64_t s_rb[BM];
  __shared__ int64_t s_rb2[BM];
  const int tid = threadIdx.x;
  const GemmTile t = gemm_tile(a, bop, M, K, kchunk, s_rb, s_rb2);
  __syncthreads();
  const int ty = tid / 16, tx = tid % 16;
  float acc[4][4] = {};
  for (int k0 = t.kbeg; k0 < t.kend; k0 += BK) {
    gemm_fetch(a, bop, t, k0, N, K, s_rb, s_rb2, [&](int, int kk, int mm, float v) { As[kk][mm] = v; },
               [&](int, int kk, int nn, float v) { Bs[kk][nn] = v; });
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bv[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) gemm_store(t, acc[i][j], t.m0 + ty * 4 + i, t.n0 + tx * 4 + j, bias, relu, C, M, N);
}

// ---- 3xTF32 tensor-core bodies of the training products (ovn_set_train_precision) -------------------------
// x = hi + lo with hi = tf32_rna(x) and lo = tf32_rna(x - hi) (x - hi is exact in fp32), so |x - hi - lo| <=
// 2^-22 |x|.  A product a b is lo_a hi_b + hi_a lo_b + hi_a hi_b, three mma.sync m16n8k8 into fp32 accumulators
// in that order (the small terms first); lo_a lo_b <= 2^-22 |a b| is dropped.
// The tensor core truncates (rounds toward zero) when it adds to its accumulator, so a chain of MMAs into one
// accumulator drifts toward zero by up to an ulp per MMA: 3 K / 8 of them, 4e-5 of the overlap loss at K = 1920
// on an H100.  So the six MMAs of a K16 tile start from zero and the tile's partial is added to the running sum
// with a rounded FADD (add_tile): the truncation error then stays a few ulp of the sum of |terms| at any K.
// Fragment ownership (PTX ISA, "Matrix fragments for mma.m16n8k8", .tf32): g = lane / 4, t = lane % 4;
//   A (16 x 8, row): a0 = (g, t), a1 = (g + 8, t), a2 = (g, t + 4), a3 = (g + 8, t + 4)
//   B (8 x 8, col):  b0 = (k = t, n = g), b1 = (k = t + 4, n = g)
//   C (16 x 8):      c0 = (g, 2t), c1 = (g, 2t + 1), c2 = (g + 8, 2t), c3 = (g + 8, 2t + 1)
// The shared tiles are k-major [k][kTcPitch] hi and lo planes.  A fragment load reads word t * kTcPitch + g
// (+ a constant) in each lane; kTcPitch = 8 (mod 32) puts the 32 lanes on 32 different banks.
constexpr int kTcPitch = BM + 8;

__device__ __forceinline__ uint32_t tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r & 0xffffe000u;                 // the low 13 bits are not part of the tf32 value
}

__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = __uint_as_float(tf32_rna(x));
  lo = __uint_as_float(tf32_rna(__fsub_rn(x, hi)));
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// One K8 step of a warp's 32 x 16 tile at rows wm, columns wn: acc[mi][ni] (rows wm + 16 mi, columns wn + 8 ni)
// += A[rows][k, k + 8) B[k, k + 8)[columns] in 3xTF32.  A: ah / al [k][m], B: bh / bl [k][n].
__device__ __forceinline__ void warp_mma_3xtf32(float (&acc)[2][2][4], const float (*ah)[kTcPitch],
                                                const float (*al)[kTcPitch], const float (*bh)[kTcPitch],
                                                const float (*bl)[kTcPitch], int k, int wm, int wn, int g, int t) {
  uint32_t a_hi[2][4], a_lo[2][4], b_hi[2][2], b_lo[2][2];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi) {
    const int r = wm + mi * 16 + g;
    a_hi[mi][0] = __float_as_uint(ah[k + t][r]);
    a_hi[mi][1] = __float_as_uint(ah[k + t][r + 8]);
    a_hi[mi][2] = __float_as_uint(ah[k + t + 4][r]);
    a_hi[mi][3] = __float_as_uint(ah[k + t + 4][r + 8]);
    a_lo[mi][0] = __float_as_uint(al[k + t][r]);
    a_lo[mi][1] = __float_as_uint(al[k + t][r + 8]);
    a_lo[mi][2] = __float_as_uint(al[k + t + 4][r]);
    a_lo[mi][3] = __float_as_uint(al[k + t + 4][r + 8]);
  }
#pragma unroll
  for (int ni = 0; ni < 2; ++ni) {
    const int c = wn + ni * 8 + g;
    b_hi[ni][0] = __float_as_uint(bh[k + t][c]);
    b_hi[ni][1] = __float_as_uint(bh[k + t + 4][c]);
    b_lo[ni][0] = __float_as_uint(bl[k + t][c]);
    b_lo[ni][1] = __float_as_uint(bl[k + t + 4][c]);
  }
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 2; ++ni) {
      mma_tf32(acc[mi][ni], a_lo[mi], b_hi[ni]);
      mma_tf32(acc[mi][ni], a_hi[mi], b_lo[ni]);
      mma_tf32(acc[mi][ni], a_hi[mi], b_hi[ni]);
    }
}

// The 3xTF32 product of a K16 tile (two K8 steps from zero), added to acc with round-to-nearest
__device__ __forceinline__ void add_tile(float (&acc)[2][2][4], const float (*ah)[kTcPitch],
                                         const float (*al)[kTcPitch], const float (*bh)[kTcPitch],
                                         const float (*bl)[kTcPitch], int k, int wm, int wn, int g, int t) {
  float part[2][2][4] = {};
  warp_mma_3xtf32(part, ah, al, bh, bl, k, wm, wn, g, t);
  warp_mma_3xtf32(part, ah, al, bh, bl, k + 8, wm, wn, g, t);
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 2; ++ni)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[mi][ni][r] = __fadd_rn(acc[mi][ni][r], part[mi][ni][r]);
}

// k_simt_gemm's product on tensor cores, with its arguments, grid, 64 x 64 x 16 block tile and staging
// (gemm_tile, gemm_fetch, gemm_store).  Eight warps in 2 (M) x 4 (N), each a 32 x 16 tile of 2 x 2 MMA tiles.
// A thread stages its elements of the next K16 tile in registers while the warps multiply the current one.
template <class AOp>
__global__ void __launch_bounds__(256)
k_tc_gemm(AOp a, BOperand bop, const float* __restrict__ bias, float* __restrict__ C, int M, int N, int K,
          int relu, int kchunk) {
  __shared__ float Ah[BK][kTcPitch], Al[BK][kTcPitch];
  __shared__ float Bh[BK][kTcPitch], Bl[BK][kTcPitch];
  __shared__ int64_t s_rb[BM];
  __shared__ int64_t s_rb2[BM];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16;
  const GemmTile tile = gemm_tile(a, bop, M, K, kchunk, s_rb, s_rb2);
  __syncthreads();
  // the next K16 tile waits in registers
  float va[4], vb[4];
  auto load = [&](int k0) {
    gemm_fetch(a, bop, tile, k0, N, K, s_rb, s_rb2, [&](int i, int, int, float v) { va[i] = v; },
               [&](int i, int, int, float v) { vb[i] = v; });
  };
  float acc[2][2][4] = {};
  if (tile.kbeg < tile.kend) load(tile.kbeg);
  for (int k0 = tile.kbeg; k0 < tile.kend; k0 += BK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int2 qa = a_place(tid + i * 256), qb = b_place(bop.b_nk, tid + i * 256);
      split_tf32(va[i], Ah[qa.x][qa.y], Al[qa.x][qa.y]);
      split_tf32(vb[i], Bh[qb.x][qb.y], Bl[qb.x][qb.y]);
    }
    __syncthreads();
    if (k0 + BK < tile.kend) load(k0 + BK);
    add_tile(acc, Ah, Al, Bh, Bl, 0, wm, wn, g, t);
    __syncthreads();
  }
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 2; ++ni)
#pragma unroll
      for (int r = 0; r < 4; ++r)
        gemm_store(tile, acc[mi][ni][r], tile.m0 + wm + mi * 16 + g + (r >> 1) * 8,
                   tile.n0 + wn + ni * 8 + 2 * t + (r & 1), bias, relu, C, M, N);
}

// The training entry points set h->train_tc for their duration when the handle's training precision is
// OVN_TRAIN_TF32X3 (TrainPrecisionScope in api.cu); every other caller gets k_simt_gemm.
template <class AOp>
static int launch_gemm(ovn_handle* h, const AOp& a, const BOperand& b, const float* bias, float* C, int M,
                       int N, int K, int batch, int relu, cudaStream_t s, int kchunk = 0) {
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM, batch);
  if (h->train_tc) k_tc_gemm<AOp><<<grid, 256, 0, s>>>(a, b, bias, C, M, N, K, relu, kchunk);
  else k_simt_gemm<AOp><<<grid, 256, 0, s>>>(a, b, bias, C, M, N, K, relu, kchunk);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

// ---- Dense(1, sigmoid) over the flattened (H,W,C) c_conv3 output (generateNet.py:112-114) -----
__global__ void __launch_bounds__(256)
k_dense_sigmoid(const float* __restrict__ o3, const float* __restrict__ wd, const float* __restrict__ bd,
                int n_in, float* __restrict__ overlap) {
  __shared__ float red[256];
  const int p = blockIdx.x;
  const float* x = o3 + (int64_t)p * n_in;
  float acc = 0.f;
  for (int i = threadIdx.x; i < n_in; i += 256) acc = fmaf(x[i], __ldg(wd + i), acc);
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float zz = red[0] + bd[0];
    overlap[p] = 1.0f / (1.0f + expf(-zz));
  }
}

// ---- circular diagonal sums of the Gram matrix + argmax readout -------------------------------
//   corr[k] = sum_j G[(k + j + W/2) mod W, j]      (RangePadding2D.py:34 + NormalizedCorrelation2D.py:96-109)
//   yaw     = 180 - argmax_k corr[k], first maximum, at every Wf (infer.py:158, :198, :233 subtract from the
//             literal 180, not from Wf / 2)
__global__ void __launch_bounds__(384)
k_corr_readout(const float* __restrict__ G, int Wf, float* __restrict__ corr_out, int32_t* __restrict__ yaw) {
  extern __shared__ float s_corr[];
  const int p = blockIdx.x;
  const float* g = G + (int64_t)p * Wf * Wf;
  for (int k = threadIdx.x; k < Wf; k += blockDim.x) {
    float acc = 0.f;
    int i = k + Wf / 2;
    if (i >= Wf) i -= Wf;
    for (int j = 0; j < Wf; ++j) {
      acc += g[(int64_t)i * Wf + j];
      if (++i == Wf) i = 0;
    }
    s_corr[k] = acc;
    if (corr_out) corr_out[(int64_t)p * Wf + k] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int best = 0;
    float bv = s_corr[0];
    for (int k = 1; k < Wf; ++k)
      if (s_corr[k] > bv) { bv = s_corr[k]; best = k; }
    yaw[p] = 180 - best;
  }
}

// ---- drivers ----------------------------------------------------------------------------------
int leg_forward_fp32(ovn_handle* h, const float* d_input, int n, float* d_fv, cudaStream_t s) {
  const float* x = d_input;
  prof_mark(h, PROF_LEG, s);
  for (int l = 0; l < h->n_leg; ++l) {
    const ConvSpec& L = h->leg[l];
    float* y = (l == h->n_leg - 1) ? d_fv : h->d_act[l & 1];
    ConvOperand a{x, L.h_in, L.w_in, L.cin, L.kw, L.sh, L.sw, L.h_out, L.w_out};
    BOperand b{h->d_w[l], nullptr, nullptr, 0, 0};
    int rc = launch_gemm(h, a, b, h->d_b[l], y, n * L.h_out * L.w_out, L.cout, L.kh * L.kw * L.cin, 1, L.relu, s);
    if (rc != OVN_OK) return rc;
    x = y;
  }
  prof_mark(h, PROF_LEG, s);
  return OVN_OK;
}

// correlation head for <= max_batch_pairs pairs: Gram matrix per pair (fp32), then circular
// diagonal sums + argmax.  LEFT = bank[left[p]], RIGHT = query or bank[right[p]].
int corr_forward_fp32(ovn_handle* h, const float* d_bank, const float* d_query, const int32_t* left,
                      const int32_t* right, int np, int32_t* d_yaw, float* d_corr, cudaStream_t s) {
  const int Wf = h->cfg.leg_output_width, Cf = kFeatC;
  GramOperand a{d_bank, left, Wf, Cf};
  BOperand b{d_bank, d_query, right, (int64_t)Wf * Cf, 1};
  int rc = launch_gemm(h, a, b, nullptr, h->d_G, Wf, Wf, Cf, np, 0, s);
  if (rc != OVN_OK) return rc;
  k_corr_readout<<<np, 384, Wf * sizeof(float), s>>>(h->d_G, Wf, d_corr, d_yaw);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

// overlap head of np <= max_batch_pairs pairs: c_conv1 -> h->d_o1, c_conv2 -> h->d_o2, c_conv3 -> d_o3
// (which may alias d_o1: o1 is dead after c_conv2), Dense + sigmoid -> d_overlap
static int overlap_head_fp32(ovn_handle* h, const float* d_bank, const float* d_query, const int32_t* left,
                             const int32_t* right, int np, float* d_o3, float* d_overlap, cudaStream_t s) {
  const int Wf = h->cfg.leg_output_width, Cf = kFeatC, sz = h->cfg.conv1size;
  const int base = kMaxLegLayers;   // weight slots of c_conv1..3, overlap_output
  // c_conv1 (linear) on the implicit delta image
  {
    DeltaOperand a{d_bank, d_query, left, right, Wf, Cf, sz, h->o1_w};
    BOperand b{h->d_w[base + 0], nullptr, nullptr, 0, 0};
    prof_mark(h, PROF_DELTA, s);
    int rc = launch_gemm(h, a, b, h->d_b[base + 0], h->d_o1, np * h->o1_h * h->o1_w, h->head[0].cout,
                         sz * Cf, 1, 0, s);
    prof_mark(h, PROF_DELTA, s);
    if (rc != OVN_OK) return rc;
  }
  // c_conv2 (relu): (15,1) stride (15,1) over [p][360][24][64]
  {
    const ConvSpec& L = h->head[1];
    ConvOperand a{h->d_o1, L.h_in, L.w_in, L.cin, L.kw, L.sh, L.sw, L.h_out, L.w_out};
    BOperand b{h->d_w[base + 1], nullptr, nullptr, 0, 0};
    int rc = launch_gemm(h, a, b, h->d_b[base + 1], h->d_o2, np * L.h_out * L.w_out, L.cout,
                         L.kh * L.kw * L.cin, 1, 1, s);
    if (rc != OVN_OK) return rc;
  }
  // c_conv3 (relu) 3x3
  {
    const ConvSpec& L = h->head[2];
    ConvOperand a{h->d_o2, L.h_in, L.w_in, L.cin, L.kw, L.sh, L.sw, L.h_out, L.w_out};
    BOperand b{h->d_w[base + 2], nullptr, nullptr, 0, 0};
    int rc = launch_gemm(h, a, b, h->d_b[base + 2], d_o3, np * L.h_out * L.w_out, L.cout,
                         L.kh * L.kw * L.cin, 1, 1, s);
    if (rc != OVN_OK) return rc;
  }
  k_dense_sigmoid<<<np, 256, 0, s>>>(d_o3, h->d_w[base + 3], h->d_b[base + 3], h->dense_in, d_overlap);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

int heads_forward_fp32(ovn_handle* h, const float* d_bank, const float* d_query, const int32_t* d_left,
                       const int32_t* d_right, int n, float* d_overlap, int32_t* d_yaw, float* d_corr,
                       cudaStream_t s) {
  // the o3 buffer is d_o1 (o1 is dead after c_conv2)
  int rc = overlap_head_fp32(h, d_bank, d_query, d_left, d_right, n, h->d_o1, d_overlap, s);
  if (rc != OVN_OK) return rc;
  return corr_forward_fp32(h, d_bank, d_query, d_left, d_right, n, d_yaw, d_corr, s);
}

// ---- training of the overlap head with a frozen leg -------------------------------------------
// 360OutputkLegsFixed (generateNet.py:222-324): the leg is frozen, c_conv1..3 and overlap_output are
// trained.  All arithmetic is fp32, every reduction runs in a fixed order (split-K partials + a fixed-order
// reduction, no floating-point atomics), so two identical runs give bit-identical weights.

constexpr int kMaxSplit = 32;          // split-K slices of a weight-gradient product
constexpr int kSplitBlocks = 528;      // target CTAs of a split-K launch (4 per SM of a 132-SM H100)

// Losses of training.py:71-92,255-257 and dL/dz of the Dense logit.  One block: fixed summation order.
//   L_ov = mean_p sigmoid(u_p),  u_p = (|yhat_p - y_p| + 0.25) * 24 - 12
//   L_or = mean_p mean_k wce(t_pk, corr_pk, pos_weight = Wf),  t_pk = [k == gt_or_p and gt_ov_p > min_ov]
//          (targets of ImagePairOverlapOrientationSequence.py:118-121; the stable form of
//          tf.nn.weighted_cross_entropy_with_logits, the logits are raw correlation sums)
//   L = 5 L_ov + L_or;  dL/dyhat_p = 5 sigmoid'(u_p) * 24 * sign(yhat_p - y_p) / B  (sign(0) = 0, TF's abs)
//   dz_p = dL/dyhat_p * yhat_p (1 - yhat_p);  the Dense bias gradient = sum_p dz_p.
// dz is evaluated in double from the float32 yhat and y and rounded once, with sigmoid'(u) = e / (1 + e)^2,
// e = exp(-u): in float32, 1 - sigmoid(u) cancels as |yhat - y| grows (29 % off at 0.9, 0 at 0.95).  1 - yhat is
// exact for yhat >= 1/2, so yhat (1 - yhat) adds no cancellation of its own to the stored yhat's.
__global__ void __launch_bounds__(256)
k_train_loss(const float* __restrict__ ov, const float* __restrict__ corr, const float* __restrict__ gt_ov,
             const int32_t* __restrict__ gt_or, int np, int Wf, float min_ov, float* __restrict__ dz,
             float* __restrict__ g_bias_dense, float* __restrict__ loss) {
  __shared__ double r_ov[256], r_or[256];
  const int t = threadIdx.x;
  double a = 0.0, b = 0.0;
  for (int p = t; p < np; p += 256) {
    const float y = ov[p], d = y - gt_ov[p];
    const float u = (fabsf(d) + 0.25f) * 24.f - 12.f;
    const float sg = 1.f / (1.f + expf(-u));
    a += sg;
    const double dd = (double)y - (double)gt_ov[p];
    const double e = exp(-((fabs(dd) + 0.25) * 24.0 - 12.0));
    const double sgn = dd > 0.0 ? 1.0 : (dd < 0.0 ? -1.0 : 0.0);
    dz[p] = (float)(5.0 * 24.0 * e / ((1.0 + e) * (1.0 + e)) * sgn / np * ((double)y * (1.0 - (double)y)));
  }
  const float q = (float)Wf;
  for (int e = t; e < np * Wf; e += 256) {
    const int p = e / Wf, k = e - p * Wf;
    const float x = corr[e];
    const float z = (k == gt_or[p] && gt_ov[p] > min_ov) ? 1.f : 0.f;
    b += (1.f - z) * x + (1.f + (q - 1.f) * z) * (log1pf(expf(-fabsf(x))) + fmaxf(-x, 0.f));
  }
  r_ov[t] = a;
  r_or[t] = b;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (t < o) { r_ov[t] += r_ov[t + o]; r_or[t] += r_or[t + o]; }
    __syncthreads();
  }
  if (t == 0) {
    const double l_ov = r_ov[0] / np, l_or = r_or[0] / ((double)np * Wf);
    loss[0] = (float)(5.0 * l_ov + l_or);
    loss[1] = (float)l_ov;
    loss[2] = (float)l_or;
    float g = 0.f;
    for (int p = 0; p < np; ++p) g += dz[p];
    *g_bias_dense = g;
  }
}

// Dense backward: g_wd[i] = sum_p dz_p * x4[p, i] (pairs in order); then x4 is overwritten with
// dL/d(pre-activation of c_conv3) = dz_p * wd[i] where x4 > 0 (ReLU), 0 elsewhere.
__global__ void __launch_bounds__(256)
k_dense_backward(float* __restrict__ x4, const float* __restrict__ wd, const float* __restrict__ dz, int np,
                 int n_in, float* __restrict__ g_wd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_in) return;
  const float w = __ldg(wd + i);
  float g = 0.f;
  for (int p = 0; p < np; ++p) {
    float* x = x4 + (int64_t)p * n_in + i;
    const float v = *x;
    const float d = __ldg(dz + p);
    g = fmaf(d, v, g);
    *x = v > 0.f ? d * w : 0.f;
  }
  g_wd[i] = g;
}

// d <- d where x > 0, else 0 (gradient through a ReLU whose output is x)
__global__ void k_relu_grad(float* __restrict__ d, const float* __restrict__ x, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !(x[i] > 0.f)) d[i] = 0.f;
}

// conv kernel [taps][cin][cout] -> [taps][cout][cin] (the B operand of the input gradient)
__global__ void k_swap_io(const float* __restrict__ w, float* __restrict__ wt, int taps, int cin, int cout) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)taps * cin * cout) return;
  const int n = (int)(i % cout);
  const int64_t r = i / cout;
  const int c = (int)(r % cin);
  const int tap = (int)(r / cin);
  wt[((int64_t)tap * cout + n) * cin + c] = w[i];
}

// out[i] = sum_{z < nsplit} part[z][i], z in order
__global__ void k_splitk_reduce(const float* __restrict__ part, int nsplit, int64_t count, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float v = 0.f;
  for (int z = 0; z < nsplit; ++z) v += part[(int64_t)z * count + i];
  out[i] = v;
}

static unsigned blocks_for(int64_t n) { return (unsigned)((n + 255) / 256); }

// rows K and columns N of the gradient of head layer l (c_conv1..3, overlap_output); the gradient
// buffer holds [K + 1][N] per layer: the kernel in Keras layout, then the bias
static void head_dims(const ovn_handle* h, int l, int* K, int* N) {
  if (l < 3) { const ConvSpec& L = h->head[l]; *K = L.kh * L.kw * L.cin; *N = L.cout; }
  else { *K = h->dense_in; *N = 1; }
}

// The bytes of the buffers train_alloc makes, in its order: x4, dx3, corr, overlap, dz, yaw, w3t, grad, accum,
// loss, then the split-K partials (part, which net_alloc may grow)
constexpr int kTrainBufs = 11;
static void train_sizes(const ovn_handle* h, size_t b[kTrainBufs]) {
  const int64_t maxp = h->cfg.max_batch_pairs, Wf = h->cfg.leg_output_width;
  const ConvSpec& L3 = h->head[2];
  const int64_t total = h->params.n_total;
  int64_t max_part = 0;
  for (int l = 0; l < 3; ++l) {
    int K, N;
    head_dims(h, l, &K, &N);
    if ((int64_t)(K + 1) * N > max_part) max_part = (int64_t)(K + 1) * N;
  }
  const size_t sizes[kTrainBufs] = {
      (size_t)maxp * h->dense_in * sizeof(float), (size_t)maxp * L3.h_in * L3.w_in * L3.cin * sizeof(float),
      (size_t)maxp * Wf * sizeof(float), (size_t)maxp * sizeof(float), (size_t)maxp * sizeof(float),
      (size_t)maxp * sizeof(int32_t), (size_t)L3.kh * L3.kw * L3.cin * L3.cout * sizeof(float),
      (size_t)total * sizeof(float), (size_t)total * sizeof(float), 4 * sizeof(float),
      (size_t)kMaxSplit * max_part * sizeof(float)};
  for (int i = 0; i < kTrainBufs; ++i) b[i] = sizes[i];
}

// h->train, complete or not at all
int train_alloc(ovn_handle* h) {
  const int64_t total = h->params.n_total;
  std::unique_ptr<TrainState> t(new TrainState());
  size_t b[kTrainBufs];
  train_sizes(h, b);
  int rc;
  if ((rc = t->x4.ensure(h, b[0])) != OVN_OK) return rc;
  if ((rc = t->dx3.ensure(h, b[1])) != OVN_OK) return rc;
  if ((rc = t->corr.ensure(h, b[2])) != OVN_OK) return rc;
  if ((rc = t->overlap.ensure(h, b[3])) != OVN_OK) return rc;
  if ((rc = t->dz.ensure(h, b[4])) != OVN_OK) return rc;
  if ((rc = t->yaw.ensure(h, b[5])) != OVN_OK) return rc;
  if ((rc = t->w3t.ensure(h, b[6])) != OVN_OK) return rc;
  if ((rc = t->part.ensure(h, b[10])) != OVN_OK) return rc;
  if ((rc = t->grad.ensure(h, b[7])) != OVN_OK) return rc;
  if ((rc = t->accum.ensure(h, b[8])) != OVN_OK) return rc;
  if ((rc = t->loss.ensure(h, b[9])) != OVN_OK) return rc;
  OVN_CUDA(h, cudaMemset(t->accum, 0, (size_t)total * sizeof(float)));
  h->train = std::move(t);
  return OVN_OK;
}

// [Kc + 1][N] weight + bias gradient = A^T dY summed over Kred rows, split over K in fixed slices
template <class AOp>
static int wgrad_gemm(ovn_handle* h, const AOp& a, const float* dY, int Kc, int N, int Kred, float* grad,
                      cudaStream_t s) {
  const int M = Kc + 1;
  const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
  int nsplit = (kSplitBlocks + tiles - 1) / tiles;
  if (nsplit > kMaxSplit) nsplit = kMaxSplit;
  int kchunk = (Kred + nsplit - 1) / nsplit;
  kchunk = (kchunk + BK - 1) / BK * BK;
  nsplit = (Kred + kchunk - 1) / kchunk;
  BOperand b{dY, nullptr, nullptr, 0, 0};
  int rc = launch_gemm(h, a, b, nullptr, h->train->part, M, N, Kred, nsplit, 0, s, kchunk);
  if (rc != OVN_OK) return rc;
  k_splitk_reduce<<<blocks_for((int64_t)M * N), 256, 0, s>>>(h->train->part, nsplit, (int64_t)M * N, grad);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

// Forward of both heads, the losses and the backward of the overlap head for np <= max_batch_pairs pairs
// (indices already bounds-checked).  Activations kept for the backward: o1 (h->d_o1), x3 = c_conv2 output
// (h->d_o2), x4 = c_conv3 output (train->x4).  Each buffer is reused for a gradient once it is dead:
// x4 -> dL/d(pre-act c_conv3), o1 -> dL/do1.  The losses are left in ch.loss.
// The forward, every input gradient and every ReLU mask compute each pair on its own, so they run once over all np
// pairs.  Where the batch enters a sum or a scale -- the losses and dz's 1 / n, the Dense sums over pairs and every
// split-K weight gradient, whose slices follow its own reduction length -- each chunk runs on its own pairs, one
// chunk after the other, into its own gradients.  One chunk is the launch sequence of a plain call.
int head_gradients_fp32(ovn_handle* h, const float* d_bank, const int32_t* left, const int32_t* right, int np,
                        const float* d_gt_overlap, const int32_t* d_gt_orientation, float min_overlap,
                        const GradChunks& ch, cudaStream_t s) {
  TrainState& t = *h->train;
  const int Wf = h->cfg.leg_output_width, Cf = kFeatC, sz = h->cfg.conv1size;
  const int base = kMaxLegLayers;
  const int64_t* off = h->params.off + base;   // gradients of c_conv1..3, overlap_output
  const ConvSpec& L1 = h->head[0];
  const ConvSpec& L2 = h->head[1];
  const ConvSpec& L3 = h->head[2];
  const int64_t o1_pair = (int64_t)L2.h_in * L2.w_in * L2.cin, x3_pair = (int64_t)L3.h_in * L3.w_in * L3.cin;
  int K[4], N[4];
  for (int l = 0; l < 4; ++l) head_dims(h, l, &K[l], &N[l]);
  int rc = overlap_head_fp32(h, d_bank, nullptr, left, right, np, t.x4, t.overlap, s);
  if (rc == OVN_OK) rc = corr_forward_fp32(h, d_bank, nullptr, left, right, np, t.yaw, t.corr, s);
  if (rc != OVN_OK) return rc;
  if (train_stop_here(t, OVN_TRAIN_STAGE_O1, 0, h->d_o1) || train_stop_here(t, OVN_TRAIN_STAGE_X4, 0, t.x4))
    return OVN_OK;
  for (int c = 0; c < ch.n; ++c) {
    const int a = ch.off[c], n = ch.size(c);
    if (n == 0) continue;
    float* g = ch.grad + c * ch.stride;
    k_train_loss<<<1, 256, 0, s>>>(t.overlap + a, t.corr + (int64_t)a * Wf, d_gt_overlap + a, d_gt_orientation + a,
                                   n, Wf, min_overlap, t.dz + a, g + off[3] + K[3], ch.loss + 3 * c);
    OVN_LAUNCH_CHECK(h);
    // overlap_output (Dense): dWd, and x4 becomes dL/d(pre-activation of c_conv3)
    k_dense_backward<<<blocks_for(h->dense_in), 256, 0, s>>>(t.x4 + (int64_t)a * h->dense_in, h->d_w[base + 3],
                                                             t.dz + a, n, h->dense_in, g + off[3]);
    OVN_LAUNCH_CHECK(h);
  }
  // c_conv3: dW3 = patches(x3)^T dpre3 (+ db3), then dx3 = transposed 3x3 conv of dpre3, masked by x3 > 0
  {
    for (int c = 0; c < ch.n; ++c) {
      const int a = ch.off[c], n = ch.size(c);
      if (n == 0) continue;
      ConvWgradOperand op{h->d_o2 + a * x3_pair, L3.h_in, L3.w_in, L3.cin, L3.kw, L3.sh, L3.sw, L3.h_out, L3.w_out,
                          K[2]};
      rc = wgrad_gemm(h, op, t.x4 + (int64_t)a * h->dense_in, K[2], N[2], n * L3.h_out * L3.w_out,
                      ch.grad + c * ch.stride + off[2], s);
      if (rc != OVN_OK) return rc;
    }
    k_swap_io<<<blocks_for((int64_t)K[2] * N[2]), 256, 0, s>>>(h->d_w[base + 2], t.w3t, L3.kh * L3.kw, L3.cin,
                                                               L3.cout);
    OVN_LAUNCH_CHECK(h);
    ConvDgradOperand d{t.x4, L3.h_out, L3.w_out, L3.cout, L3.kw, L3.h_in, L3.w_in};
    BOperand b{t.w3t, nullptr, nullptr, 0, 0};
    rc = launch_gemm(h, d, b, nullptr, t.dx3, np * L3.h_in * L3.w_in, L3.cin, L3.kh * L3.kw * L3.cout, 1, 0, s);
    if (rc != OVN_OK) return rc;
    const int64_t n3 = (int64_t)np * L3.h_in * L3.w_in * L3.cin;
    k_relu_grad<<<blocks_for(n3), 256, 0, s>>>(t.dx3, h->d_o2, n3);
    OVN_LAUNCH_CHECK(h);
  }
  // c_conv2: dW2 = patches(o1)^T dpre2 (+ db2); do1 = dpre2 W2^T.  Stride = kernel, so every o1 row belongs to
  // exactly one output pixel: do1 is stored per output pixel, [p][ho][wo][dh][c], over the dead o1
  {
    for (int c = 0; c < ch.n; ++c) {
      const int a = ch.off[c], n = ch.size(c);
      if (n == 0) continue;
      ConvWgradOperand op{h->d_o1 + a * o1_pair, L2.h_in, L2.w_in, L2.cin, L2.kw, L2.sh, L2.sw, L2.h_out, L2.w_out,
                          K[1]};
      rc = wgrad_gemm(h, op, t.dx3 + a * x3_pair, K[1], N[1], n * L2.h_out * L2.w_out,
                      ch.grad + c * ch.stride + off[1], s);
      if (rc != OVN_OK) return rc;
    }
    ConvOperand g{t.dx3, L2.h_out, L2.w_out, L2.cout, 1, 1, 1, L2.h_out, L2.w_out};
    BOperand w2t{h->d_w[base + 1], h->d_w[base + 1], nullptr, 0, 1};     // W2 read as [(dh, c)][n]
    rc = launch_gemm(h, g, w2t, nullptr, h->d_o1, np * L2.h_out * L2.w_out, K[1], L2.cout, 1, 0, s);
    if (rc != OVN_OK) return rc;
  }
  // c_conv1 (linear): dW1[dj, c, o] = sum |L[i, c] - R[15 jb + dj, c]| do1[i, jb, o], db1 = sum do1
  for (int c = 0; c < ch.n; ++c) {
    const int a = ch.off[c], n = ch.size(c);
    if (n == 0) continue;
    DeltaWgradOperand op{d_bank, left + a, right + a, Wf, Cf, sz, h->o1_w, L2.h_out, K[0]};
    rc = wgrad_gemm(h, op, h->d_o1 + a * o1_pair, K[0], N[0], n * L1.h_out * L1.w_out,
                    ch.grad + c * ch.stride + off[0], s);
    if (rc != OVN_OK) return rc;
  }
  return OVN_OK;
}

// ---- training of the whole network (360OutputkLegs) -------------------------------------------
// The leg is trained too: the gradient of both heads flows back into the two feature volumes (through |l - r|
// and the correlation head) and from there through the leg's convolutions.  Same rules as the head: fp32,
// fixed-order reductions, no floating-point atomics.

constexpr int kDgT = 64;         // k_delta_dgrad tile: 64 rows i x 64 channels c, K = the 64 c_conv1 outputs
constexpr int kCorrRows = 8;     // k_corr_backward: output rows per CTA

// out[v] = images[left[v]] for v < np, images[right[v - np]] for v >= np  (indices already bounds-checked)
__global__ void k_gather_images(const float* __restrict__ images, const int32_t* __restrict__ left,
                                const int32_t* __restrict__ right, int np, int64_t img, float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * np * img) return;
  const int v = (int)(i / img);
  const int src = v < np ? left[v] : right[v - np];
  out[i] = __ldg(images + (int64_t)src * img + (i - (int64_t)v * img));
}

__global__ void k_pair_rows(int32_t* __restrict__ rows, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rows[i] = i;
}

// The volume rows of a chunked batch, whose images are chunk after chunk, each [LEFT of its pairs, RIGHT of its
// pairs] from 2 off[c]: rows[p] = p + off[c] (LEFT of pair p of chunk c), rows[np + p] = p + off[c + 1] (RIGHT)
__global__ void k_chunk_pair_rows(int32_t* __restrict__ rows, int np, const __grid_constant__ GradChunks ch) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= np) return;
  int c = 0;
  while (p >= ch.off[c + 1]) ++c;
  rows[p] = p + ch.off[c];
  rows[np + p] = p + ch.off[c + 1];
}

// dL/d(correlation logit) of the orientation loss of k_train_loss (loss weight 1):
//   dcorr[p, k] = ((1 - t) - (1 + (Wf - 1) t) sigmoid(-corr)) / (np Wf),  t = [k == gt_or_p and gt_ov_p > min_ov]
__global__ void k_corr_dlogit(const float* __restrict__ corr, const float* __restrict__ gt_ov,
                              const int32_t* __restrict__ gt_or, int np, int Wf, float min_ov, float* __restrict__ dcorr) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= np * Wf) return;
  const int p = e / Wf, k = e - p * Wf;
  const float t = (k == gt_or[p] && gt_ov[p] > min_ov) ? 1.f : 0.f;
  const float sg = 1.f / (1.f + expf(corr[e]));
  dcorr[e] = ((1.f - t) - (1.f + ((float)Wf - 1.f) * t) * sg) / ((float)np * (float)Wf);
}

// Backward of corr[p, k] = sum_{j,c} L[(k + j + Wf/2) mod Wf, c] R[j, c]  (RangePadding2D.py:31-38 +
// NormalizedCorrelation2D.py:96-109), a circulant times a volume:
//   side 0: dL[p, i, :] = sum_j dcorr[p, (i - j - Wf/2) mod Wf] R[j, :]  -> dfv[p]
//   side 1: dR[p, j, :] = sum_i dcorr[p, (i - j - Wf/2) mod Wf] L[i, :]  -> dfv[np + p]
// CTA = (kCorrRows output rows, pair, side), one thread per channel; the sum runs over q in order.
__global__ void __launch_bounds__(kFeatC)
k_corr_backward(const float* __restrict__ dcorr, const float* __restrict__ fv, const int32_t* __restrict__ left,
                const int32_t* __restrict__ right, int np, int Wf, float* __restrict__ dfv) {
  extern __shared__ float s_d[];
  const int r0 = blockIdx.x * kCorrRows, p = blockIdx.y, side = blockIdx.z, c = threadIdx.x;
  for (int k = c; k < Wf; k += kFeatC) s_d[k] = dcorr[(int64_t)p * Wf + k];
  __syncthreads();
  const float* X = fv + (int64_t)(side ? left[p] : right[p]) * Wf * kFeatC;
  const int half = Wf / 2;
  // index of dcorr for output row r0 + rr and input row q: side 0 (r0 + rr - q - half), side 1 (q - r0 - rr - half)
  int base = side ? (-r0 - half) % Wf : (r0 - half) % Wf;
  if (base < 0) base += Wf;
  float acc[kCorrRows] = {};
  for (int q = 0; q < Wf; ++q) {
    const float x = __ldg(X + (int64_t)q * kFeatC + c);
#pragma unroll
    for (int rr = 0; rr < kCorrRows; ++rr) {
      int idx = side ? base - rr : base + rr;   // wraps once when Wf >= kCorrRows, more often below that
      while (idx < 0) idx += Wf;
      while (idx >= Wf) idx -= Wf;
      acc[rr] = fmaf(s_d[idx], x, acc[rr]);
    }
    base = side ? (base + 1 == Wf ? 0 : base + 1) : (base == 0 ? Wf - 1 : base - 1);
  }
#pragma unroll
  for (int rr = 0; rr < kCorrRows; ++rr)
    if (r0 + rr < Wf) dfv[(((int64_t)side * np + p) * Wf + r0 + rr) * kFeatC + c] = acc[rr];
}

// Backward of c_conv1 on |l - r| (generateNet.py:45-59,96-100) without the 66 MB delta tensor.  With
// do1[p, i, jb, o] = dL/d(c_conv1 output) (h->d_o1, stored [p][ho][jb][dh][o], i = s ho + dh), j = s jb + dj:
//   G[i, dj, c] = sum_o do1[p, i, jb, o] W1[dj, c, o],   sg = sign(L[i, c] - R[j, c])  (sign(0) = 0, TF's abs)
//   dL[p, i, c] = sum_{jb, dj} sg G,   dR[p, j, c] = -sum_i sg G
// CTA = (64 channels, 64 rows i, jb + nb p): the do1 tile stays in shared memory while the CTA loops over the
// s taps dj; each tap is a 64 x 64 x 64 product in registers whose epilogue applies the signs.  Fixed-order
// partials, reduced by k_delta_dgrad_reduce:  part_l[p][jb][i][c] (this CTA's sum over dj) and
// part_r[p][row tile][j][c] (this CTA's sum over its 64 rows, in order).
//
// k_delta_dgrad and k_delta_dgrad_tc share the CTA's addresses (DeltaDgradCta) and the staging of its do1 and W1
// tiles.  The tiles are stored transposed: a thread reads 4 consecutive o of one row and consecutive threads take
// consecutive rows, so the shared-memory stores of a warp hit 32 different banks.
struct DeltaDgradCta {
  int c0, itile, i0, jb, p, nit;
  __device__ __forceinline__ explicit DeltaDgradCta(int nb)
      : c0(blockIdx.x * kDgT), itile(blockIdx.y), i0(blockIdx.y * kDgT), jb(blockIdx.z % nb), p(blockIdx.z / nb),
        nit(gridDim.y) {}
  // the pair's LEFT (rows = left) or RIGHT (rows = right) volume
  __device__ __forceinline__ const float* volume(const float* fv, const int32_t* rows, int Wf) const {
    return fv + (int64_t)rows[p] * Wf * kFeatC;
  }
  // channel c0 of row i of this CTA's part_l, and of column j of its part_r
  __device__ __forceinline__ float* part_l_at(float* part_l, int nb, int Wf, int i) const {
    return part_l + (((int64_t)p * nb + jb) * Wf + i) * kFeatC + c0;
  }
  __device__ __forceinline__ float* part_r_at(float* part_r, int Wf, int j) const {
    return part_r + (((int64_t)p * nit + itile) * Wf + j) * kFeatC + c0;
  }
};

// put(o, r, v) for the do1 tile's 64 rows i0 + r (zero past Wf) and 64 outputs o
template <class Put>
__device__ __forceinline__ void stage_do1(const DeltaDgradCta& cta, const float* do1, int Wf, int s, int nb, int nho,
                                          Put put) {
  for (int f = threadIdx.x; f < kDgT * kDgT / 4; f += 256) {
    const int r = f % kDgT, o = (f / kDgT) * 4, i = cta.i0 + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i < Wf) {
      const int ho = i / s, dh = i - ho * s;
      v = __ldg(reinterpret_cast<const float4*>(do1 + ((((int64_t)cta.p * nho + ho) * nb + cta.jb) * s + dh) * kDgT + o));
    }
    put(o, r, v.x); put(o + 1, r, v.y); put(o + 2, r, v.z); put(o + 3, r, v.w);
  }
}

// put(o, c, v) for tap dj's W1 tile: 64 channels c0 + c, 64 outputs o
template <class Put>
__device__ __forceinline__ void stage_w1(const DeltaDgradCta& cta, const float* w1, int dj, Put put) {
  for (int f = threadIdx.x; f < kDgT * kDgT / 4; f += 256) {
    const int c = f % kDgT, o = (f / kDgT) * 4;
    const float4 v = __ldg(reinterpret_cast<const float4*>(w1 + ((int64_t)dj * kFeatC + cta.c0 + c) * kDgT + o));
    put(o, c, v.x); put(o + 1, c, v.y); put(o + 2, c, v.z); put(o + 3, c, v.w);
  }
}

__global__ void __launch_bounds__(256)
k_delta_dgrad(const float* __restrict__ do1, const float* __restrict__ w1, const float* __restrict__ fv,
              const int32_t* __restrict__ left, const int32_t* __restrict__ right, int Wf, int s, int nb, int nho,
              float* __restrict__ part_l, float* __restrict__ part_r) {
  __shared__ __align__(16) float As[kDgT][kDgT + 4];     // [o][i]
  __shared__ __align__(16) float Bs[kDgT][kDgT + 4];     // [o][c]
  __shared__ float red[16][kDgT];
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  const DeltaDgradCta cta(nb);
  stage_do1(cta, do1, Wf, s, nb, nho, [&](int o, int r, float v) { As[o][r] = v; });
  const float* L = cta.volume(fv, left, Wf);
  const float* R = cta.volume(fv, right, Wf);
  float lv[4][4], accl[4][4];
#pragma unroll
  for (int ii = 0; ii < 4; ++ii) {
    const int i = cta.i0 + ty * 4 + ii;
    const float4 v = i < Wf ? __ldg(reinterpret_cast<const float4*>(L + (int64_t)i * kFeatC + cta.c0 + tx * 4))
                            : make_float4(0.f, 0.f, 0.f, 0.f);
    lv[ii][0] = v.x; lv[ii][1] = v.y; lv[ii][2] = v.z; lv[ii][3] = v.w;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) accl[ii][jj] = 0.f;
  }
  for (int dj = 0; dj < s; ++dj) {
    stage_w1(cta, w1, dj, [&](int o, int c, float v) { Bs[o][c] = v; });
    __syncthreads();
    float acc[4][4] = {};
#pragma unroll 8
    for (int o = 0; o < kDgT; ++o) {
      const float4 a = *reinterpret_cast<const float4*>(&As[o][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[o][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int ii = 0; ii < 4; ++ii)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) acc[ii][jj] = fmaf(av[ii], bv[jj], acc[ii][jj]);
    }
    const int j = s * cta.jb + dj;
    const float4 r4 = __ldg(reinterpret_cast<const float4*>(R + (int64_t)j * kFeatC + cta.c0 + tx * 4));
    const float rv[4] = {r4.x, r4.y, r4.z, r4.w};
    float col[4] = {};
#pragma unroll
    for (int ii = 0; ii < 4; ++ii)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const float d = lv[ii][jj] - rv[jj];
        const float v = d > 0.f ? acc[ii][jj] : (d < 0.f ? -acc[ii][jj] : 0.f);
        accl[ii][jj] += v;
        col[jj] += v;
      }
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) red[ty][tx * 4 + jj] = col[jj];
    __syncthreads();
    if (tid < kDgT) {
      float v = 0.f;
#pragma unroll
      for (int y = 0; y < 16; ++y) v += red[y][tid];
      cta.part_r_at(part_r, Wf, j)[tid] = -v;
    }
  }
#pragma unroll
  for (int ii = 0; ii < 4; ++ii) {
    const int i = cta.i0 + ty * 4 + ii;
    if (i < Wf)
      *reinterpret_cast<float4*>(cta.part_l_at(part_l, nb, Wf, i) + tx * 4) =
          make_float4(accl[ii][0], accl[ii][1], accl[ii][2], accl[ii][3]);
  }
}

// k_delta_dgrad with its per-tap G = do1 W1^T on 3xTF32 mma.sync: the same grid, CTA tile, partial layout and
// sign rule.  The do1 tile is split into hi / lo planes once, each tap's W1 tile when it is staged.  Eight warps
// in 2 (rows i) x 4 (channels c), each a 32 x 16 tile; the signs are applied to the accumulator fragments.  A
// tap's column sums for part_r add a thread's four rows, then the eight lanes of a column (butterfly over lane
// bits 2..4), then the two row warps, always in that order.
constexpr int kDgTcSmem = (4 * kDgT * kTcPitch + 2 * kDgT) * (int)sizeof(float);

__global__ void __launch_bounds__(256)
k_delta_dgrad_tc(const float* __restrict__ do1, const float* __restrict__ w1, const float* __restrict__ fv,
                 const int32_t* __restrict__ left, const int32_t* __restrict__ right, int Wf, int s, int nb, int nho,
                 float* __restrict__ part_l, float* __restrict__ part_r) {
  extern __shared__ __align__(16) float smem[];
  float (*Ah)[kTcPitch] = reinterpret_cast<float (*)[kTcPitch]>(smem);     // [o][i]
  float (*Al)[kTcPitch] = Ah + kDgT;
  float (*Bh)[kTcPitch] = Al + kDgT;                                      // [o][c]
  float (*Bl)[kTcPitch] = Bh + kDgT;
  float (*red)[kDgT] = reinterpret_cast<float (*)[kDgT]>(Bl + kDgT);    // [row warp][c]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16;
  const DeltaDgradCta cta(nb);
  stage_do1(cta, do1, Wf, s, nb, nho, [&](int o, int r, float v) { split_tf32(v, Ah[o][r], Al[o][r]); });
  const float* L = cta.volume(fv, left, Wf);
  const float* R = cta.volume(fv, right, Wf);
  // fragment element (mi, ni, r): row i0 + wm + 16 mi + g + 8 (r / 2), channel c0 + wn + 8 ni + 2 t + r % 2
  float lv[2][2][4], accl[2][2][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int h8 = 0; h8 < 2; ++h8) {
      const int i = cta.i0 + wm + mi * 16 + g + h8 * 8;
#pragma unroll
      for (int ni = 0; ni < 2; ++ni) {
        const float2 v = i < Wf ? __ldg(reinterpret_cast<const float2*>(L + (int64_t)i * kFeatC + cta.c0 + wn + ni * 8 + 2 * t))
                                : make_float2(0.f, 0.f);
        lv[mi][ni][2 * h8] = v.x;
        lv[mi][ni][2 * h8 + 1] = v.y;
        accl[mi][ni][2 * h8] = 0.f;
        accl[mi][ni][2 * h8 + 1] = 0.f;
      }
    }
  for (int dj = 0; dj < s; ++dj) {
    stage_w1(cta, w1, dj, [&](int o, int c, float v) { split_tf32(v, Bh[o][c], Bl[o][c]); });
    __syncthreads();
    float acc[2][2][4] = {};
#pragma unroll
    for (int k = 0; k < kDgT; k += 16) add_tile(acc, Ah, Al, Bh, Bl, k, wm, wn, g, t);
    const int j = s * cta.jb + dj;
    float rv[2][2], col[2][2] = {};
#pragma unroll
    for (int ni = 0; ni < 2; ++ni) {
      const float2 v = __ldg(reinterpret_cast<const float2*>(R + (int64_t)j * kFeatC + cta.c0 + wn + ni * 8 + 2 * t));
      rv[ni][0] = v.x;
      rv[ni][1] = v.y;
    }
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 2; ++ni)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const float d = lv[mi][ni][r] - rv[ni][r & 1];
          const float a = acc[mi][ni][r];
          const float v = d > 0.f ? a : (d < 0.f ? -a : 0.f);
          accl[mi][ni][r] += v;
          col[ni][r & 1] += v;
        }
#pragma unroll
    for (int ni = 0; ni < 2; ++ni)
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        float v = col[ni][b];
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        v += __shfl_xor_sync(0xffffffffu, v, 8);
        v += __shfl_xor_sync(0xffffffffu, v, 16);
        if (g == 0) red[wm / 32][wn + ni * 8 + 2 * t + b] = v;
      }
    __syncthreads();
    if (tid < kDgT) cta.part_r_at(part_r, Wf, j)[tid] = -(red[0][tid] + red[1][tid]);
  }
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int h8 = 0; h8 < 2; ++h8) {
      const int i = cta.i0 + wm + mi * 16 + g + h8 * 8;
      if (i >= Wf) continue;
#pragma unroll
      for (int ni = 0; ni < 2; ++ni)
        *reinterpret_cast<float2*>(cta.part_l_at(part_l, nb, Wf, i) + wn + ni * 8 + 2 * t) =
            make_float2(accl[mi][ni][2 * h8], accl[mi][ni][2 * h8 + 1]);
    }
}

// dfv[v] += the partials of volume v in order: LEFT p (v = p) sums nb partials, RIGHT p (v = np + p) nit
__global__ void k_delta_dgrad_reduce(const float* __restrict__ part_l, const float* __restrict__ part_r, int np, int nb,
                                     int nit, int64_t vol, float* __restrict__ dfv) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * np * vol) return;
  const int v = (int)(i / vol);
  const int64_t e = i - (int64_t)v * vol;
  const float* src = v < np ? part_l + (int64_t)v * nb * vol + e : part_r + (int64_t)(v - np) * nit * vol + e;
  const int n = v < np ? nb : nit;
  float acc = dfv[i];
  for (int z = 0; z < n; ++z) acc += src[(int64_t)z * vol];
  dfv[i] = acc;
}

constexpr int64_t kMaxGridY = 65535;   // k_simt_gemm puts row tiles on grid.y, k_delta_dgrad pairs x jb on grid.z

// Images per k_simt_gemm launch of the leg, whose rows are `rows` per image: the row tiles must fit grid.y.
// Every output element is computed the same way in any launch, so splitting changes no result.
static int images_per_launch(int64_t rows) {
  const int64_t n = kMaxGridY * BM / rows;
  return n < 1 ? 1 : (int)(n > INT32_MAX ? INT32_MAX : n);
}

// The largest batch ovn_net_gradients can launch: the heads put np * 360 * 24 rows of c_conv1 on one grid
// (485 pairs at Wf = 360), k_delta_dgrad puts np * 24 CTAs on grid.z.  The leg launches split over images.
int net_max_pairs(const ovn_handle* h) {
  const int64_t by_rows = kMaxGridY * BM / ((int64_t)h->o1_h * h->o1_w);
  const int64_t by_z = kMaxGridY / h->o1_w;
  return (int)(by_rows < by_z ? by_rows : by_z);
}

// The bytes of the whole-network buffers of an np-pair batch, in net_alloc's order: images, acts, dact[0],
// dact[1], dfv_part, dcorr, pair_rows, wt, then the split-K partials (part, shared with train_alloc)
constexpr int kNetBufs = 9;
static void net_sizes(const ovn_handle* h, int np, size_t b[kNetBufs]) {
  const int64_t n2 = 2 * (int64_t)np, Wf = h->cfg.leg_output_width, vol = Wf * kFeatC;
  const int64_t img = (int64_t)h->cfg.proj_H * h->cfg.proj_W * h->C;
  const int nb = h->o1_w, nit = (int)((Wf + kDgT - 1) / kDgT);
  int64_t acts = 0, max_act = vol, max_w = 0, max_part = 0;
  for (int l = 0; l < h->n_leg; ++l) {
    const ConvSpec& L = h->leg[l];
    const int64_t a = (int64_t)L.h_out * L.w_out * L.cout;
    acts += a;
    if (a > max_act) max_act = a;
    if (l > 0 && (int64_t)L.h_in * L.w_in * L.cin > max_act) max_act = (int64_t)L.h_in * L.w_in * L.cin;
    const int64_t w = h->params.n_kernel[l], g = w + L.cout;
    if (w > max_w) max_w = w;
    if (g > max_part) max_part = g;
  }
  const size_t sizes[kNetBufs] = {
      (size_t)(n2 * img) * sizeof(float), (size_t)(n2 * acts) * sizeof(float),
      (size_t)(n2 * max_act) * sizeof(float), (size_t)(n2 * max_act) * sizeof(float),
      (size_t)(np * (int64_t)(nb + nit) * vol) * sizeof(float), (size_t)(np * Wf) * sizeof(float),
      (size_t)n2 * sizeof(int32_t), (size_t)max_w * sizeof(float), (size_t)kMaxSplit * max_part * sizeof(float)};
  for (int i = 0; i < kNetBufs; ++i) b[i] = sizes[i];
}

static int net_alloc(ovn_handle* h, int np) {
  TrainState& t = *h->train;
  size_t b[kNetBufs];
  net_sizes(h, np, b);
  int rc;
  if ((rc = t.images.ensure(h, b[0])) != OVN_OK) return rc;
  if ((rc = t.acts.ensure(h, b[1])) != OVN_OK) return rc;
  for (int k = 0; k < 2; ++k)
    if ((rc = t.dact[k].ensure(h, b[2 + k])) != OVN_OK) return rc;
  if ((rc = t.dfv_part.ensure(h, b[4])) != OVN_OK) return rc;
  if ((rc = t.dcorr.ensure(h, b[5])) != OVN_OK) return rc;
  if ((rc = t.pair_rows.ensure(h, b[6])) != OVN_OK) return rc;
  if ((rc = t.wt.ensure(h, b[7])) != OVN_OK) return rc;
  return t.part.ensure(h, b[8]);
}

// The device bytes the training buffers of a handle take once it has trained n_pairs-pair batches: train_alloc's,
// and with whole_network net_alloc's; the split-K partials are one buffer, the larger of the two
int64_t train_workspace_bytes(const ovn_handle* h, bool whole_network, int np) {
  size_t t[kTrainBufs], n[kNetBufs];
  train_sizes(h, t);
  int64_t bytes = 0;
  for (int i = 0; i < kTrainBufs - 1; ++i) bytes += (int64_t)t[i];
  size_t part = t[kTrainBufs - 1];
  if (whole_network) {
    net_sizes(h, np, n);
    for (int i = 0; i < kNetBufs - 1; ++i) bytes += (int64_t)n[i];
    if (n[kNetBufs - 1] > part) part = n[kNetBufs - 1];
  }
  return bytes + (int64_t)part;
}

// Forward of the leg on the 2 np gathered images (the launches of leg_forward_fp32, every output kept), both
// heads, the losses, and the backward of the whole network.  The gradients of every layer land in train->grad,
// the losses in train->loss; d_fv_grad (may be null) receives dL/d(volumes) before s_conv10's ReLU mask,
// [2][np][Wf][128].
// With chunks (head_gradients_fp32), the images of chunk c are gathered as a call on its pairs alone gathers them,
// [LEFT, RIGHT] from image 2 off[c], so that a leg layer's weight gradient of chunk c reduces over the same rows in
// the same order.  dL/d(volumes), which the head backward leaves as [LEFT][RIGHT] over all pairs, is copied into
// that order before the leg backward.
int net_gradients_fp32(ovn_handle* h, const float* d_images, const int32_t* left, const int32_t* right, int np,
                       const float* d_gt_overlap, const int32_t* d_gt_orientation, float min_overlap,
                       float* d_fv_grad, const GradChunks& ch, cudaStream_t s) {
  int rc = net_alloc(h, np);
  if (rc != OVN_OK) return rc;
  TrainState& t = *h->train;
  const int Wf = h->cfg.leg_output_width, n2 = 2 * np, sz = h->cfg.conv1size;
  const int64_t img = (int64_t)h->cfg.proj_H * h->cfg.proj_W * h->C, vol = (int64_t)Wf * kFeatC;
  const int nb = h->o1_w, nit = (Wf + kDgT - 1) / kDgT;
  for (int c = 0; c < ch.n; ++c) {
    const int a = ch.off[c], n = ch.size(c);
    if (n == 0) continue;
    k_gather_images<<<blocks_for(2 * n * img), 256, 0, s>>>(d_images, left + a, right + a, n, img,
                                                            t.images + 2 * a * img);
    OVN_LAUNCH_CHECK(h);
  }
  // leg forward
  float* act[kMaxLegLayers];
  {
    float* y = t.acts;
    const float* x = t.images;
    prof_mark(h, PROF_LEG, s);
    for (int l = 0; l < h->n_leg; ++l) {
      const ConvSpec& L = h->leg[l];
      act[l] = y;
      BOperand b{h->d_w[l], nullptr, nullptr, 0, 0};
      const int per = images_per_launch((int64_t)L.h_out * L.w_out);
      for (int i0 = 0; i0 < n2; i0 += per) {
        const int ni = n2 - i0 < per ? n2 - i0 : per;
        ConvOperand a{x + (int64_t)i0 * L.h_in * L.w_in * L.cin, L.h_in, L.w_in, L.cin, L.kw, L.sh, L.sw, L.h_out,
                      L.w_out};
        rc = launch_gemm(h, a, b, h->d_b[l], y + (int64_t)i0 * L.h_out * L.w_out * L.cout, ni * L.h_out * L.w_out,
                         L.cout, L.kh * L.kw * L.cin, 1, L.relu, s);
        if (rc != OVN_OK) return rc;
      }
      x = y;
      y += (int64_t)n2 * L.h_out * L.w_out * L.cout;
    }
    prof_mark(h, PROF_LEG, s);
  }
  const float* fv = act[h->n_leg - 1];
  t.net_fv_off = fv - t.acts.get();
  t.net_np = np;
  if (ch.n == 1) k_pair_rows<<<blocks_for(n2), 256, 0, s>>>(t.pair_rows, n2);
  else k_chunk_pair_rows<<<blocks_for(np), 256, 0, s>>>(t.pair_rows, np, ch);
  OVN_LAUNCH_CHECK(h);
  const int32_t* lrow = t.pair_rows;
  const int32_t* rrow = t.pair_rows + np;
  // both heads forward, losses, overlap-head backward: do1 = dL/d(c_conv1 output) is left in h->d_o1
  rc = head_gradients_fp32(h, fv, lrow, rrow, np, d_gt_overlap, d_gt_orientation, min_overlap, ch, s);
  if (rc != OVN_OK || t.stopped) return rc;
  // dL/d(volumes) = correlation-head part + |l - r| part
  float* dfv = t.dact[0];
  for (int c = 0; c < ch.n; ++c) {            // the orientation loss's 1 / (n Wf) is the chunk's
    const int a = ch.off[c], n = ch.size(c);
    if (n == 0) continue;
    k_corr_dlogit<<<blocks_for((int64_t)n * Wf), 256, 0, s>>>(t.corr + (int64_t)a * Wf, d_gt_overlap + a,
                                                               d_gt_orientation + a, n, Wf, min_overlap,
                                                               t.dcorr + (int64_t)a * Wf);
    OVN_LAUNCH_CHECK(h);
  }
  k_corr_backward<<<dim3((Wf + kCorrRows - 1) / kCorrRows, np, 2), kFeatC, Wf * sizeof(float), s>>>(
      t.dcorr, fv, lrow, rrow, np, Wf, dfv);
  OVN_LAUNCH_CHECK(h);
  if (train_stop_here(t, OVN_TRAIN_STAGE_DFV_CORR, 0, dfv)) return OVN_OK;
  float* part_l = t.dfv_part;
  float* part_r = part_l + (int64_t)np * nb * vol;
  const dim3 dg_grid(kFeatC / kDgT, nit, nb * np);
  if (h->train_tc) {
    if (!h->dgrad_tc_smem) {
      OVN_CUDA(h, cudaFuncSetAttribute(k_delta_dgrad_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, kDgTcSmem));
      h->dgrad_tc_smem = true;
    }
    k_delta_dgrad_tc<<<dg_grid, 256, kDgTcSmem, s>>>(h->d_o1, h->d_w[kMaxLegLayers], fv, lrow, rrow, Wf, sz, nb,
                                                     h->head[1].h_out, part_l, part_r);
  } else {
    k_delta_dgrad<<<dg_grid, 256, 0, s>>>(h->d_o1, h->d_w[kMaxLegLayers], fv, lrow, rrow, Wf, sz, nb,
                                          h->head[1].h_out, part_l, part_r);
  }
  OVN_LAUNCH_CHECK(h);
  k_delta_dgrad_reduce<<<blocks_for(n2 * vol), 256, 0, s>>>(part_l, part_r, np, nb, nit, vol, dfv);
  OVN_LAUNCH_CHECK(h);
  if (d_fv_grad) OVN_CUDA(h, cudaMemcpyAsync(d_fv_grad, dfv, (size_t)(n2 * vol) * sizeof(float),
                                             cudaMemcpyDeviceToDevice, s));
  // leg backward: dy = dL/d(pre-activation of layer l), then its weight + bias gradient and its input gradient
  float* dy = dfv;
  float* dx = t.dact[1];
  if (ch.n > 1) {                             // into the images' order: chunk after chunk, LEFT then RIGHT
    for (int c = 0; c < ch.n; ++c) {
      const int64_t a = ch.off[c], n = ch.size(c);
      if (n == 0) continue;
      OVN_CUDA(h, cudaMemcpyAsync(dx + 2 * a * vol, dfv + a * vol, (size_t)(n * vol) * sizeof(float),
                                  cudaMemcpyDeviceToDevice, s));
      OVN_CUDA(h, cudaMemcpyAsync(dx + (2 * a + n) * vol, dfv + (np + a) * vol, (size_t)(n * vol) * sizeof(float),
                                  cudaMemcpyDeviceToDevice, s));
    }
    dy = dx;
    dx = dfv;
  }
  k_relu_grad<<<blocks_for(n2 * vol), 256, 0, s>>>(dy, fv, n2 * vol);
  OVN_LAUNCH_CHECK(h);
  for (int l = h->n_leg - 1; l >= 0; --l) {
    if (train_stop_here(t, OVN_TRAIN_STAGE_LEG_DY, l, dy)) return OVN_OK;
    const ConvSpec& L = h->leg[l];
    const float* X = l ? act[l - 1] : t.images;
    const int Kc = L.kh * L.kw * L.cin;
    const int64_t in_img = (int64_t)L.h_in * L.w_in * L.cin, out_img = (int64_t)L.h_out * L.w_out * L.cout;
    for (int c = 0; c < ch.n; ++c) {
      const int64_t a = ch.off[c];
      const int n = ch.size(c);
      if (n == 0) continue;
      ConvWgradOperand op{X + 2 * a * in_img, L.h_in, L.w_in, L.cin, L.kw, L.sh, L.sw, L.h_out, L.w_out, Kc};
      rc = wgrad_gemm(h, op, dy + 2 * a * out_img, Kc, L.cout, 2 * n * L.h_out * L.w_out,
                      ch.grad + c * ch.stride + h->params.off[l], s);
      if (rc != OVN_OK) return rc;
    }
    if (l == 0) break;
    k_swap_io<<<blocks_for(h->params.n_kernel[l]), 256, 0, s>>>(h->d_w[l], t.wt, L.kh * L.kw, L.cin, L.cout);
    OVN_LAUNCH_CHECK(h);
    BOperand b{t.wt, nullptr, nullptr, 0, 0};
    const int64_t rows_in = (int64_t)L.h_in * L.w_in, K = L.kh * L.kw * L.cout;
    const int per = images_per_launch(rows_in);
    for (int i0 = 0; i0 < n2 && rc == OVN_OK; i0 += per) {
      const int ni = n2 - i0 < per ? n2 - i0 : per;
      const float* dyi = dy + (int64_t)i0 * L.h_out * L.w_out * L.cout;
      float* dxi = dx + (int64_t)i0 * rows_in * L.cin;
      if (L.sh == 1 && L.sw == 1) {
        ConvDgradOperand d{dyi, L.h_out, L.w_out, L.cout, L.kw, L.h_in, L.w_in};
        rc = launch_gemm(h, d, b, nullptr, dxi, (int)(ni * rows_in), L.cin, (int)K, 1, 0, s);
      } else {
        ConvDgradStridedOperand d{dyi, L.h_out, L.w_out, L.cout, L.kw, L.h_in, L.w_in, L.sh, L.sw};
        rc = launch_gemm(h, d, b, nullptr, dxi, (int)(ni * rows_in), L.cin, (int)K, 1, 0, s);
      }
    }
    if (rc != OVN_OK) return rc;
    const int64_t nx = n2 * rows_in * L.cin;
    k_relu_grad<<<blocks_for(nx), 256, 0, s>>>(dx, X, nx);
    OVN_LAUNCH_CHECK(h);
    float* tmp = dy;
    dy = dx;
    dx = tmp;
  }
  return OVN_OK;
}

// ---- data-parallel training -------------------------------------------------------------------------

// The volumes of the last ovn_net_gradients batch, [2][np][Wf][128] (LEFT, then RIGHT): the leg's output as that
// call computed it, at its training precision (the backward reads every activation, and none is overwritten)
int copy_net_volumes_fp32(ovn_handle* h, float* d_out, cudaStream_t s) {
  const TrainState& t = *h->train;
  const size_t n = (size_t)2 * t.net_np * h->cfg.leg_output_width * kFeatC;
  OVN_CUDA(h, cudaMemcpyAsync(d_out, t.acts + t.net_fv_off, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return OVN_OK;
}

// ---- stages of the last gradient call (ovn_copy_train_stage) ----------------------------------------------
// Where a stage lives and how many floats it has, for the np pairs of the last call: *src = null for a stop stage,
// whose buffer the call recorded when it stopped
static int64_t train_stage_at(const ovn_handle* h, int stage, int layer, const float** src) {
  const TrainState& t = *h->train;
  const int64_t np = t.stage_np, n2 = 2 * np, Wf = h->cfg.leg_output_width, vol = Wf * kFeatC;
  const int64_t nb = h->o1_w, nit = (Wf + kDgT - 1) / kDgT;
  const ConvSpec& L2 = h->head[1];
  const ConvSpec& L3 = h->head[2];
  const int64_t o1_pair = (int64_t)L2.h_in * L2.w_in * L2.cin, x3_pair = (int64_t)L3.h_in * L3.w_in * L3.cin;
  auto leg_out = [&](int l) { const ConvSpec& L = h->leg[l]; return n2 * L.h_out * L.w_out * L.cout; };
  *src = nullptr;
  switch (stage) {
    case OVN_TRAIN_STAGE_O1: return np * o1_pair;
    case OVN_TRAIN_STAGE_X4: return np * h->dense_in;
    case OVN_TRAIN_STAGE_DFV_CORR: return n2 * vol;
    case OVN_TRAIN_STAGE_LEG_DY: return leg_out(layer);
    case OVN_TRAIN_STAGE_X3: *src = h->d_o2; return np * x3_pair;
    case OVN_TRAIN_STAGE_OVERLAP: *src = t.overlap; return np;
    case OVN_TRAIN_STAGE_CORR: *src = t.corr; return np * Wf;
    case OVN_TRAIN_STAGE_DZ: *src = t.dz; return np;
    case OVN_TRAIN_STAGE_DPRE3: *src = t.x4; return np * h->dense_in;
    case OVN_TRAIN_STAGE_DX3: *src = t.dx3; return np * x3_pair;
    case OVN_TRAIN_STAGE_DO1: *src = h->d_o1; return np * o1_pair;
    case OVN_TRAIN_STAGE_DCORR: *src = t.dcorr; return np * Wf;
    case OVN_TRAIN_STAGE_PART_L: *src = t.dfv_part; return np * nb * vol;
    case OVN_TRAIN_STAGE_PART_R: *src = t.dfv_part + np * nb * vol; return np * nit * vol;
    case OVN_TRAIN_STAGE_IMAGES: *src = t.images; return n2 * h->cfg.proj_H * h->cfg.proj_W * h->C;
    case OVN_TRAIN_STAGE_ACT: {
      int64_t off = 0;
      for (int l = 0; l < layer; ++l) off += leg_out(l);
      *src = t.acts + off;
      return leg_out(layer);
    }
  }
  return 0;
}

int64_t train_stage_floats(const ovn_handle* h, int stage, int layer) {
  const float* src;
  return train_stage_at(h, stage, layer, &src);
}

int copy_train_stage_fp32(ovn_handle* h, int stage, int layer, float* d_out, cudaStream_t s) {
  const float* src;
  const int64_t n = train_stage_at(h, stage, layer, &src);
  if (!src) src = h->train->stop_buf;
  OVN_CUDA(h, cudaMemcpyAsync(d_out, src, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return OVN_OK;
}

// One weight tensor's run of the flat vector: elements [start, next segment's start) update w[i - start] and
// a[i - start]
struct SumSegment {
  int64_t start;
  float* w;
  float* a;
};
constexpr int kMaxSumSegments = 2 * (kMaxLegLayers + 4);
struct SumArgs {
  SumSegment seg[kMaxSumSegments];   // in flat order
  int64_t n;                         // floats per part
  int n_seg;
  int n_parts;                       // the parts with a nonzero weight, in part order
  int part[kMaxSumParts];
  float weight[kMaxSumParts];
};

// g = w0 p0 + w1 p1 + ... in part order, every product and sum rounded on its own, then Adagrad as Keras 2.1.5
// does it: a += g^2 as one FMA;  w -= lr * g / (sqrt(a) + 1e-7) with IEEE sqrt and division.  The table is read
// through the constant bank (__grid_constant__), so the segment search does not copy it to local memory.
__global__ void k_adagrad_sum(const float* __restrict__ parts, const __grid_constant__ SumArgs p, float lr) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n) return;
  float g = 0.f;
  for (int k = 0; k < p.n_parts; ++k) {
    const float v = __fmul_rn(p.weight[k], parts[(int64_t)p.part[k] * p.n + i]);
    g = k ? __fadd_rn(g, v) : v;
  }
  int s = 0;
  while (s + 1 < p.n_seg && i >= p.seg[s + 1].start) ++s;
  const int64_t j = i - p.seg[s].start;
  float* w = p.seg[s].w;
  float* a = p.seg[s].a;
  const float ai = __fmaf_rn(g, g, a[j]);
  a[j] = ai;
  w[j] = __fsub_rn(w[j], __fdiv_rn(__fmul_rn(lr, g), __fadd_rn(__fsqrt_rn(ai), 1e-7f)));
}

int adagrad_sum_fp32(ovn_handle* h, bool whole_network, const float* d_parts, int n_parts, const float* h_weights,
                     float lr, cudaStream_t s) {
  const ParamLayout& L = h->params;
  float* accum = h->train->accum;
  SumArgs p = {};
  const int n_layers = whole_network ? 4 + h->n_leg : 4;
  for (int i = 0; i < n_layers; ++i) {
    const int slot = flat_slot(i);
    const int64_t o = L.off[slot], ob = o + L.n_kernel[slot];
    p.seg[2 * i] = {o, h->d_w[slot], accum + o};
    p.seg[2 * i + 1] = {ob, h->d_b[slot], accum + ob};
  }
  p.n_seg = 2 * n_layers;
  p.n = whole_network ? L.n_total : L.n_head;
  for (int r = 0; r < n_parts; ++r) {
    if (h_weights[r] == 0.f) continue;
    p.part[p.n_parts] = r;
    p.weight[p.n_parts++] = h_weights[r];
  }
  k_adagrad_sum<<<blocks_for(p.n), 256, 0, s>>>(d_parts, p, lr);
  OVN_LAUNCH_CHECK(h);
  return OVN_OK;
}

}  // namespace ovn
