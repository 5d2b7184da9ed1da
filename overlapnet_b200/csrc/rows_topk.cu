// rows_topk.cu -- k_rows_topk: the best k <= 32 records (overlap, index, yaw) of each row of an overlap / yaw matrix,
// each row with its own length (ovn_rows_topk, ovn_heads_prefix_topk, DESIGN.md section 4).
//
// A record's rank is one unique 64-bit key: the overlap mapped to an unsigned order in the high word (NaN above
// +inf, -0 equal to +0) and the inverted index in the low word, so that equal overlaps rank by index, ascending.
// Every key of a row is distinct, so the best k keys are one set whatever order the merge visits them in: the
// result is deterministic by construction, with no atomics.  Key 0 is below every real key and marks "none".
#include "common.cuh"
#include <algorithm>

namespace ovn {

constexpr int kTopkThreads = 128;

static __device__ __forceinline__ unsigned long long topk_key(float v, int idx) {
  uint32_t u = __float_as_uint(v);
  uint32_t o;
  if (v != v) o = 0xffffffffu;                         // NaN: above every number, whatever its sign bit
  else if (v == 0.0f) o = 0x80000000u;                 // -0 ranks as +0
  else o = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)o << 32) | (uint32_t)~(uint32_t)idx;
}

// Block b reduces row b: element j of the row is at row_off[b] + j, j < row_len[b].  Each thread keeps the best
// kTopkMax keys of a strided pass in registers, sorted descending; a tree of pairwise merges in shared memory
// leaves the row's best keys in thread 0's list.
static __global__ void __launch_bounds__(kTopkThreads)
k_rows_topk(const float* __restrict__ ov, const int32_t* __restrict__ yaw, const int64_t* __restrict__ row_off,
            const int32_t* __restrict__ row_len, int k, float* __restrict__ top_ov, int32_t* __restrict__ top_idx,
            int32_t* __restrict__ top_yaw) {
  __shared__ unsigned long long lists[kTopkThreads][kTopkMax + 1];   // +1: no bank conflicts on the column walk
  const int row = blockIdx.x;
  const int64_t off = row_off[row];
  const int n = row_len[row];
  unsigned long long best[kTopkMax];
#pragma unroll
  for (int j = 0; j < kTopkMax; ++j) best[j] = 0ull;
  for (int i = threadIdx.x; i < n; i += kTopkThreads) {
    unsigned long long x = topk_key(ov[off + i], i);
    if (x > best[kTopkMax - 1]) {
#pragma unroll
      for (int j = 0; j < kTopkMax; ++j) {                // insertion into the sorted registers
        const unsigned long long hi = best[j] > x ? best[j] : x;
        x = best[j] > x ? x : best[j];
        best[j] = hi;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < kTopkMax; ++j) lists[threadIdx.x][j] = best[j];
  __syncthreads();
  for (int s = kTopkThreads / 2; s >= 1; s >>= 1) {
    if (threadIdx.x < s) {
      const unsigned long long* a = lists[threadIdx.x];
      const unsigned long long* b = lists[threadIdx.x + s];
      int ia = 0, ib = 0;
#pragma unroll
      for (int j = 0; j < kTopkMax; ++j) {                // the best kTopkMax of two sorted lists
        const unsigned long long ka = ia < kTopkMax ? a[ia] : 0ull;
        const unsigned long long kb = ib < kTopkMax ? b[ib] : 0ull;
        const bool take_a = ka > kb;
        best[j] = take_a ? ka : kb;
        ia += take_a;
        ib += !take_a;
      }
#pragma unroll
      for (int j = 0; j < kTopkMax; ++j) lists[threadIdx.x][j] = best[j];   // only this thread reads list t
    }
    __syncthreads();
  }
  if (threadIdx.x < k) {
    const unsigned long long key = lists[0][threadIdx.x];
    const int64_t o = (int64_t)row * k + threadIdx.x;
    if (key == 0ull) {
      top_ov[o] = -1.0f;
      top_idx[o] = -1;
      top_yaw[o] = 0;
    } else {
      const int idx = (int)~(uint32_t)(key & 0xffffffffull);
      top_ov[o] = ov[off + idx];
      top_idx[o] = idx;
      top_yaw[o] = yaw[off + idx];
    }
  }
}

int rows_topk(ovn_handle* h, const float* d_ov, const int32_t* d_yaw, const int64_t* h_off, const int32_t* h_len,
              int64_t rows, int k, float* d_top_ov, int32_t* d_top_idx, int32_t* d_top_yaw, cudaStream_t s) {
  if (rows <= 0) return OVN_OK;
  const int64_t cap = kTopkRowsPerLaunch;
  int rc = h->d_topk_rows.ensure(h, (size_t)std::min(rows, cap) * (sizeof(int64_t) + sizeof(int32_t)));
  if (rc != OVN_OK) return rc;
  int64_t* d_off = reinterpret_cast<int64_t*>(h->d_topk_rows.get());
  int32_t* d_len = reinterpret_cast<int32_t*>(d_off + std::min(rows, cap));
  for (int64_t r0 = 0; r0 < rows; r0 += cap) {
    const int64_t m = std::min(rows - r0, cap);
    // pageable sources: the copies return once the host arrays are staged, and run in stream order, after the
    // launches of earlier chunks that read the same metadata
    OVN_CUDA(h, cudaMemcpyAsync(d_off, h_off + r0, m * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    OVN_CUDA(h, cudaMemcpyAsync(d_len, h_len + r0, m * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    prof_mark(h, PROF_ROWS_TOPK, s);
    k_rows_topk<<<(unsigned)m, kTopkThreads, 0, s>>>(d_ov, d_yaw, d_off, d_len, k, d_top_ov + r0 * k,
                                                     d_top_idx + r0 * k, d_top_yaw + r0 * k);
    OVN_LAUNCH_CHECK(h);
    prof_mark(h, PROF_ROWS_TOPK, s);
  }
  return OVN_OK;
}

}  // namespace ovn
