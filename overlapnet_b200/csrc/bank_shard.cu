// bank_shard.cu -- k_gather_rows: a step's rows of a training image bank sharded over the GPUs of a node,
// copied into one device slot straight from the owners' memory (ovn_gather_rows, DESIGN.md section 6).
#include "common.cuh"
#include <algorithm>

namespace ovn {

// The source of every row of one launch, by value in the kernel's parameters (sm_90 takes up to 32 764 bytes
// there): nothing the caller may reuse after the call returns, and nothing two calls in flight share.
struct GatherRowsSrc {
  const uint4* row[kGatherRowsCap];
};

constexpr int kGatherThreads = 256;
constexpr int kGatherUnroll = 4;        // 16-byte words in flight per thread

// Block (x, y) copies the x-th run of kGatherThreads * kGatherUnroll words of row y; all loads of a thread are
// issued before its stores.
static __global__ void __launch_bounds__(kGatherThreads)
k_gather_rows(const GatherRowsSrc src, int64_t words, uint4* __restrict__ dst) {
  const uint4* __restrict__ s = src.row[blockIdx.y];
  uint4* __restrict__ d = dst + (int64_t)blockIdx.y * words;
  const int64_t stride = (int64_t)gridDim.x * kGatherThreads * kGatherUnroll;
  for (int64_t w0 = (int64_t)blockIdx.x * kGatherThreads * kGatherUnroll + threadIdx.x; w0 < words; w0 += stride) {
    uint4 v[kGatherUnroll];
#pragma unroll
    for (int u = 0; u < kGatherUnroll; ++u) {
      const int64_t w = w0 + (int64_t)u * kGatherThreads;
      if (w < words) v[u] = s[w];
    }
#pragma unroll
    for (int u = 0; u < kGatherUnroll; ++u) {
      const int64_t w = w0 + (int64_t)u * kGatherThreads;
      if (w < words) d[w] = v[u];
    }
  }
}

int gather_rows(ovn_handle* h, const void* const* h_src, int n, int64_t row_bytes, void* d_dst, cudaStream_t s) {
  const int64_t words = row_bytes / 16;
  const int64_t per_block = (int64_t)kGatherThreads * kGatherUnroll;
  const unsigned gx = (unsigned)std::min<int64_t>((words + per_block - 1) / per_block, 1 << 16);
  GatherRowsSrc src;
  for (int i0 = 0; i0 < n; i0 += kGatherRowsCap) {
    const int m = std::min(n - i0, kGatherRowsCap);
    for (int i = 0; i < m; ++i) src.row[i] = static_cast<const uint4*>(h_src[i0 + i]);
    prof_mark(h, PROF_GATHER_ROWS, s);
    k_gather_rows<<<dim3(gx, m), kGatherThreads, 0, s>>>(src, words, static_cast<uint4*>(d_dst) + i0 * words);
    OVN_LAUNCH_CHECK(h);
    prof_mark(h, PROF_GATHER_ROWS, s);
  }
  return OVN_OK;
}

}  // namespace ovn
