// hopper.cuh -- hand-written PTX wrappers for the Hopper (sm_90a) building blocks used by network_tc.cu:
// wgmma (warpgroup MMA; B from shared memory, A from registers or shared memory), mbarrier and the pipeline
// ring built on it, cp.async.bulk (TMA engine, 1-D, both directions).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace hopper {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier -------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}\n" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}\n"
               :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline that never completes raises an error instead of hanging.  False on time-out.
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, long long max_cycles) {
  if (mbar_try_wait(bar, parity)) return true;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > max_cycles) return false;
  return true;
}
constexpr long long kMbarWaitCycles = 1ll << 28;

// A ring of D pipeline stages, each guarded by a full / empty mbarrier pair.  The producer fills the stages in
// order; fill i uses stage i % D in phase (i / D) & 1.  The fill counters belong to the kernels, which pass the
// fill index.  full[s] completes on the producer's arrive plus the bytes of its bulk copies; empty[s] completes
// when every consumer arrival has released the stage.
//
// A ring can also be filled by threads rather than by bulk copies: init with one producer arrival per writing
// warp; each writing warp waits with wait_free, writes, and signals the fill with publish.
template <int D>
struct MbarRing {
  uint64_t full[D], empty[D];
  __device__ __forceinline__ void init(uint32_t consumer_arrivals, uint32_t producer_arrivals = 1) {
    for (int s = 0; s < D; ++s) { mbar_init(&full[s], producer_arrivals); mbar_init(&empty[s], consumer_arrivals); }
  }
  static __device__ __forceinline__ uint32_t slot(uint32_t i) { return i % D; }
  static __device__ __forceinline__ uint32_t parity(uint32_t i) { return (i / D) & 1; }
  // producer: wait (bounded) until fill i's stage is free, then expect `bytes` on it.  False on time-out.
  __device__ __forceinline__ bool acquire(uint32_t i, uint32_t bytes) {
    if (!mbar_wait(&empty[slot(i)], parity(i) ^ 1, kMbarWaitCycles)) return false;
    mbar_arrive_expect_tx(&full[slot(i)], bytes);
    return true;
  }
  // producer, without waiting: false if fill i's stage is not free yet
  __device__ __forceinline__ bool try_acquire(uint32_t i, uint32_t bytes) {
    if (!mbar_try_wait(&empty[slot(i)], parity(i) ^ 1)) return false;
    mbar_arrive_expect_tx(&full[slot(i)], bytes);
    return true;
  }
  // the barrier the bulk copies of fill i complete on
  __device__ __forceinline__ uint64_t* bar(uint32_t i) { return &full[slot(i)]; }
  // consumer: wait (bounded) until fill i has landed.  False on time-out.
  __device__ __forceinline__ bool wait(uint32_t i) { return mbar_wait(&full[slot(i)], parity(i), kMbarWaitCycles); }
  // consumer: this warp is done with fill i's stage (one arrival per warp)
  __device__ __forceinline__ void release(uint32_t i) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[slot(i)]);
  }
  // consumer that is a single thread: it is done with fill i's stage
  __device__ __forceinline__ void release_thread(uint32_t i) { mbar_arrive(&empty[slot(i)]); }
  // writing warp: wait (bounded) until fill i's stage is free.  False on time-out.
  __device__ __forceinline__ bool wait_free(uint32_t i) {
    return mbar_wait(&empty[slot(i)], parity(i) ^ 1, kMbarWaitCycles);
  }
  // writing warp: this warp has written its part of fill i (one arrival per warp).  Writes that a bulk copy will
  // read must be followed by fence_proxy_async_smem() in each writing thread first.
  __device__ __forceinline__ void publish(uint32_t i) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&full[slot(i)]);
  }
};

// The bounded waits of a kernel with an `int* err` flag and a `done:` label before its end; `ok` is a ring's
// acquire or wait, `code` an ovn::DeviceError.
// A producer, or a consumer with no wgmma groups in flight: on time-out raise `code` and leave the kernel.
#define PIPE_WAIT(ok, code) \
  if (!(ok)) { atomicExch(err, (code)); goto done; }
// A consumer with wgmma groups in flight: leaving the loop there would make the compiler wait for them on a
// divergent path, which serialises every wgmma of the kernel.  A time-out raises `code` and sets the local
// `failed`; later waits are skipped, and the consumer leaves (`if (failed) goto done`) once its groups retire.
#define INFLIGHT_WAIT(ok, code) \
  if (!failed && !(ok)) { atomicExch(err, (code)); failed = true; }

// barrier `id` (1..15) among the `count` threads (a multiple of 32) that reach it, e.g. one warpgroup
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(count) : "memory");
}

// ---- per-warpgroup register budget: every warp of a warpgroup executes the same call.  A producer warpgroup
// gives registers back (dec) so that the consumer warpgroups can take them (inc blocks until they are free).
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" :: "n"(N)); }
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" :: "n"(N)); }

// ---- bulk async copy global -> shared, completes on an mbarrier (bytes and addresses multiples of 16)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---- bulk async copy shared -> global, tracked by bulk async-groups (bytes and addresses multiples of 16)
__device__ __forceinline__ void bulk_s2g(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               :: "l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's committed groups still read their shared-memory sources (which may then be rewritten)
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory"); }
// at most N of this thread's committed groups are still incomplete (their global writes not yet performed)
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" :: "n"(N) : "memory"); }
// orders this thread's earlier shared-memory writes before later bulk copies (async proxy) that read them
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma ------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor of a K-major operand (16-bit types):
//   bits [0,14) start >> 4, [16,30) LBO >> 4, [32,46) SBO >> 4, [62,64) layout
// kNoSwizzle: 8 x 16-byte core matrices, 16-byte aligned,
//   element (row r, k) at start + (r / 8) * SBO + (r % 8) * 16 + (k / 8) * LBO + (k % 8) * 2
// kSwizzle128B: rows of 128 bytes (64 K values) whose 16-byte chunk c is stored at c ^ (r % 8), 8-row atoms of
//   1024 bytes (SBO = 1024, LBO unused), tile on a 1024-byte boundary; the K16 step k of a 64-wide tile starts
//   at tile + 32 k bytes (the hardware applies the XOR to the final address).
constexpr uint32_t kNoSwizzle = 0, kSwizzle128B = 1;
__device__ __forceinline__ uint64_t desc_kmajor(uint32_t smem_addr, uint32_t lbo, uint32_t sbo, uint32_t layout) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3FFF) << 32) | ((uint64_t)layout << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }

// D[64 x 64] (fp32, registers) += A[64 x 16] (fp16, registers: the mma.m16n8k16 A fragment of each warp's
// 16 rows) * B[16 x 64] (fp16, shared memory, K-major).  Executed by all 128 threads of a warpgroup.
// D fragment: d[4 j + {0, 1}] = (row 16 w + g, col 8 j + 2 t + {0, 1}), d[4 j + {2, 3}] = row + 8.
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1)
      : "memory");
}

// D[64 x 128] (fp32, registers) += A[64 x 16] * B[16 x 128], both fp16 K-major in shared memory.  Executed by all
// 128 threads of a warpgroup.  D fragment: d[4 j + {0, 1}] = (row 16 w + g, col 8 j + 2 t + {0, 1}),
// d[4 j + {2, 3}] = row + 8, j < 16.
__device__ __forceinline__ void wgmma_m64n128k16_ss(float (&d)[64], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(1)
      : "memory");
}

}  // namespace hopper
