// Shared device helpers for the sbi_b200 kernels (sm_90a).
//
//  * mbarrier + cp.async.bulk (TMA bulk copy, SASS UBLKCP) wrappers used by the
//    warp-specialised weight pipeline: one producer warp streams weight chunks from
//    L2/HBM into a shared-memory ring while 8 consumer warps run the tile math.
//  * small math helpers restating the exact PyTorch definitions the reference uses
//    (softplus threshold 20, sigmoid, relu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#ifndef SBI_PRODUCER_SLEEP_NS
#define SBI_PRODUCER_SLEEP_NS 20
#endif

namespace sbi {

constexpr int kConsumerThreads = 256;   // 8 consumer warps
constexpr int kProducerThreads = 32;    // 1 producer warp (one elected lane works)
constexpr int kThreads = kConsumerThreads + kProducerThreads;

__host__ __device__ constexpr int round4(int x) { return (x + 3) & ~3; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
  }
}
// producer-side wait: back off between probes so the spinning lane does not eat issue slots
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  uint32_t ok = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
    if (ok) break;
    __nanosleep(SBI_PRODUCER_SLEEP_NS);
  }
}
// TMA bulk copy global -> shared, completion signalled on an mbarrier (complete_tx).
// bytes must be a multiple of 16; both addresses 16-byte aligned.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// named barrier for the consumer warps only (the producer warp never joins it)
__device__ __forceinline__ void consumer_sync() {
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
}

// ---- weight pipeline -------------------------------------------------------------
// Ring of NBUF shared-memory buffers of `cap` floats.  Chunk i lives in slot i % NBUF.
// full[s]  : producer arrive.expect_tx + TMA complete_tx   (count 1)
// empty[s] : one arrive per consumer warp after its last read (count 8)
struct WPipe {
  float* buf;        // NBUF * cap floats, 128B aligned
  uint64_t* full;    // NBUF
  uint64_t* empty;   // NBUF
  int cap;           // floats per slot
  int nbuf;
  uint32_t it;       // chunk counter (same sequence on producer and consumers)

  __device__ __forceinline__ int slot() const { return it % nbuf; }
  __device__ __forceinline__ uint32_t phase() const { return (it / nbuf) & 1u; }

  // producer (single elected thread): up to two source ranges into one slot
  __device__ __forceinline__ void produce(const float* src0, int n0, const float* src1 = nullptr,
                                          int n1 = 0) {
    int s = slot();
    mbar_wait_backoff(&empty[s], phase() ^ 1u);
    float* dst = buf + (size_t)s * cap;
    mbar_arrive_expect_tx(&full[s], (uint32_t)(n0 + n1) * 4u);
    bulk_g2s(dst, src0, (uint32_t)n0 * 4u, &full[s]);
    if (n1 > 0) bulk_g2s(dst + n0, src1, (uint32_t)n1 * 4u, &full[s]);
    ++it;
  }
  // consumers: wait for the current chunk, get its base
  __device__ __forceinline__ const float* acquire() {
    int s = slot();
    mbar_wait(&full[s], phase());
    return buf + (size_t)s * cap;
  }
  // consumers: all lanes of a warp done reading -> lane 0 arrives
  __device__ __forceinline__ void release() {
    int s = slot();
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[s]);
    ++it;
  }
};

// ---- math ----------------------------------------------------------------------
__device__ __forceinline__ float relu_f(float x) { return x > 0.f ? x : 0.f; }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }
// torch.nn.functional.softplus(beta=1, threshold=20)
__device__ __forceinline__ float softplus_f(float x) { return x > 20.f ? x : log1pf(expf(x)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// dst (+)= v on a partial-gradient slab owned by this CTA.  The accumulate form is a fire-and-forget RED: no load, no
// scoreboard wait (the read-modify-write of the slab was the top stall of the SIMT VJP kernels: 300+ dependent L2
// round trips per thread and tile).  Every address is written by ONE thread, first with a plain store, then with
// REDs in tile order, so the sum order is fixed and nothing ever reads the slab inside the kernel (an L1-cached
// load could not see the REDs).
__device__ __forceinline__ void grad_out(float* dst, float v, bool accumulate) {
  if (accumulate) asm volatile("red.global.add.f32 [%0], %1;" ::"l"(dst), "f"(v) : "memory");
  else *dst = v;
}

}  // namespace sbi
