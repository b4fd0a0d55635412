// Shared device-side primitives for the sm_90a kernels of gen3c_b200:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (fences / groups / shared-memory descriptors).
// Raw PTX only; no CUTLASS dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/gen3c_b200.h"
#include "wgmma_ops.cuh"

namespace g3c {

// ----------------------------------------------------------------------------------------------
// error plumbing (host)
// ----------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);
#define G3C_CUDA(x)                                                         \
  do {                                                                      \
    cudaError_t _e = (x);                                                   \
    if (_e != cudaSuccess) return ::g3c::cuda_fail(_e, #x, __FILE__, __LINE__); \
  } while (0)
#define G3C_REQUIRE(cond, ...)        \
  do {                                \
    if (!(cond)) {                    \
      ::g3c::set_error(__VA_ARGS__);  \
      return G3C_EINVAL;       \
    }                                 \
  } while (0)

// Host: encode a tiled TMA descriptor (128-byte swizzle) of bf16 elements, or of `dtype` (UINT8 for e4m3 codes).
// dims/strides innermost first, rank 2 or 3.  strides_bytes has rank-1 entries (stride of dim 1.., dim 0 is contiguous).
int make_tmap_bf16_sw128(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes, const uint32_t* box,
                         CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
// Same for a 2-D fp32 tensor (box inner extent 32 floats = one 128-byte swizzle span).
int make_tmap_f32_sw128(CUtensorMap* out, const void* base, const uint64_t* dims,
                        const uint64_t* strides_bytes, const uint32_t* box);

int sm_count();

#ifdef __CUDACC__
// ----------------------------------------------------------------------------------------------
// small helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ uint32_t warp_id() { return __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
// G3C_MBAR_SUSPEND_NS: suspend-time hint of mbarrier.try_wait — the thread may sleep that long before the instruction
// returns false (it still wakes as soon as the phase completes), so a waiting warp re-issues the poll loop less often.
// Off by default.
#ifndef G3C_MBAR_SUSPEND_NS
#define G3C_MBAR_SUSPEND_NS 0
#endif
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
#if G3C_MBAR_SUSPEND_NS > 0
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"((uint32_t)G3C_MBAR_SUSPEND_NS)
      : "memory");
#else
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
#endif
  return ok != 0;
}
// non-blocking phase test (no suspend): true once the phase with this parity has completed
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin with a generous bound so that a protocol bug traps instead of hanging the GPU.
#ifndef G3C_MBAR_TIMEOUT_NS
#define G3C_MBAR_TIMEOUT_NS 4000000000ull
#endif
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;\n" : "=l"(t));
  return t;
}
// A protocol bug must trap instead of hanging the GPU.  No function call / printf here: a call inside a
// setmaxnreg region forces ptxas to size the whole kernel for the smallest register budget.
#ifdef G3C_MBAR_DEBUG
#define G3C_MBAR_TIMEOUT_ACTION(bar, parity)                                                                 \
  do {                                                                                                       \
    printf("g3c: mbarrier timeout block(%d,%d) thread %d bar@%u parity %u\n", blockIdx.x, blockIdx.y,        \
           threadIdx.x, bar, parity);                                                                        \
    __trap();                                                                                                \
  } while (0)
#else
#define G3C_MBAR_TIMEOUT_ACTION(bar, parity) asm volatile("trap;\n")
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0xFFFu) == 0) {
      uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > G3C_MBAR_TIMEOUT_NS) G3C_MBAR_TIMEOUT_ACTION(smem_u32(bar), parity);
    }
  }
}

// Same, with a run-time bound: kernels whose progress depends on another PROCESS (context-parallel K/V arrival) pass
// the inter-process timeout so that rank skew of seconds (lazy module load, allocation, host jitter) is waited out.
__device__ __forceinline__ void mbar_wait_ns(uint64_t* bar, uint32_t parity, unsigned long long timeout_ns) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0xFFFu) == 0) {
      uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > timeout_ns) G3C_MBAR_TIMEOUT_ACTION(smem_u32(bar), parity);
    }
  }
}

// Same bound, but on timeout the thread exits instead of trapping.  For warpgroups that raised their budget with
// setmaxnreg.inc: a trap anywhere in such a region makes ptxas allocate it for a smaller budget (the attention consumers
// then spill and serialise their wgmma).  The kernel still traps: a thread outside the region waits (mbar_wait_ns) on a
// barrier that these threads only arrive on when they finish normally.
__device__ __forceinline__ void mbar_wait_ns_or_exit(uint64_t* bar, uint32_t parity, unsigned long long timeout_ns) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0xFFFu) == 0) {
      uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > timeout_ns) asm volatile("exit;\n");
    }
  }
}

// OR of `pred` over the `nthreads` threads (a multiple of 32, every one of them executing this) that meet at named
// barrier `id` (not 0, which __syncthreads uses): all of them get the same result, so a branch on it is uniform over
// their warps, e.g. around a wgmma that all four warps of a warpgroup must issue together.
__device__ __forceinline__ bool bar_red_or(uint32_t id, uint32_t nthreads, bool pred) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred P, Q;\n\t"
      "setp.ne.u32 P, %1, 0;\n\t"
      "bar.red.or.pred Q, %2, %3, P;\n\t"
      "selp.u32 %0, 1, 0, Q;\n\t}\n"
      : "=r"(r)
      : "r"((uint32_t)pred), "r"(id), "r"(nthreads)
      : "memory");
  return r != 0;
}

// Named barrier `id` (not 0, which __syncthreads uses) over `nthreads` threads (a multiple of 32).
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA loads (tile mode, mbarrier completion)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// TMA stores (shared -> global, bulk async-group completion).  `reduce_add` accumulates into global.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.bulk_group [%0, {%2, %3}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
// wait until at most N of this thread's bulk groups still READ their shared-memory source
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;\n" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;\n" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma (Hopper warpgroup MMA): fences, groups, shared-memory descriptors
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory");
}
// The accumulators of an asynchronous wgmma are written behind the compiler's back: pin every register read or written
// around it to this point of the instruction stream (after wgmma_wait, before the next wgmma).
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
// Same for the register A fragments of a wgmma still in flight: keeps them live (their registers are not reused) until here.
template <int N>
__device__ __forceinline__ void fence_regs(uint32_t (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}

// Shared-memory matrix descriptor of a K-major tile stored with the 128-byte swizzle (rows of 64 bf16 = 128 B, 8-row
// groups 1024 B apart, tile base 1024-B aligned): start_address[0,14) = addr>>4, LBO[16,30) (unused for swizzled
// K-major), SBO[32,46) = 1024>>4, layout_type[62,64) = 1 (SWIZZLE_128B).
__device__ __forceinline__ uint64_t make_sdesc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024u >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// Same for an MN-major tile (PTX ISA, "Matrix Descriptor Format"; the B operand of a wgmma with imm-trans-b = 1): each
// 128-byte row holds 64 consecutive MN elements of one k, rows of consecutive k follow each other, so 8 k form one
// 1024-B swizzle atom.  For the swizzled MN-major layouts LBO is the stride between the 64-element MN blocks of the atom
// (`mn_block_bytes`) and SBO the stride between 8-k row groups (1024 B).
__device__ __forceinline__ uint64_t make_sdesc_sw128_mn(uint32_t smem_addr, uint32_t mn_block_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((mn_block_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>(1024u >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// advance along K inside the 128-byte swizzle span: +bytes on the (unswizzled) start address
__device__ __forceinline__ uint64_t sdesc_advance(uint64_t d, uint32_t bytes) {
  return d + static_cast<uint64_t>(bytes >> 4);
}

// Register budget of a warpgroup (all 128 threads execute it): producers give registers back, MMA warpgroups take them.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N));
}

// ----------------------------------------------------------------------------------------------
// numerics helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
#endif  // __CUDACC__

}  // namespace g3c
