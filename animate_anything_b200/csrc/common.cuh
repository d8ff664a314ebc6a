// Shared device helpers for the sm_90a kernels: mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA (wgmma).
// All hand-written inline PTX; the bit layout of the wgmma shared-memory matrix descriptor follows the PTX ISA
// "Asynchronous Warpgroup Level Matrix Multiply-Accumulate" chapter.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <atomic>

#define AAB_OK 0
#define AAB_ERR_ARG 1
#define AAB_ERR_CUDA 2
#define AAB_ERR_DRIVER 3

namespace aab {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "elect.sync _|P1, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P1;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return done != 0;
}
// non-blocking peek
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return done != 0;
}
// Bounded wait: a protocol bug traps (sticky CUDA error) instead of hanging the GPU.  No printf here: a call inside a
// kernel makes ptxas serialise the wgmma pipeline around it.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// fire-and-forget L2 prefetch of a tensor-map box (no shared memory, no barrier)
__device__ __forceinline__ void tma_prefetch_l2_5d(const CUtensorMap* m, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.prefetch.tensor.5d.L2.global.tile [%0, {%1, %2, %3, %4, %5}];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2,
                                             int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (TMA store / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- thread-block clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the copy of `bar` (same shared-memory offset) in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n"
      ".reg .b32 ra;\n"
      "mapa.shared::cluster.u32 ra, %0, %1;\n"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}
// wait that also orders after arrivals released by the other CTAs of the cluster
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  for (;;) {
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) return;
    if (++spins > (1u << 26)) __trap();
  }
}
// TMA load delivered to the same shared-memory offset of every CTA in `cta_mask`; each destination's bytes are credited to
// the barrier at the same offset in that CTA
__device__ __forceinline__ void tma_load_3d_mcast(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                                  uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5, %6}], [%2], %3;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "h"(cta_mask), "r"(c0),
      "r"(c1), "r"(c2)
      : "memory");
}

// ---------------------------------------------------------------- named barriers
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
// Shared-memory matrix descriptor of an operand tile stored as rows of 128 bytes (64 x 16-bit) with the 128-byte swizzle
// that TMA SWIZZLE_128B produces; 8-row groups are 1024 B apart.  Bits: [0,14) addr>>4, [16,30) LBO>>4, [32,46) SBO>>4,
// [62,64) layout (1 = SWIZZLE_128B).  K-major (K contiguous in a row): SBO = 1024, LBO unused; a K step of 16 elements
// advances the start address by 32 bytes inside the swizzle atom.  MN-major (a row is one K index holding 64 consecutive
// MN elements): 8-row K groups are 1024 B apart and an MN extent of 64 needs no second chunk, so both offsets are 1024.
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ uint64_t make_desc_kmajor_sw128(uint32_t smem_addr) { return make_desc_sw128(smem_addr, 16); }
__device__ __forceinline__ uint64_t make_desc_mnmajor_sw128(uint32_t smem_addr) { return make_desc_sw128(smem_addr, 1024); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of accumulator registers across wgmma issue / wait points
template <int N>
__device__ __forceinline__ void fence_regs(float* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
// register budget of a warpgroup (producer warpgroups give registers to the accumulator-holding consumers)
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}

// ---------------------------------------------------------------- host: per-device opt-in to > 48 KiB dynamic smem
// cudaFuncSetAttribute is a per-DEVICE setting: a process that drives several GPUs must opt in on each of them.
// `done` is a per-kernel bitmask of device ordinals already configured (atomic: first calls may race across threads).
template <typename Kernel>
inline int ensure_dyn_smem(Kernel kernel, int bytes, std::atomic<unsigned long long>& done) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return AAB_ERR_CUDA;
  const unsigned long long bit = 1ull << (dev & 63);
  if (done.load(std::memory_order_acquire) & bit) return AAB_OK;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) return AAB_ERR_CUDA;
  done.fetch_or(bit, std::memory_order_release);
  return AAB_OK;
}

// ---------------------------------------------------------------- programmatic dependent launch (PDL)
// Every kernel of the path is launched with cudaLaunchAttributeProgrammaticStreamSerialization and follows one rule:
//   pdl_trigger()  at the very top   -- the NEXT kernel of the stream may be scheduled as soon as every CTA of this grid
//                                       has started (its CTAs take the SM resources this grid frees while draining);
//   pdl_wait()     before the first global-memory access (read OR write) -- blocks until the PREVIOUS grid has completed
//                                       and its memory is visible.
// So only set-up work (barrier init, descriptor prefetch, index math) overlaps the predecessor's tail; data hazards are
// impossible by construction.  Off by default (launches carry no attribute and both calls are no-ops); AAB_PDL=1 enables it.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("AAB_PDL");
    on = (e && e[0] == '1') ? 1 : 0;
  }
  return on != 0;
}

// kernel<<<grid, block, smem, stream>>>(args...) with the PDL attribute (and an optional cluster dimension)
template <typename... P, typename... A>
inline cudaError_t launch_k(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, A&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<P>(args)...);
}

// ---------------------------------------------------------------- numeric helpers
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
// transformers "quick_gelu" (OpenAI CLIP text towers): x * sigmoid(1.702 x)
__device__ __forceinline__ float quick_gelu_f(float x) { return x / (1.0f + __expf(-1.702f * x)); }
// MUFU without the denormal-scaling wrappers nvcc emits for non-ftz ex2/rcp (2 FSETP + 3 FMUL + FSEL per call)
__device__ __forceinline__ float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_ftz(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// x * sigmoid(x): 2 MUFU + 3 FP32 ops
__device__ __forceinline__ float silu_fast_f(float x) { return x * rcp_ftz(1.0f + ex2_ftz(-1.4426950408889634f * x)); }
// exact-erf GELU with erf by Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, below the rounding of a 16-bit result):
// 2 MUFU + 12 FP32 ops, branch-free (libdevice erff: ~25 instructions with a branch).
__device__ __forceinline__ float gelu_fast_f(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = rcp_ftz(fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float ex = ex2_ftz((x * x) * -0.72134752044448170f);   // exp(-x^2 / 2)
  const float e = fmaf(-(poly * t), ex, 1.0f);                  // erf(|x| / sqrt 2)
  const float h = 0.5f * x;
  return fmaf(fabsf(h), e, h);                                  // 0.5 x (1 + sign(x) e)
}

__device__ __forceinline__ uint32_t pack2(float a, float b, bool bf16) {
  if (bf16) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  } else {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
}
__device__ __forceinline__ float2 unpack2(uint32_t u, bool bf16) {
  if (bf16) {
    __nv_bfloat162 h = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(h);
  } else {
    __half2 h = *reinterpret_cast<__half2*>(&u);
    return __half22float2(h);
  }
}
// value after a round trip through the 16-bit type (what a torch op on a 16-bit tensor leaves behind)
__device__ __forceinline__ float round16(float v, bool bf16) {
  return bf16 ? __bfloat162float(__float2bfloat16_rn(v)) : __half2float(__float2half_rn(v));
}
__device__ __forceinline__ float load_elem(const void* p, size_t i, bool bf16) {
  return bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i])
              : __half2float(reinterpret_cast<const __half*>(p)[i]);
}
__device__ __forceinline__ void store_elem(void* p, size_t i, float v, bool bf16) {
  if (bf16) reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
  else reinterpret_cast<__half*>(p)[i] = __float2half_rn(v);
}

}  // namespace aab
