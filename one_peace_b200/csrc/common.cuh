// Shared device helpers for the sm_90a kernels: mbarrier, TMA, small math and packing helpers.
// Everything here is inline PTX for sm_90a; there is no fallback path for other architectures.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define OPB_DEVICE __device__ __forceinline__

// status codes shared with include/onepeace_b200.h
#define OPB_OK 0
#define OPB_ERR_INVALID 1
#define OPB_ERR_CUDA 2
#define OPB_ERR_UNSUPPORTED 3

namespace opb {

// ----------------------------------------------------------------------------------------------
// misc
// ----------------------------------------------------------------------------------------------
OPB_DEVICE uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
OPB_DEVICE uint32_t lane_id() { return threadIdx.x & 31; }

OPB_DEVICE bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

OPB_DEVICE uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
OPB_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
OPB_DEVICE void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
OPB_DEVICE void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

OPB_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
OPB_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// one thread arriving on behalf of `count` (e.g. every warp of its warpgroup)
OPB_DEVICE void mbar_arrive_count(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
OPB_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

// Bounded wait: a protocol bug must trap (and surface as a CUDA error) instead of hanging the GPU.
#ifndef OPB_WATCHDOG_NS
#define OPB_WATCHDOG_NS 4000000000ull
#endif
OPB_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint64_t t0 = globaltimer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3ff) == 0) {
      if (globaltimer_ns() - t0 > OPB_WATCHDOG_NS) {
        printf("[opb] mbarrier watchdog: block %d thread %d bar@%u parity %u\n", (int)blockIdx.x,
               (int)threadIdx.x, smem_u32(bar), parity);
        __trap();
      }
    }
  }
}

// Bounded wait without mbar_wait's printf: a function call anywhere in a kernel makes ptxas serialise its wgmma pipeline
OPB_DEVICE void mbar_wait_quiet(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  while (!mbar_try_wait(bar, parity)) {
    if (globaltimer_ns() - t0 > OPB_WATCHDOG_NS) __trap();
  }
}

// ----------------------------------------------------------------------------------------------
// wgmma
// ----------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (sm_90), 128-byte swizzle.  K-major: rows of 128 B, 8-row groups SBO = 1024 B apart (LBO
// unused).  MN-major: atoms of 64 MN elements x 8 k-rows (1024 B), k groups SBO = 1024 B apart, 64-wide MN chunks LBO apart.
OPB_DEVICE uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t lbo) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;   // layout type 1 = SWIZZLE_128B
  return d;
}

OPB_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
OPB_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
OPB_DEVICE void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// SM count of the current device, queried once per translation unit (persistent grids)
static inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) — 2D tiles global -> shared
// ----------------------------------------------------------------------------------------------
OPB_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

OPB_DEVICE void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
OPB_DEVICE void tma_load_3d(const CUtensorMap* m, uint64_t* bar, void* dst, int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      :
      : "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// 1-D bulk copy global -> shared (size multiple of 16 B, both addresses 16-B aligned), completion on an mbarrier
OPB_DEVICE void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// TMA store (shared -> global), bulk-group completion
OPB_DEVICE void tma_store_2d(const CUtensorMap* m, const void* src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
OPB_DEVICE void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
OPB_DEVICE void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
OPB_DEVICE void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// byte offset of 16-byte chunk `chunk` (0..3) of row `row` in a [rows][64 B] tile stored with the 64-byte swizzle
OPB_DEVICE uint32_t sw64_off(int row, int chunk) { return row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4); }
// byte offset of 16-byte chunk `chunk` of row `row` in a [rows][128 B] tile stored with the 128-byte swizzle
OPB_DEVICE uint32_t sw128_off(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }

// ----------------------------------------------------------------------------------------------
// math / packing
// ----------------------------------------------------------------------------------------------
// erf(x) after Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7, i.e. fp32 round-off level): one MUFU.RCP, one
// MUFU.EX2 and a 5-term Horner polynomial instead of libdevice erff's ~35 instructions.  The exact-GELU epilogue of
// the GeGLU GEMM evaluates it 16 M times per layer and was epilogue-compute-bound with erff.
OPB_DEVICE float fast_erf(float x) {
  const float ax = fabsf(x);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, ax, 1.0f)));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  p *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * ax * ax));
  const float r = fmaf(-p, e, 1.0f);
  return copysignf(r, x);
}
OPB_DEVICE float gelu_erf(float x) { return 0.5f * x * (1.0f + fast_erf(x * 0.70710678118654752440f)); }

// explicit shared-state-space vector accesses (pointers derived from the dynamic smem base otherwise compile to
// generic LD/ST with 64-bit addresses)
// (Plain pointer accesses: volatile inline-asm ld/st.shared would pin every access in program order and serialise the
// epilogue on shared-memory latency; the pointers must derive directly from the `extern __shared__` array so that the
// compiler keeps the shared state space and emits LDS / STS rather than generic LD / ST.)
OPB_DEVICE float4 lds128(const uint8_t* p) { return *reinterpret_cast<const float4*>(p); }
OPB_DEVICE void sts128(uint8_t* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
OPB_DEVICE void sts128u(uint8_t* p, uint4 v) { *reinterpret_cast<uint4*>(p) = v; }

OPB_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
OPB_DEVICE float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

OPB_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
OPB_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace opb
