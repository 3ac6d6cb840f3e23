// panfusion_b200 — shared device/host helpers for the sm_90a kernels.
// PTX wrappers for mbarrier, TMA (cp.async.bulk[.tensor]) and wgmma (warpgroup MMA, accumulators in registers).
// Descriptor bit layouts follow the PTX ISA "Matrix Descriptor Format" table of the wgmma section.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/panfusion_b200.h"

namespace pf {

// ----------------------------------------------------------------------------------------------
// host-side error plumbing (thread-local message, C-ABI returns negative codes)
// ----------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int  check_cuda(cudaError_t e, const char* what);
int  sm_count();    // SMs of the current device (cached; 132 on an H100 SXM when no device can be queried)

#define PF_CHECK_ARG(cond, ...)                      \
  do {                                               \
    if (!(cond)) {                                   \
      ::pf::set_error(__VA_ARGS__);                  \
      return PF_ERR_INVALID;                         \
    }                                                \
  } while (0)

#define PF_CHECK_LAUNCH(what)                                         \
  do {                                                                \
    int _rc = ::pf::check_cuda(cudaGetLastError(), what);             \
    if (_rc) return _rc;                                              \
  } while (0)

// TMA tensor-map encoding through the driver entry point (no -lcuda link dependency).
// dims/strides innermost-first; strides in bytes for dims 1..rank-1.
int make_tmap(CUtensorMap* out, int dtype /*PF_BF16|PF_F16*/, int rank, const void* base,
              const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
              int swizzle_bytes /*128|64|32|0*/);

// ----------------------------------------------------------------------------------------------
// device helpers
// ----------------------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier -------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// generic-proxy writes (st.shared) -> visible to the async proxy (TMA / UMMA operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a launch failure (trap), never as a hung GPU. No printf here: a function
// call in a kernel makes ptxas serialize its wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();  // ~2 s at 2 GHz
  }
}

// ---- TMA ------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* t) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(t) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* t, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(t), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* t, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(t), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// TMA tile store shared -> global (bulk async group); rows/cols outside the tensor are clipped by the hardware
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* t, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(t),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until the bulk stores of this thread have finished READING shared memory (safe to exit / reuse smem)
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// 1-D bulk copy global -> shared (UBLKCP); bytes multiple of 16, both addresses 16 B aligned
__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA) -------------------------------------------------------------
// All four warps of a warpgroup execute these together. fence: orders register accesses to the accumulators before
// the next wgmma; commit: closes a group of issued wgmma; wait<N>: until at most N groups are still in flight.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads/writes across the asynchronous wgmma
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor of wgmma (sm_90).
//   [0,14) start>>4  [16,30) LBO>>4  [32,46) SBO>>4  [49,52) base offset (0: tiles are swizzle-pattern aligned)
//   [62,64) layout type: 0 none, 1 = 128B swizzle, 2 = 64B swizzle, 3 = 32B swizzle
// K-major operands: SBO = bytes between 8-row groups, LBO unused; a 16-element K step inside a swizzle row is +32 B.
// MN-major operands: SBO = bytes between 8-row groups along K, LBO = bytes between swizzle atoms along MN.
__device__ __forceinline__ uint64_t make_wgmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                    uint32_t layout_type) {
  return uint64_t((saddr & 0x3FFFFu) >> 4) | (uint64_t(lbo_bytes >> 4) << 16) | (uint64_t(sbo_bytes >> 4) << 32) |
         (uint64_t(layout_type) << 62);
}

// ---- small numeric helpers -----------------------------------------------------------------
template <typename T>
struct Cvt;
template <>
struct Cvt<float> {
  static __device__ __forceinline__ float to_f(float v) { return v; }
  static __device__ __forceinline__ float from_f(float v) { return v; }
};
template <>
struct Cvt<__nv_bfloat16> {
  static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
template <>
struct Cvt<__half> {
  static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};

// pack two floats into one 32-bit word of 16-bit elements (lo = a, hi = b)
template <bool BF16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  if constexpr (BF16) {
    __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&t);
  } else {
    __half2 t = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&t);
  }
}
template <bool BF16>
__device__ __forceinline__ float2 unpack2(uint32_t w) {
  if constexpr (BF16) {
    __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&w);
    return __bfloat1622float2(t);
  } else {
    __half2 t = *reinterpret_cast<__half2*>(&w);
    return __half22float2(t);
  }
}

// MUFU wrappers without the denormal range fix-ups nvcc wraps around expf / division (2 FSETP + FSEL + 3 FMUL per
// call — the GEGLU epilogue evaluates one erf-GELU per output): results feed 16-bit stores.
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// x * sigmoid(x): FMUL, MUFU.EX2, FADD, MUFU.RCP, FMUL (relative error ~3e-7)
__device__ __forceinline__ float silu_f(float x) {
  return x * rcp_approx(1.0f + ex2_approx(-1.4426950408889634f * x));
}
// CLIP's quick_gelu, x * sigmoid(1.702 x): the same five instructions with the factor 1.702 * log2(e) folded in
__device__ __forceinline__ float quick_gelu_f(float x) {
  return x * rcp_approx(1.0f + ex2_approx(-2.4554669595930157f * x));
}
// exact-erf GELU (F.gelu default) with erf from Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7 + MUFU round-off,
// three orders of magnitude below one 16-bit output ulp): 2 MUFU + 7 FFMA + 5 FMUL + 1 LOP3 instead of erff()'s
// branchy ~30-instruction sequence — the GEGLU epilogue evaluates it 80x per thread per tile.
__device__ __forceinline__ float erf_as_f(float x) {
  const float ax = fabsf(x);
  const float t = rcp_approx(fmaf(0.3275911f, ax, 1.0f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float r = fmaf(-p * t, ex2_approx(ax * (ax * -1.4426950408889634f)), 1.0f);
  return copysignf(r, x);
}
__device__ __forceinline__ float gelu_erf_f(float x) {
  const float hx = 0.5f * x;
  return fmaf(hx, erf_as_f(x * 0.70710678118654752440f), hx);
}

// (a0 + ba0) * gelu(g0 + bg0), (a1 + ba1) * gelu(g1 + bg1) for two neighbouring GEGLU columns
__device__ __forceinline__ void geglu_pair(float a0, float a1, float g0, float g1, float ba0, float ba1, float bg0, float bg1,
                                           float& o0, float& o1) {
  o0 = (a0 + ba0) * gelu_erf_f(g0 + bg0);
  o1 = (a1 + ba1) * gelu_erf_f(g1 + bg1);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

#endif  // __CUDACC__

}  // namespace pf
