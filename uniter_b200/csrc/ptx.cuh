// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor, with cluster
// multicast), clusters, wgmma shared-memory descriptors.  The wgmma instructions themselves are
// in wgmma.cuh.  Everything here is hand-written for H100; there is no fallback path.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ub {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- programmatic dependent launch
// Every kernel of the library is launched with programmaticStreamSerialization allowed: it
// lets its dependents start launching right away (they only run their prologue) and waits
// here until the preceding grid has completed and its writes are visible.  Hides launch latency
// and prologues behind the previous kernel's tail (~250 launches of ~20 us per step).
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// explicit shared-space accesses (the dynamic-smem base is re-aligned with integer arithmetic,
// after which the compiler only knows a generic pointer and would emit generic ST.E / LD.E)
__device__ __forceinline__ void st_shared_f32(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ float ld_shared_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}

// ---------------------------------------------------------------- fences
__device__ __forceinline__ void fence_proxy_async_smem() {
  // make generic-proxy smem writes visible to the async proxy (wgmma / TMA reads)
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load, completes on an mbarrier with transaction bytes. c0 = innermost coordinate.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
        "r"(c1)
      : "memory");
}

// 2-D tiled load multicast to the CTAs of `cta_mask` in the cluster: the tile lands at the same
// shared-memory offset in each of them and completes on the mbarrier at the same offset there.
__device__ __forceinline__ void tma_load_2d_mc(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                               int c0, int c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
        "r"(c1), "h"(cta_mask)
      : "memory");
}

// ---------------------------------------------------------------- clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// shared::cluster address of `local` (a shared::cta address of this CTA) in CTA `cta` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t local, uint32_t cta) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local), "r"(cta));
  return r;
}
// arrive (count 1) on an mbarrier given by shared::cluster address (possibly in the peer CTA).
// Default (.release.cta) semantics on purpose: `.release.cluster` compiles to MEMBAR.ALL.GPU +
// ERRBAR, which serialised the pipeline when used once per k-block.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar_cluster_addr) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(bar_cluster_addr) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---------------------------------------------------------------- wgmma descriptors
// Shared-memory matrix descriptor, 128-byte swizzle (layout type 1 in bits [62,64)).
//   K-major  tile: rows of 128 B (64 x 16-bit along K); 8-row groups 1024 B apart (SBO).
//   MN-major tile: rows of 128 B (64 x 16-bit along M/N), one row per K index; 8-K groups
//                  1024 B apart (SBO); 64-wide M/N groups `lbo_bytes` apart (LBO).
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);              // [0,14)  start address
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;     // [16,30) leading byte offset
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;     // [32,46) stride byte offset
  d |= static_cast<uint64_t>(1) << 62;                              // SWIZZLE_128B
  return d;
}

// ---------------------------------------------------------------- 16-bit storage types
template <bool kBF16>
struct Elem;
template <>
struct Elem<true> {
  using T = __nv_bfloat16;
  using T2 = __nv_bfloat162;
  static __device__ __forceinline__ float to_f(T v) { return __bfloat162float(v); }
  static __device__ __forceinline__ T from_f(float v) { return __float2bfloat16_rn(v); }
  static __device__ __forceinline__ uint32_t pack(float lo, float hi) {
    __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&t);
  }
  static __device__ __forceinline__ float2 unpack(uint32_t u) {
    __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(t);
  }
};
template <>
struct Elem<false> {
  using T = __half;
  using T2 = __half2;
  static __device__ __forceinline__ float to_f(T v) { return __half2float(v); }
  static __device__ __forceinline__ T from_f(float v) { return __float2half_rn(v); }
  static __device__ __forceinline__ uint32_t pack(float lo, float hi) {
    __half2 t = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&t);
  }
  static __device__ __forceinline__ float2 unpack(uint32_t u) {
    __half2 t = *reinterpret_cast<__half2*>(&u);
    return __half22float2(t);
  }
};

// ---------------------------------------------------------------- counter-based RNG (dropout)
// Philox-4x32-10; one call yields 128 random bits = eight 16-bit lanes => eight dropout
// decisions.  Element e uses counter (e >> 3) and 16-bit lane (e & 7).  Forward and backward
// regenerate the same mask from (seed, stream, element index), nothing is stored.
__device__ __forceinline__ uint4 philox4x32(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                            uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}
struct DropoutRng {
  uint32_t k0, k1, s0, s1;  // key = seed, (s0,s1) = stream id (site / layer / offset)
  uint32_t thr16;           // drop iff rand16 < thr16
  float inv_keep;
  __device__ __forceinline__ uint4 draw8(uint64_t group) const {
    return philox4x32(static_cast<uint32_t>(group), static_cast<uint32_t>(group >> 32), s0, s1, k0,
                      k1);
  }
};
// Optional device-side stream offset: stream64 += (*dev << 20).  The host-side arguments of a
// launch are frozen inside a CUDA graph; the counter lives in device memory and is bumped between
// replays, so every replay draws fresh dropout masks (forward and backward of one replay read the
// same value).
__device__ __forceinline__ void rng_add_dev_offset(const unsigned long long* dev, uint32_t& s0, uint32_t& s1) {
  if (dev != nullptr) {
    const unsigned long long st = ((static_cast<unsigned long long>(s1) << 32) | s0) + (__ldg(dev) << 20);
    s0 = static_cast<uint32_t>(st);
    s1 = static_cast<uint32_t>(st >> 32);
  }
}
__device__ __forceinline__ uint32_t rand16_of(const uint4& r, int lane8) {
  uint32_t w = (lane8 & 4) ? ((lane8 & 2) ? r.w : r.z) : ((lane8 & 2) ? r.y : r.x);
  return (lane8 & 1) ? (w >> 16) : (w & 0xFFFFu);
}

// ---------------------------------------------------------------- fixed-order column reduction
// Deterministic mode: a 256-thread CTA owns 8 columns; thread t has summed rows t, t + 256, ... in
// ascending order into v[8].  The 256 partials meet in a fixed binary tree, so the result is a
// function of the values and their row indices only (never of the grid).  Returns the total of
// column e in thread e (e < 8).  `red` is 256 x 9 floats of shared memory.
__device__ __forceinline__ float det_tree_sum8(const float (&v)[8], float (*red)[9]) {
  const int t = threadIdx.x;
  __syncthreads();                       // `red` may still be read by a previous call
#pragma unroll
  for (int e = 0; e < 8; ++e) red[t][e] = v[e];
  __syncthreads();
#pragma unroll
  for (int s = 128; s > 0; s >>= 1) {
    if (t < s) {
#pragma unroll
      for (int e = 0; e < 8; ++e) red[t][e] += red[t + s][e];
    }
    __syncthreads();
  }
  return t < 8 ? red[0][t] : 0.f;
}

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

// Standard-normal CDF Phi(x) through erf(|x|/sqrt2) = 1 - poly(t) * exp(-x^2/2),
// t = 1/(1 + p|x|/sqrt2)  (Abramowitz & Stegun 7.1.26).  The formula's 1.5e-7 is an ABSOLUTE error
// of erf; evaluated in fp32 with the MUFU forms below, Phi is within 4e-7 of the exact value (absolute,
// tests/gemm_check.py DELTA_PHI, checked over every 16-bit x).  That is far below the 16-bit rounding
// of gelu(x) = x Phi(x) wherever Phi is not small, but for x < -4 it is a large RELATIVE error of Phi
// (about 3e-4 at -4, 4e-2 at -5; Phi is 0 below about -6): the GELU tail is accurate to |x| * 4e-7
// absolute, still closer than the reference model's composed 16-bit GELU, whose 1 + erf is quantised
// to the 16-bit spacing below 1 (it gives gelu(-4) = 0).  `ex` returns exp(-x^2/2), shared with the pdf
// in the derivative.
// The reciprocal and the exponential are the bare MUFU approximations (rcp.approx.ftz on an
// argument >= 1, ex2.approx.ftz on x^2 * -log2(e)/2), without the range-handling FSETP / FMUL /
// branch sequences __fdividef / __expf add: the GELU epilogues run once per output element and
// compete for issue slots with the rest of the epilogue.
__device__ __forceinline__ float normal_cdf(float x, float& ex) {
  const float ax = fabsf(x) * 0.70710678118654752440f;
  const float t = rcp_approx(fmaf(0.3275911f, ax, 1.0f));
  ex = ex2_approx((x * x) * -0.72134752044448170368f);     // exp(-x^2 / 2)
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float erf_abs = fmaf(-poly * t, ex, 1.0f);
  return fmaf(0.5f, copysignf(erf_abs, x), 0.5f);
}
__device__ __forceinline__ float gelu_erf(float x) {
  float ex;
  return x * normal_cdf(x, ex);          // x * 0.5 * (1 + erf(x / sqrt2)), model/layer.py:31-37
}
__device__ __forceinline__ float dgelu_erf(float x) {
  float ex;                               // d/dx [x Phi(x)] = Phi(x) + x phi(x)
  const float cdf = normal_cdf(x, ex);
  return fmaf(x * 0.39894228040143267794f, ex, cdf);
}

}  // namespace ub
