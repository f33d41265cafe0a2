// Common device-side PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor) and small
// numeric helpers (the wgmma wrappers are in wgmma.cuh).  Everything here is hand-written inline
// PTX; no CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>

// 16-bit storage type of this build of the library.  The library is compiled twice from the same sources:
// libidiff_b200.so (fp16 activations / weights, the reference's autocast type, inference.py:94) and
// libidiff_b200_bf16.so (-DIDIFF_STORAGE_BF16=1, BASELINE config 3).  Accumulation, statistics and the
// sampler state are fp32 in both; only the operand format of the wgmmas and the pack / unpack at the
// edges of each kernel differ, so every kernel below is written against h16 / pack_half2 / unpack_half2.
#ifndef IDIFF_STORAGE_BF16
#define IDIFF_STORAGE_BF16 0
#endif
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <math.h>

namespace idiff {

#define IDIFF_DEVICE __device__ __forceinline__

// Programmatic dependent launch (host.cuh launch_pdl): launch_dependents lets the next kernel in the
// stream become resident and run its prologue while this one is still working; wait blocks until the
// previous kernel has completed and its global writes are visible.  Both are no-ops for a kernel
// launched without the attribute.
IDIFF_DEVICE void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory"); }
IDIFF_DEVICE void pdl_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }

IDIFF_DEVICE uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

IDIFF_DEVICE bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------
IDIFF_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
IDIFF_DEVICE void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
IDIFF_DEVICE void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
// expect `bytes` more transaction bytes in the current phase without arriving (the arrival comes separately)
IDIFF_DEVICE void mbar_expect_tx_only(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
IDIFF_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
IDIFF_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Non-blocking probe (try_wait may suspend the thread for a system-defined time; a polling loop over
// several barriers wants the immediate answer).
IDIFF_DEVICE bool mbar_test(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trapped launch (an error code at the C ABI),
// never as a hung GPU.  ~4 s at 2 GHz.  (No printf here: a function call in a kernel that issues
// wgmma makes ptxas serialise every wgmma.)
IDIFF_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3ff) == 0 && (clock64() - t0) > 8000000000LL) __trap();
  }
}

// generic-proxy smem writes -> visible to the async proxy (wgmma / TMA reads)
IDIFF_DEVICE void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}

// Named barriers (ids 1..15; 0 is __syncthreads): `nthreads` counts the threads of every warp that
// syncs or arrives, so one group can wait on a barrier that another group only arrives at.
IDIFF_DEVICE void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(nthreads) : "memory");
}
IDIFF_DEVICE void named_bar_arrive(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.arrive %0, %1;\n" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------------
// TMA tiled loads (global -> shared, completion on an mbarrier)
// ----------------------------------------------------------------------------------
IDIFF_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
IDIFF_DEVICE void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];\n" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
IDIFF_DEVICE void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                              int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];\n" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
IDIFF_DEVICE void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                              int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];\n" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// TMA tiled stores (shared -> global, bulk async-group completion)
IDIFF_DEVICE void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
IDIFF_DEVICE void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];\n" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
IDIFF_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
// all bulk groups of this thread have finished READING shared memory (buffers reusable)
IDIFF_DEVICE void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory"); }
// all bulk groups of this thread have completed (their global writes are done)
IDIFF_DEVICE void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;\n" ::: "memory"); }

// ----------------------------------------------------------------------------------
// ldmatrix / stmatrix: four 8x8 16-bit matrices between shared memory and the mma fragment layout
// (thread t holds row t/4, columns 2(t%4) and 2(t%4)+1 of matrix i in r[i]); lanes 8i..8i+7 give the
// row addresses (16 B each) of matrix i.
// ----------------------------------------------------------------------------------
IDIFF_DEVICE void ldmatrix_x4(uint32_t (&r)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(saddr)
               : "memory");
}
IDIFF_DEVICE void stmatrix_x4(uint32_t saddr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};\n" ::"r"(saddr), "r"(r[0]),
               "r"(r[1]), "r"(r[2]), "r"(r[3])
               : "memory");
}

// ----------------------------------------------------------------------------------
// numerics
// ----------------------------------------------------------------------------------
#if IDIFF_STORAGE_BF16
using h16 = __nv_bfloat16;
IDIFF_DEVICE uint32_t pack_half2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
IDIFF_DEVICE float2 unpack_half2(uint32_t u) {  // bf16 is the upper half of an fp32: two integer ops
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
IDIFF_DEVICE float h2f(h16 x) { return __bfloat162float(x); }
IDIFF_DEVICE h16 f2h(float x) { return __float2bfloat16_rn(x); }
#else
using h16 = __half;
IDIFF_DEVICE uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
IDIFF_DEVICE float2 unpack_half2(uint32_t u) {
  __half2 h = *reinterpret_cast<__half2*>(&u);
  return __half22float2(h);
}
IDIFF_DEVICE float h2f(h16 x) { return __half2float(x); }
IDIFF_DEVICE h16 f2h(float x) { return __float2half_rn(x); }
#endif
IDIFF_DEVICE float silu_f(float x) { return x / (1.0f + __expf(-x)); }
// LayerNorm scale of a row from its (sum, sum of squares) over K elements: y = rstd * x + nmean
IDIFF_DEVICE void ln_scale(float sum, float sumsq, int K, float eps, float& rstd, float& nmean) {
  const float inv_k = 1.0f / (float)K;
  const float mean = sum * inv_k;
  rstd = rsqrtf(fmaxf(sumsq * inv_k - mean * mean, 0.f) + eps);
  nmean = -mean * rstd;
}
// Exact (erf) GELU of attention.py:43, x * 0.5 * (1 + erf(x / sqrt 2)), with erf from
// Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7, far below the fp16 output resolution): one MUFU.RCP,
// one MUFU.EX2 and ten FMAs instead of libdevice erff (~2x the instructions).  1 + erf is formed
// without cancellation on the negative side: 1 + erf(-z) = poly(t) * exp(-z^2).
IDIFF_DEVICE float gelu_erf_f(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  float poly = fmaf(t, 1.061405429f, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(z * z * -1.4426950408889634f));
  const float pe = poly * e;                       // = 1 - erf(z)
  const float one_plus_erf = (x >= 0.f) ? (2.0f - pe) : pe;
  return 0.5f * x * one_plus_erf;
}
IDIFF_DEVICE float exp2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Philox4x32-10 (Salmon et al., SC'11; the Random123 constants): a counter-based generator, so a draw is a pure
// function of (counter, key) and needs no state carried between launches.
IDIFF_DEVICE uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}
// uint32 -> uniform (v + 0.5) * 2^-32 in (0, 1), rounded to fp32
IDIFF_DEVICE float u01_open(uint32_t v) { return ((float)v + 0.5f) * 2.3283064365386963e-10f; }
// Box-Muller on two uniform words: z0 = r cos(2 pi u_b), z1 = r sin(2 pi u_b), r = sqrt(-2 ln u_a), u = (v + 0.5) 2^-32.
// For u_a above 1/2, ln u_a is log1p(-(1 - u_a)) with 1 - u_a = (~a + 0.5) 2^-32 formed exactly, so small radii keep
// their precision (u_a rounded to fp32 would lose most of the bits of 1 - u_a).  Precise logf / sincospif throughout.
IDIFF_DEVICE void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
  const float ln_u = a < 0x80000000u ? logf(u01_open(a)) : log1pf(-u01_open(~a));
  const float r = sqrtf(-2.0f * ln_u);
  float s, c;
  sincospif(2.0f * u01_open(b), &s, &c);
  z0 = r * c;
  z1 = r * s;
}

}  // namespace idiff
