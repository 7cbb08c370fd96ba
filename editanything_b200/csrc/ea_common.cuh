// ea_common.cuh — sm_90a PTX wrappers shared by every kernel in this library.
//
// Everything here is hand-written inline PTX for Hopper (H100, sm_90a):
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / commit / wait) and the wgmma
// shared-memory descriptor encoders.  No CUTLASS.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "ea_wgmma.cuh"

// ---------------------------------------------------------------------------
// Storage dtype.  fp16 by default (the reference runs fp16 weights/activations
// on GPU: editany_lora.py:372-377 torch_dtype=torch.float16); -DEA_USE_BF16
// switches the whole library to bf16.  Accumulation is always fp32.
// ---------------------------------------------------------------------------
#ifdef EA_USE_BF16
typedef __nv_bfloat16 ea_half;
typedef __nv_bfloat162 ea_half2;
#define EA_TMAP_DTYPE CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
__device__ __forceinline__ float ea_h2f(ea_half h) { return __bfloat162float(h); }
__device__ __forceinline__ ea_half ea_f2h(float f) { return __float2bfloat16_rn(f); }
__device__ __forceinline__ uint32_t ea_pack2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 ea_unpack2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
#else
typedef __half ea_half;
typedef __half2 ea_half2;
#define EA_TMAP_DTYPE CU_TENSOR_MAP_DATA_TYPE_FLOAT16
__device__ __forceinline__ float ea_h2f(ea_half h) { return __half2float(h); }
__device__ __forceinline__ ea_half ea_f2h(float f) { return __float2half_rn(f); }
__device__ __forceinline__ uint32_t ea_pack2(float a, float b) {
  __half2 v = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 ea_unpack2(uint32_t u) {
  __half2 v = *reinterpret_cast<__half2*>(&u);
  return __half22float2(v);
}
#endif

namespace ea {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------- mbarrier ---------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
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
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a wrong expect_tx count or a faulted TMA must not hang the GPU
// (the box is shared; a hung kernel is a strike).  ~2^28 polls (seconds) then trap.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 28)) { asm volatile("trap;"); }
  }
}

// --------------------------------- TMA -------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// L2 prefetch of one box (no shared memory, no barrier): a hint, out-of-range boxes are harmless
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* m, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// The same with an L2 eviction-priority hint (createpolicy encodings: 0x12F0000000000000 = evict first,
// 0x14F0000000000000 = evict last); policy 0 = plain load.
__device__ __forceinline__ void tma_load_2d_hint(void* smem, const CUtensorMap* m, uint64_t* bar, int c0,
                                                 int c1, uint64_t policy) {
  if (policy == 0ull) {
    tma_load_2d(smem, m, bar, c0, c1);
    return;
  }
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, "
      "%4}], [%2], %5;" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
      "%4, %5, %6}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// -------------------------------- wgmma -------------------------------------
// Warpgroup MMA (sm_90a): 128 threads issue one wgmma.mma_async together; the fp32 accumulator lives in
// their registers (layout: ea_wgmma.cuh).  fence before the first wgmma that reads registers written by
// ordinary instructions, commit closes a group, wait<N> leaves at most N groups in flight.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// The accumulator registers are written asynchronously: this empty asm pins every access to them on its side
// of a wgmma_wait (without it the compiler may read an accumulator before the MMA that writes it completed).
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Warp-specialised register budgets: every warp of a warp-group executes the same setmaxnreg; .dec hands registers
// back to the SM's pool, .inc waits until the pool can grant the larger budget.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// --------------------------- wgmma descriptors -------------------------------
// Shared-memory matrix descriptor (64-bit), sm_90 layout:
//   [0,14)  start address >> 4        [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset>>4 [49,52) base offset = 0
//   [62,64) layout: 0 none, 1 = SW128, 2 = SW64, 3 = SW32
//
// K-major operand, SWIZZLE_128B: rows are 128 B (64 halves) apart, groups of 8 rows are
// `sbo_bytes` apart (1024 for a dense tile); LBO is unused.  Stepping K by 16 halves inside the
// 128 B swizzle atom = +32 B on the start address.
__device__ __forceinline__ uint64_t gmma_desc_k_sw128(uint32_t saddr, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;  // LBO (ignored for swizzled K-major)
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}
// MN-major operand, SWIZZLE_128B: the atom is 64 MN-elements (128 B) x 8 K-rows (1024 B);
// atoms along MN are `lbo_bytes` apart, groups of 8 K-rows are `sbo_bytes` apart.
__device__ __forceinline__ uint64_t gmma_desc_mn_sw128(uint32_t saddr, uint32_t lbo_bytes,
                                                       uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// MN-major operand, SWIZZLE_32B: the atom is 16 MN-elements (32 B) x 8 K-rows (256 B), so N may be any multiple
// of 16; 16-wide column blocks are `lbo_bytes` apart, groups of 8 K-rows `sbo_bytes` apart.
__device__ __forceinline__ uint64_t gmma_desc_mn_sw32(uint32_t saddr, uint32_t lbo_bytes,
                                                      uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)3 << 62;
  return d;
}

// ------------------------- programmatic dependent launch -------------------
// wait: all prerequisite grids have completed and their writes are visible (no-op when the kernel
// was not launched with the programmatic-serialisation attribute).  launch_dependents: the next
// kernel on the stream may start its prologue once every CTA of this grid has issued it.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// --------------------------------- math ------------------------------------
// Compact forms on purpose: these are inlined 32x per epilogue chunk, and with IEEE division / libdevice
// erff they were HALF of the GEMM kernel's 240 KB of SASS - the epilogue ran out of the instruction
// cache whenever launches of different shapes alternated.
__device__ __forceinline__ float mufu_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float mufu_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float silu_f(float x) {
  return x * mufu_rcp(1.0f + mufu_ex2(x * -1.4426950408889634f));
}
// exact-erf GELU (F.gelu default) with erf from Abramowitz & Stegun 7.1.26, |abs err| < 1.5e-7:
// erf(z) = 1 - (a1 t + .. + a5 t^5) exp(-z^2), t = 1 / (1 + p z), z >= 0.  ~17 instructions.
__device__ __forceinline__ float gelu_erf_f(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = mufu_rcp(fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float e = fmaf(-poly * t, mufu_ex2(z * z * -1.4426950408889634f), 1.0f);   // erf(|x| / sqrt 2)
  return 0.5f * x * (1.0f + copysignf(e, x));
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

}  // namespace ea
