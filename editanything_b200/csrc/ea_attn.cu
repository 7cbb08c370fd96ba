// ea_attn.cu — fused attention on wgmma (sm_90a): O = softmax(Q K^T * scale [+ bias]) V.
//
// Replaces the einsum -> softmax -> einsum of CrossAttention.forward
// (ldm/modules/attention.py:170-193; QK^T accumulated in fp32 like the reference's
// _ATTN_PRECISION="fp32" path) and SAM's windowed / global attention with decomposed relative
// position bias (SURVEY.md App. C).  The N x N logits never touch HBM.
//
// One CTA = one (batch, head) and a tile of 128 query rows; two warp-groups, warp-group g owns query rows
// 64g .. 64g+63.  Per 128-key tile:
//              S = Q K^T with wgmma (A = Q, B = K, both K-major from shared memory) into 64 fp32 registers per
//              thread; scale (+ the SAM rel-pos bias in the BIAS kernels), mask of missing keys, online softmax
//              with the running max / sum per row (a row's 128 logits sit on the 4 lanes of a quad); P packed to
//              16 bit straight from the accumulator layout into the A-operand fragments of the second wgmma,
//              O += P V (B = V, MN-major from its row-major tile) into DO / 2 registers per thread.  Final 1 / l
//              normalisation and stores.
// Thread 0 also drives TMA: the Q tile once, then K/V tiles into a `stages`-deep ring, refilling a stage with the
// tile `stages` ahead as soon as every warp has released it (a separate producer warp would put three warps on one
// SM sub-partition and cap every thread at 168 registers: the 192-wide P V accumulator alone is 96).  Head dims that are not a multiple of 64 (40, 80, 160) are zero-padded for free by TMA
// out-of-bounds fill (tensor-map inner extent d, box 64 wide).
#include <stdlib.h>
#include "ea_common.cuh"
#include "ea_internal.h"

namespace ea {

static constexpr int AT_BQ = 128;
static constexpr int AT_BKV = 128;
static constexpr int AT_ATOM = 128 * 128;  // bytes of one 128-row x 64-half swizzled atom
static constexpr int AT_MAX_STAGES = 4;
static constexpr int AT_THREADS = 256;   // no separate producer warp: 8 warps may use up to 255 registers a thread
static constexpr int AT_WARPS = 8;

struct AttnKParams {
  int Nq, Nkv, d, heads;
  int nd;      // ceil(d / 64) atoms along the head dim
  int ksteps;  // ceil(d / 16) MMA K-steps for Q K^T
  int stages;
  float scale_log2;
  ea_half* out;
  long long o_bs, o_ns;
  const float* rel_h;
  const float* rel_w;
  int rel_s;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int R>
__device__ __forceinline__ void wgmma_fence_regs_u32(uint32_t (&a)[R][4]) {
#pragma unroll
  for (int i = 0; i < R; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) asm volatile("" : "+r"(a[i][k])::"memory");
}

// DO: width of the P V accumulator (64 / 128 / 192, >= d; the columns past d are TMA zero fill)
template <int DO, bool BIAS>
__global__ void __launch_bounds__(AT_THREADS, 1)
ea_attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, const AttnKParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~uintptr_t(1023));
  // layout: Q[nd] | KV[stages][K nd | V nd] | rel_w rows (BIAS) | barriers
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + p.nd * AT_ATOM;
  const int kv_stage_bytes = 2 * p.nd * AT_ATOM;
  float* rw_s = reinterpret_cast<float*>(sKV + p.stages * kv_stage_bytes);   // [128][rel_s + 1]
  const int bias_floats = BIAS ? ((AT_BQ * (p.rel_s + 1) + 3) & ~3) : 0;
  uint64_t* bars = reinterpret_cast<uint64_t*>(rw_s + bias_floats);
  uint64_t* q_full = bars;                      // [1]
  uint64_t* kv_full = bars + 1;                 // [AT_MAX_STAGES]
  uint64_t* kv_empty = kv_full + AT_MAX_STAGES; // [AT_MAX_STAGES]

  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int qb = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int n_tiles = (p.Nkv + AT_BKV - 1) / AT_BKV;
  const bool producer = threadIdx.x == 0;

  if (producer) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int s = 0; s < AT_MAX_STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], AT_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  // K/V tile jj into its stage of the ring (thread 0; the stage's previous tile has been released)
  auto load_kv = [&](int jj) {
    const int st = jj % p.stages;
    uint8_t* sK = sKV + st * kv_stage_bytes;
    uint8_t* sV = sK + p.nd * AT_ATOM;
    mbar_expect_tx(&kv_full[st], (uint32_t)kv_stage_bytes);
    for (int a = 0; a < p.nd; ++a) {
      tma_load_4d(sK + a * AT_ATOM, &tmK, &kv_full[st], a * 64, head, jj * AT_BKV, b);
      tma_load_4d(sV + a * AT_ATOM, &tmV, &kv_full[st], a * 64, head, jj * AT_BKV, b);
    }
  };
  if (producer) {
    mbar_expect_tx(q_full, (uint32_t)(p.nd * AT_ATOM));
    for (int a = 0; a < p.nd; ++a) tma_load_4d(sQ + a * AT_ATOM, &tmQ, q_full, a * 64, head, qb * AT_BQ, b);
    for (int jj = 0; jj < p.stages && jj < n_tiles; ++jj) load_kv(jj);
  }

  const int wg = warp >> 2, wq = warp & 3;
  const int g = lane >> 2, t4 = lane & 3;
  // accumulator layout (ea_wgmma.cuh): this thread holds rows rl (i % 4 < 2) and rl + 8 (i % 4 >= 2) of the tile,
  // columns 8 (i / 4) + 2 t4 + i % 2
  const int rl = wg * 64 + wq * 16 + g;
  const int q_lo = qb * AT_BQ + rl, q_hi = q_lo + 8;
  const float LOG2E = 1.4426950408889634f;
  const float* rh_lo = nullptr;
  const float* rh_hi = nullptr;
  if (BIAS) {
    // rel_w rows of the CTA's queries (pre-multiplied by log2e) in shared memory; rel_h comes through L1
    const long long bh = (long long)b * p.heads + head;
    for (int idx = threadIdx.x; idx < AT_BQ * p.rel_s; idx += AT_THREADS) {
      const int row = idx / p.rel_s, i = idx - row * p.rel_s;
      const int q = qb * AT_BQ + row;
      rw_s[row * (p.rel_s + 1) + i] = q < p.Nq ? __ldg(p.rel_w + (bh * p.Nq + q) * p.rel_s + i) * LOG2E : 0.f;
    }
    rh_lo = p.rel_h + (bh * p.Nq + (q_lo < p.Nq ? q_lo : 0)) * p.rel_s;
    rh_hi = p.rel_h + (bh * p.Nq + (q_hi < p.Nq ? q_hi : 0)) * p.rel_s;
    asm volatile("bar.sync 1, 256;" ::: "memory");
  }
  const uint64_t dQ0 = gmma_desc_k_sw128(smem_u32(sQ) + (uint32_t)(wg * 64 * 128), 1024);
  const uint64_t dK0 = gmma_desc_k_sw128(smem_u32(sKV), 1024);
  const uint64_t dV0 = gmma_desc_mn_sw128(smem_u32(sKV) + (uint32_t)(p.nd * AT_ATOM), AT_ATOM, 1024);
  const uint32_t kv_stage16 = (uint32_t)kv_stage_bytes >> 4;

  float o[DO / 2];
#pragma unroll
  for (int i = 0; i < DO / 2; ++i) o[i] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY;   // running max in the scaled log2 domain
  float l_lo = 0.f, l_hi = 0.f;               // this thread's share of the running sum
  mbar_wait(q_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int j = 0; j < n_tiles; ++j) {
    mbar_wait(&kv_full[stage], phase);
    // ---- S = Q K^T.  K-step ks sits at atom (ks >> 2), +32 B * (ks & 3)
    float s[64];
    {
      uint64_t dq = dQ0, dk = dK0 + (uint64_t)(stage * kv_stage16);
      wgmma_fence();
      Wgmma<128>::ss(s, dq, dk, 0u);
      for (int ks = 1; ks < p.ksteps; ++ks) {
        const uint32_t step = (ks & 3) ? 2u : (uint32_t)((AT_ATOM >> 4) - 6);
        dq += step;
        dk += step;
        Wgmma<128>::ss(s, dq, dk, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(s);
    }
    // ---- scaled logits (+ bias), missing keys of the last tile -> -inf, row max
    const int valid = min(AT_BKV, p.Nkv - j * AT_BKV);  // keys of this tile that exist (>= 1)
    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int col = 8 * (i >> 2) + 2 * t4;
      const bool hi = (i >> 1) & 1;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float x = s[i + e] * p.scale_log2;
        if (BIAS) {
          const int key = j * AT_BKV + col + e;
          const int kh = key / p.rel_s, kw = key - kh * p.rel_s;
          x += rw_s[(rl + (hi ? 8 : 0)) * (p.rel_s + 1) + kw] + __ldg((hi ? rh_hi : rh_lo) + min(kh, p.rel_s - 1)) * LOG2E;
        }
        if (col + e >= valid) x = -INFINITY;
        s[i + e] = x;
        if (hi) mx_hi = fmaxf(mx_hi, x);
        else mx_lo = fmaxf(mx_lo, x);
      }
    }
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
    const float mn_lo = fmaxf(m_lo, mx_lo), mn_hi = fmaxf(m_hi, mx_hi);
    const float a_lo = ex2_approx(m_lo - mn_lo), a_hi = ex2_approx(m_hi - mn_hi);   // 0 on the first tile
    m_lo = mn_lo;
    m_hi = mn_hi;
    l_lo *= a_lo;
    l_hi *= a_hi;
#pragma unroll
    for (int i = 0; i < DO / 2; ++i) o[i] *= ((i >> 1) & 1) ? a_hi : a_lo;
    // ---- P = exp2(x - m), packed to 16 bit as the A fragments of the 8 K-steps (16 keys each) of P V
    uint32_t pa[8][4];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const int i = 8 * kk + 2 * h;
        const float m = (h & 1) ? m_hi : m_lo;
        const float e0 = ex2_approx(s[i] - m), e1 = ex2_approx(s[i + 1] - m);
        if (h & 1) l_hi += e0 + e1;
        else l_lo += e0 + e1;
        pa[kk][h] = ea_pack2(e0, e1);
      }
    }
    // ---- O += P V ; V K-step kk = 16 key rows = +2048 B
    {
      uint64_t dv = dV0 + (uint64_t)(stage * kv_stage16);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) Wgmma<DO>::rs(o, pa[kk], dv + (uint64_t)(kk * ((16 * 128) >> 4)), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      wgmma_fence_regs_u32(pa);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[stage]);
    if (producer && j + p.stages < n_tiles) {   // every warp has released tile j's stage: refill it
      mbar_wait(&kv_empty[stage], phase);
      load_kv(j + p.stages);
    }
    if (++stage == p.stages) { stage = 0; phase ^= 1u; }
  }
  // ---- epilogue: O / l
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
  const float inv_lo = 1.f / l_lo, inv_hi = 1.f / l_hi;
  ea_half* orow_lo = p.out + (long long)b * p.o_bs + (long long)q_lo * p.o_ns + (long long)head * p.d;
  ea_half* orow_hi = orow_lo + 8 * p.o_ns;
#pragma unroll
  for (int i = 0; i < DO / 2; i += 4) {
    const int col = 8 * (i >> 2) + 2 * t4;
    if (col < p.d) {
      if (q_lo < p.Nq) *reinterpret_cast<uint32_t*>(orow_lo + col) = ea_pack2(o[i] * inv_lo, o[i + 1] * inv_lo);
      if (q_hi < p.Nq) *reinterpret_cast<uint32_t*>(orow_hi + col) = ea_pack2(o[i + 2] * inv_hi, o[i + 3] * inv_hi);
    }
  }
}

static int encode_qkv(CUtensorMap* m, const void* base, int d, int heads, int N, int B,
                      long long ns, long long bs) {
  cuuint64_t dims[4] = {(cuuint64_t)d, (cuuint64_t)heads, (cuuint64_t)N, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)d * 2, (cuuint64_t)ns * 2, (cuuint64_t)bs * 2};
  cuuint32_t box[4] = {64, 1, 128, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = ea_tmap_encode()(m, EA_TMAP_DTYPE, 4, const_cast<void*>(base), dims, strides, box,
                                estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

template <int DO, bool BIAS>
static int launch_attn(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                       const AttnKParams& p, dim3 grid, int smem_bytes, cudaStream_t stream) {
  static int max_set_dev[EA_MAX_DEV];
  int& max_set = max_set_dev[ea_dev()];
  if (smem_bytes > max_set) {
    const cudaError_t e = cudaFuncSetAttribute(ea_attn_kernel<DO, BIAS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               smem_bytes);
    if (e != cudaSuccess) return ea_cuda_fail(e, "ea_attention: cudaFuncSetAttribute(MaxDynamicSharedMemorySize)");
    max_set = smem_bytes;
  }
  const cudaError_t e = ea_launch(ea_attn_kernel<DO, BIAS>, grid, dim3(AT_THREADS), (size_t)smem_bytes, stream,
                                  tq, tk, tv, p);
  return e == cudaSuccess ? 0 : ea_cuda_fail(e, "ea_attention: kernel launch");
}

}  // namespace ea

using namespace ea;

extern "C" int ea_attention(const ea_attn_args* a, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!a || !a->q || !a->k || !a->v || !a->out) return EA_ERR_ARG;
  if (a->d % 8 != 0 || a->d < 8 || a->d > 192) return EA_ERR_SHAPE;
  if (a->Nq <= 0 || a->Nkv <= 0 || a->B <= 0 || a->heads <= 0) return EA_ERR_SHAPE;
  if (a->q_ns % 8 || a->k_ns % 8 || a->v_ns % 8 || a->q_bs % 8 || a->k_bs % 8 || a->v_bs % 8 ||
      a->o_ns % 8 || a->o_bs % 8)
    return EA_ERR_SHAPE;
  if ((a->rel_h != nullptr) != (a->rel_w != nullptr)) return EA_ERR_ARG;
  if (a->rel_h && a->rel_s <= 0) return EA_ERR_ARG;

  AttnKParams p;
  memset(&p, 0, sizeof(p));
  p.Nq = a->Nq; p.Nkv = a->Nkv; p.d = a->d; p.heads = a->heads;
  p.nd = (a->d + 63) / 64;
  p.ksteps = (a->d + 15) / 16;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.out = reinterpret_cast<ea_half*>(a->out);
  p.o_bs = a->o_bs; p.o_ns = a->o_ns;
  p.rel_h = a->rel_h; p.rel_w = a->rel_w; p.rel_s = a->rel_s;

  const bool bias = a->rel_h != nullptr;
  const int budget = 227 * 1024 - 1024 - 256;
  const int bias_bytes = bias ? ((AT_BQ * (a->rel_s + 1) + 3) & ~3) * 4 : 0;
  int stages = (budget - p.nd * AT_ATOM - bias_bytes) / (2 * p.nd * AT_ATOM);
  if (stages > AT_MAX_STAGES) stages = AT_MAX_STAGES;
  if (stages < 1) return EA_ERR_SHAPE;
  const int n_tiles = (a->Nkv + AT_BKV - 1) / AT_BKV;
  if (stages > n_tiles) stages = n_tiles;
  p.stages = stages;

  CUtensorMap tq, tk, tv;
  if (encode_qkv(&tq, a->q, a->d, a->heads, a->Nq, a->B, a->q_ns, a->q_bs)) return EA_ERR_TMAP;
  if (encode_qkv(&tk, a->k, a->d, a->heads, a->Nkv, a->B, a->k_ns, a->k_bs)) return EA_ERR_TMAP;
  if (encode_qkv(&tv, a->v, a->d, a->heads, a->Nkv, a->B, a->v_ns, a->v_bs)) return EA_ERR_TMAP;

  const int smem_bytes = p.nd * AT_ATOM + stages * 2 * p.nd * AT_ATOM + bias_bytes + (1 + 2 * AT_MAX_STAGES) * 8 + 1024;
  dim3 grid((unsigned)((a->Nq + AT_BQ - 1) / AT_BQ), (unsigned)a->heads, (unsigned)a->B);
  int st;
  if (a->d <= 64) st = bias ? launch_attn<64, true>(tq, tk, tv, p, grid, smem_bytes, stream)
                            : launch_attn<64, false>(tq, tk, tv, p, grid, smem_bytes, stream);
  else if (a->d <= 128) st = bias ? launch_attn<128, true>(tq, tk, tv, p, grid, smem_bytes, stream)
                                  : launch_attn<128, false>(tq, tk, tv, p, grid, smem_bytes, stream);
  else st = bias ? launch_attn<192, true>(tq, tk, tv, p, grid, smem_bytes, stream)
                 : launch_attn<192, false>(tq, tk, tv, p, grid, smem_bytes, stream);
  if (st) return st;
  ea_count_launch();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : ea_cuda_fail(e, "ea_attention: after the kernel launch");
}
