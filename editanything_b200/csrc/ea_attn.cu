// ea_attn.cu — fused attention on wgmma (sm_90a): O = softmax(Q K^T * scale [+ bias]) V.
//
// Replaces the einsum -> softmax -> einsum of CrossAttention.forward
// (ldm/modules/attention.py:170-193; QK^T accumulated in fp32 like the reference's
// _ATTN_PRECISION="fp32" path) and SAM's windowed / global attention with decomposed relative
// position bias (SURVEY.md App. C).  The N x N logits never touch HBM.
//
// One CTA = one (batch, head) and a tile of 128 query rows; 384 threads = three warp-groups, one CTA per SM, launched
// at 168 registers per thread and re-divided by setmaxnreg (24 per producer thread, 240 per consumer thread):
//   producer (warp-group 2; one thread, the other producer warps exit): TMA of the Q tile once, then K/V tiles into a
//            `stages`-deep shared-memory ring with full / empty mbarriers.  Q and K are K-major SWIZZLE_128B boxes of
//            64 columns; V is ceil(d / 16) SWIZZLE_32B boxes of 16 columns, so the P V accumulator is DO = d rounded
//            up to an instantiated multiple of 16 (48, 64, 80, 160, 192) rather than to 64.  Columns past d (and keys
//            past Nkv) are TMA out-of-bounds zero fill: the tensor maps' inner extent is d.
//   consumers (warp-groups 0-1): warp-group g owns query rows 64g .. 64g+63.  Per 128-key tile j: S = Q K^T (64 fp32
//            registers per thread), [+ the SAM rel-pos bias in the BIAS kernels], missing keys -> -inf on a ragged last
//            tile only, online softmax with the running max / sum per row (a row's 128 logits sit on the 4 lanes of
//            a quad), P packed to 16 bit straight from the accumulator layout into the A fragments of O += P V
//            (DO / 2 registers per thread).  Final 1 / l normalisation and stores.
// ptxas still compiles every thread for the 168-register launch ceiling, so S over 128 keys fits next to O only up to
// DO = 80; the DO >= 160 kernels take each stage as two 64-key sub-tiles.
// Two overlaps keep the tensor cores busy while the softmax runs (FlashAttention-3, Shah et al. 2024, §3.1-3.2):
//   * within a warp-group (DO <= 80 without the bias, two or more stages), S_j = Q K_j^T and O += P_{j-1} V_{j-1} are
//     issued together and the softmax of S_j runs while P_{j-1} V_{j-1} is still in flight; the other kernels, and a
//     one-stage ring, run one MMA at a time per warp-group;
//   * between the warp-groups, named barriers 2 and 3 hand the right to issue wgmmas back and forth, so one
//     warp-group's MMAs run while the other one computes exponentials.
#include <stdlib.h>
#include "ea_common.cuh"
#include "ea_internal.h"

namespace ea {

static constexpr int AT_BQ = 128;
static constexpr int AT_BKV = 128;
static constexpr int AT_ATOM = 128 * 128;    // bytes of one 128-row x 64-half SWIZZLE_128B box (Q, K)
static constexpr int AT_VBOX = AT_BKV * 32;  // bytes of one 128-key x 16-half SWIZZLE_32B box (V)
static constexpr int AT_MAX_STAGES = 4;
static constexpr int AT_THREADS = 384;
static constexpr int AT_CONSUMER_WARPS = 8;
static constexpr int AT_PRODUCER_REGS = 24, AT_CONSUMER_REGS = 240;
static_assert(128 * AT_PRODUCER_REGS + 256 * AT_CONSUMER_REGS <= AT_THREADS * 168,
              "setmaxnreg.inc can only take what .dec released from the CTA's launch allocation");

struct AttnKParams {
  int Nq, Nkv, d, heads;
  int nd;      // ceil(d / 64) Q / K boxes along the head dim
  int ksteps;  // ceil(d / 16) MMA K-steps for Q K^T
  int stages;
  float scale_log2;
  ea_half* out;
  long long o_bs, o_ns;
  const float* rel_h;
  const float* rel_w;
  int rel_s;
};

template <int R>
__device__ __forceinline__ void wgmma_fence_regs_u32(uint32_t (&a)[R][4]) {
#pragma unroll
  for (int i = 0; i < R; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) asm volatile("" : "+r"(a[i][k])::"memory");
}

// Named barriers over the 256 consumer threads: 1 = both warp-groups, 2 + g = warp-group g may issue its wgmmas.
__device__ __forceinline__ void consumer_bar_sync(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void consumer_bar_arrive(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }

// DO: width of the P V accumulator (a multiple of 16, >= d; the columns past d are TMA zero fill)
template <int DO, bool BIAS>
__global__ void __launch_bounds__(AT_THREADS, 1)
ea_attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, const AttnKParams p) {
  constexpr int NV = DO / 16;   // V boxes per stage
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~uintptr_t(1023));
  // layout: Q[nd] | KV[stages][K nd | V NV] | rel_w rows (BIAS) | barriers
  const int k_bytes = p.nd * AT_ATOM;
  const int kv_stage_bytes = k_bytes + NV * AT_VBOX;
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + k_bytes;
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

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < AT_MAX_STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], AT_CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= AT_CONSUMER_WARPS) {
    setmaxnreg_dec<AT_PRODUCER_REGS>();
    if (threadIdx.x != AT_CONSUMER_WARPS * 32) return;
    // ============================ TMA producer ============================
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    pdl_wait();
    mbar_expect_tx(q_full, (uint32_t)k_bytes);
    for (int a = 0; a < p.nd; ++a) tma_load_4d(sQ + a * AT_ATOM, &tmQ, q_full, a * 64, head, qb * AT_BQ, b);
    int stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < n_tiles; ++j) {
      mbar_wait(&kv_empty[stage], phase ^ 1u);
      uint8_t* sK = sKV + stage * kv_stage_bytes;
      uint8_t* sV = sK + k_bytes;
      mbar_expect_tx(&kv_full[stage], (uint32_t)kv_stage_bytes);
      for (int a = 0; a < p.nd; ++a) tma_load_4d(sK + a * AT_ATOM, &tmK, &kv_full[stage], a * 64, head, j * AT_BKV, b);
#pragma unroll
      for (int c = 0; c < NV; ++c) tma_load_4d(sV + c * AT_VBOX, &tmV, &kv_full[stage], c * 16, head, j * AT_BKV, b);
      if (++stage == p.stages) { stage = 0; phase ^= 1u; }
    }
    return;
  }

  // ================================ consumers =================================
  setmaxnreg_inc<AT_CONSUMER_REGS>();
  pdl_wait();
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
    for (int idx = threadIdx.x; idx < AT_BQ * p.rel_s; idx += AT_CONSUMER_WARPS * 32) {
      const int row = idx / p.rel_s, i = idx - row * p.rel_s;
      const int q = qb * AT_BQ + row;
      rw_s[row * (p.rel_s + 1) + i] = q < p.Nq ? __ldg(p.rel_w + (bh * p.Nq + q) * p.rel_s + i) * LOG2E : 0.f;
    }
    rh_lo = p.rel_h + (bh * p.Nq + (q_lo < p.Nq ? q_lo : 0)) * p.rel_s;
    rh_hi = p.rel_h + (bh * p.Nq + (q_hi < p.Nq ? q_hi : 0)) * p.rel_s;
    consumer_bar_sync(1);
  }
  const uint64_t dQ0 = gmma_desc_k_sw128(smem_u32(sQ) + (uint32_t)(wg * 64 * 128), 1024);
  const uint64_t dK0 = gmma_desc_k_sw128(smem_u32(sKV), 1024);
  const uint64_t dV0 = gmma_desc_mn_sw32(smem_u32(sKV) + (uint32_t)k_bytes, AT_VBOX, 256);
  const uint32_t kv_stage16 = (uint32_t)kv_stage_bytes >> 4;
  // BIAS: the logits are scaled when the bias is added, so the softmax below sees scale 1
  const float sc = BIAS ? 1.f : p.scale_log2;
  const int my_bar = 2 + wg, other_bar = 2 + (wg ^ 1);

  // Keys per S sub-tile: the whole 128-key stage up to DO = 80; 64 at DO >= 160, where S over 128 keys next to O does
  // not fit: ptxas allocates every thread of a 384-thread CTA at most 168 registers, setmaxnreg.inc notwithstanding.
  constexpr int SN = DO <= 80 ? AT_BKV : 64;
  constexpr int SUB = AT_BKV / SN;   // sub-tiles per stage
  // S_j in flight next to P_{j-1} V_{j-1} needs both in registers: only without the bias terms does that fit
  constexpr bool PIPELINE = SN == AT_BKV && !BIAS;
  const int n_sub = (p.Nkv + SN - 1) / SN;
  const bool ragged = p.Nkv % SN != 0;

  float o[DO / 2];
#pragma unroll
  for (int i = 0; i < DO / 2; ++i) o[i] = 0.f;
  float s[SN / 2];
  uint32_t pa[SN / 16][4];                    // P as the A fragments of the K-steps (16 keys each) of P V
  float m_lo = -INFINITY, m_hi = -INFINITY;   // running max in the scaled log2 domain
  float l_lo = 0.f, l_hi = 0.f;               // this thread's share of the running sum
  float a_lo = 0.f, a_hi = 0.f;               // rescale factor of O for the latest sub-tile

  // Every wgmma issue is bracketed by mma_begin() ... mma_end(): warp-group 1 opens the sequence for warp-group 0 and
  // skips the arrive after its last issue, so the arrivals match the syncs.
  auto mma_begin = [&]() {
    consumer_bar_sync(my_bar);
    wgmma_fence();
  };
  auto mma_end = [&](bool last) {
    if (!(last && wg == 1)) consumer_bar_arrive(other_bar);
  };
  // S = Q K^T over keys SN h .. of stage st.  K-step ks sits at box (ks >> 2), +32 B * (ks & 3)
  auto issue_s = [&](int st, int h) {
    uint64_t dq = dQ0, dk = dK0 + (uint64_t)(st * kv_stage16 + h * ((SN * 128) >> 4));
    Wgmma<SN>::ss(s, dq, dk, 0u);
    for (int ks = 1; ks < p.ksteps; ++ks) {
      const uint32_t step = (ks & 3) ? 2u : (uint32_t)((AT_ATOM >> 4) - 6);
      dq += step;
      dk += step;
      Wgmma<SN>::ss(s, dq, dk, 1u);
    }
    wgmma_commit();
  };
  // O += P V ; V K-step kk = 16 key rows = +512 B of every 16-column box
  auto issue_pv = [&](int st, int h) {
    const uint64_t dv = dV0 + (uint64_t)(st * kv_stage16 + h * ((SN * 32) >> 4));
#pragma unroll
    for (int kk = 0; kk < SN / 16; ++kk) Wgmma<DO>::rs(o, pa[kk], dv + (uint64_t)(kk * ((16 * 32) >> 4)), 1u);
    wgmma_commit();
  };
  auto wait_pv = [&]() {
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    wgmma_fence_regs_u32(pa);
  };
  auto release = [&](int st) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);
  };
  // S of sub-tile t -> exponentials in place; updates m, l and sets the O rescale factors a_lo / a_hi
  auto softmax = [&](int t) {
    if (BIAS) {
#pragma unroll
      for (int i = 0; i < SN / 2; ++i) {
        const int key = t * SN + 8 * (i >> 2) + 2 * t4 + (i & 1);
        const bool hi = (i >> 1) & 1;
        const int kh = key / p.rel_s, kw = key - kh * p.rel_s;
        s[i] = fmaf(s[i], p.scale_log2,
                    rw_s[(rl + (hi ? 8 : 0)) * (p.rel_s + 1) + kw] + __ldg((hi ? rh_hi : rh_lo) + min(kh, p.rel_s - 1)) * LOG2E);
      }
    }
    if (ragged && t == n_sub - 1) {
      const int valid = p.Nkv - t * SN;   // keys of this sub-tile that exist (>= 1)
#pragma unroll
      for (int i = 0; i < SN / 2; ++i)
        if (8 * (i >> 2) + 2 * t4 + (i & 1) >= valid) s[i] = -INFINITY;
    }
    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int i = 0; i < SN / 2; i += 4) {
      mx_lo = fmaxf(mx_lo, fmaxf(s[i], s[i + 1]));
      mx_hi = fmaxf(mx_hi, fmaxf(s[i + 2], s[i + 3]));
    }
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
    // sc > 0, so the max of the scaled logits is the scaled max
    const float mn_lo = fmaxf(m_lo, mx_lo * sc), mn_hi = fmaxf(m_hi, mx_hi * sc);
    a_lo = mufu_ex2(m_lo - mn_lo);   // 0 on the first sub-tile
    a_hi = mufu_ex2(m_hi - mn_hi);
    m_lo = mn_lo;
    m_hi = mn_hi;
    float sum_lo = 0.f, sum_hi = 0.f;
#pragma unroll
    for (int i = 0; i < SN / 2; i += 4) {
      s[i] = mufu_ex2(fmaf(s[i], sc, -mn_lo));
      s[i + 1] = mufu_ex2(fmaf(s[i + 1], sc, -mn_lo));
      s[i + 2] = mufu_ex2(fmaf(s[i + 2], sc, -mn_hi));
      s[i + 3] = mufu_ex2(fmaf(s[i + 3], sc, -mn_hi));
      sum_lo += s[i] + s[i + 1];
      sum_hi += s[i + 2] + s[i + 3];
    }
    l_lo = fmaf(l_lo, a_lo, sum_lo);
    l_hi = fmaf(l_hi, a_hi, sum_hi);
  };
  auto rescale_and_pack = [&]() {
#pragma unroll
    for (int i = 0; i < DO / 2; ++i) o[i] *= ((i >> 1) & 1) ? a_hi : a_lo;
#pragma unroll
    for (int kk = 0; kk < SN / 16; ++kk)
#pragma unroll
      for (int h = 0; h < 4; ++h) pa[kk][h] = ea_pack2(s[8 * kk + 2 * h], s[8 * kk + 2 * h + 1]);
  };

  if (wg == 1) consumer_bar_arrive(2);
  mbar_wait(q_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  if (PIPELINE && p.stages > 1) {
    // S_j and P_{j-1} V_{j-1} in flight together; the softmax of S_j runs while P_{j-1} V_{j-1} does
    mbar_wait(&kv_full[0], 0);
    mma_begin();
    issue_s(0, 0);
    mma_end(false);
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    softmax(0);
    rescale_and_pack();
    for (int j = 1; j < n_sub; ++j) {
      const int prev = stage;
      if (++stage == p.stages) { stage = 0; phase ^= 1u; }
      mbar_wait(&kv_full[stage], phase);
      mma_begin();
      issue_s(stage, 0);
      issue_pv(prev, 0);
      mma_end(false);
      wgmma_wait<1>();
      wgmma_fence_regs(s);
      softmax(j);
      wait_pv();
      release(prev);
      rescale_and_pack();
    }
    mma_begin();
    issue_pv(stage, 0);
    mma_end(true);
    wait_pv();
  } else {
    // one MMA at a time per warp-group: the BIAS kernels, 64-key sub-tiles (DO >= 160), or a one-stage ring, where
    // tile j can only be loaded once P V_{j-1} has released the stage
    for (int t = 0; t < n_sub; ++t) {
      const int h = t % SUB;
      if (h == 0) mbar_wait(&kv_full[stage], phase);
      mma_begin();
      issue_s(stage, h);
      mma_end(false);
      wgmma_wait<0>();
      wgmma_fence_regs(s);
      softmax(t);
      rescale_and_pack();
      mma_begin();
      issue_pv(stage, h);
      mma_end(t == n_sub - 1);
      wait_pv();
      if (h == SUB - 1) {
        release(stage);
        if (++stage == p.stages) { stage = 0; phase ^= 1u; }
      }
    }
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

// ---------------------------------------------------------------------------------------------------------------
// Wide heads, 192 < d <= 512 (the VAE AttnBlock: one head of d = C = 512).  The kernel above cannot take them: a
// warp-group's O tile of 64 rows x 512 fp32 is 256 registers per thread, and Q for 128 rows x 512 halves plus one
// 128-key K and V tile is past the 227 KB of shared memory.  So:
//   * one CTA = one (batch, head) and 64 query rows: Q is 64 KB (nd SWIZZLE_128B boxes of 64 rows x 64 columns);
//   * 32-key K / V tiles, 32 KB each, in a ring of >= 2 stages (K: nd boxes of 32 rows; V: 32 SWIZZLE_32B boxes of
//     16 columns, always all of them, so the accumulator is 512 wide and columns past d are TMA zero fill);
//   * 256 threads = two warp-groups and no producer warp-group: thread 0 issues the TMA loads, refilling a stage
//     once all 8 warps have released it.  A ninth warp would put three warps on one SM sub-partition's 16K
//     registers and cap every thread at 168, and setmaxnreg does not lift what ptxas compiles for (see above); at
//     256 threads each thread may hold 255, enough for O (128), S (16) and P (8) without spills;
//   * both consumer warp-groups cover the same 64 rows, and warp-group g owns O columns 256 g .. 256 g + 255.  Each
//     computes S = Q K^T over all d columns itself and runs the online softmax on it, so P stays in registers as the
//     A operand of its m64n256k16 P V wgmmas, as in the kernel above.
// That costs 1.5x the minimum MMA work (Q K^T twice).  The alternative, splitting the Q K^T reduction over d between
// the warp-groups, would need the partial S tiles exchanged through shared memory and a barrier between the two
// warp-groups on every 32-key tile; duplicating S keeps the warp-groups independent and the kernel the same shape
// as the one above.  Both warp-groups compute bit-identical S, m and l, so the two halves of a row agree.
// Per warp-group S_j = Q K_j^T is issued together with O += P_{j-1} V_{j-1}, and the softmax of S_j runs while the
// P V wgmmas are in flight (the PIPELINE schedule of the kernel above).  No rel-pos bias.
static constexpr int AW_BQ = 64;
static constexpr int AW_BKV = 32;
static constexpr int AW_DO = 512;
static constexpr int AW_QBOX = AW_BQ * 128;    // bytes of one 64-row x 64-half SWIZZLE_128B box (Q)
static constexpr int AW_KBOX = AW_BKV * 128;   // bytes of one 32-row x 64-half SWIZZLE_128B box (K)
static constexpr int AW_VBOX = AW_BKV * 32;    // bytes of one 32-key x 16-half SWIZZLE_32B box (V)
static constexpr int AW_NV = AW_DO / 16;
static constexpr int AW_MAX_STAGES = 4;
static constexpr int AW_WARPS = 8;
static constexpr int AW_THREADS = AW_WARPS * 32;
static_assert(8 * AW_QBOX + 2 * (8 * AW_KBOX + AW_NV * AW_VBOX) <= 227 * 1024 - 1024 - 256,
              "d = 512 must get a ring of two stages: the pipelined loop waits for tile j before it frees tile j - 1");

__global__ void __launch_bounds__(AW_THREADS, 1)
ea_attn_wide_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const AttnKParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~uintptr_t(1023));
  // layout: Q[nd] | KV[stages][K nd | V AW_NV] | barriers
  const int q_bytes = p.nd * AW_QBOX;
  const int k_bytes = p.nd * AW_KBOX;
  const int kv_stage_bytes = k_bytes + AW_NV * AW_VBOX;
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + q_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + p.stages * kv_stage_bytes);
  uint64_t* q_full = bars;                       // [1]
  uint64_t* kv_full = bars + 1;                  // [AW_MAX_STAGES]
  uint64_t* kv_empty = kv_full + AW_MAX_STAGES;  // [AW_MAX_STAGES]

  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int qb = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int n_tiles = (p.Nkv + AW_BKV - 1) / AW_BKV;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < AW_MAX_STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], AW_WARPS);
    }
    fence_mbar_init();
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  __syncthreads();

  // K and V of tile t into its stage t % stages (thread 0)
  auto load_tile = [&](int t) {
    const int st = t % p.stages;
    uint8_t* sK = sKV + st * kv_stage_bytes;
    uint8_t* sV = sK + k_bytes;
    mbar_expect_tx(&kv_full[st], (uint32_t)kv_stage_bytes);
    for (int a = 0; a < p.nd; ++a) tma_load_4d(sK + a * AW_KBOX, &tmK, &kv_full[st], a * 64, head, t * AW_BKV, b);
    for (int c = 0; c < AW_NV; ++c) tma_load_4d(sV + c * AW_VBOX, &tmV, &kv_full[st], c * 16, head, t * AW_BKV, b);
  };
  pdl_wait();
  if (threadIdx.x == 0) {
    mbar_expect_tx(q_full, (uint32_t)q_bytes);
    for (int a = 0; a < p.nd; ++a) tma_load_4d(sQ + a * AW_QBOX, &tmQ, q_full, a * 64, head, qb * AW_BQ, b);
    for (int t = 0; t < p.stages; ++t) load_tile(t);
  }
  __syncwarp();
  const int wg = warp >> 2, wq = warp & 3;
  const int g = lane >> 2, t4 = lane & 3;
  // accumulator layout (ea_wgmma.cuh): rows wq * 16 + g (i % 4 < 2) and + 8 (i % 4 >= 2) of the CTA's 64
  const int q_lo = qb * AW_BQ + wq * 16 + g, q_hi = q_lo + 8;
  const uint64_t dQ0 = gmma_desc_k_sw128(smem_u32(sQ), 1024);
  const uint64_t dK0 = gmma_desc_k_sw128(smem_u32(sKV), 1024);
  // warp-group g multiplies by V columns 256 g .. : its first V box is 16 g
  const uint64_t dV0 = gmma_desc_mn_sw32(smem_u32(sKV) + (uint32_t)(k_bytes + wg * 16 * AW_VBOX), AW_VBOX, 256);
  const uint32_t kv_stage16 = (uint32_t)kv_stage_bytes >> 4;
  const float sc = p.scale_log2;
  const bool ragged = p.Nkv % AW_BKV != 0;

  float o[AW_DO / 4];
#pragma unroll
  for (int i = 0; i < AW_DO / 4; ++i) o[i] = 0.f;
  float s[AW_BKV / 2];
  uint32_t pa[AW_BKV / 16][4];
  float m_lo = -INFINITY, m_hi = -INFINITY;   // running max in the scaled log2 domain
  float l_lo = 0.f, l_hi = 0.f;               // this thread's share of the running sum
  float a_lo = 0.f, a_hi = 0.f;               // rescale factor of O for the latest tile

  // S = Q K^T over the keys of stage st.  K-step ks sits at box (ks >> 2), +32 B * (ks & 3)
  auto issue_s = [&](int st) {
    uint64_t dq = dQ0, dk = dK0 + (uint64_t)(st * kv_stage16);
    Wgmma<AW_BKV>::ss(s, dq, dk, 0u);
    for (int ks = 1; ks < p.ksteps; ++ks) {
      const bool next_box = (ks & 3) == 0;
      dq += next_box ? (uint64_t)((AW_QBOX >> 4) - 6) : 2u;
      dk += next_box ? (uint64_t)((AW_KBOX >> 4) - 6) : 2u;
      Wgmma<AW_BKV>::ss(s, dq, dk, 1u);
    }
    wgmma_commit();
  };
  // O += P V ; V K-step kk = 16 key rows = +512 B of every 16-column box
  auto issue_pv = [&](int st) {
    const uint64_t dv = dV0 + (uint64_t)(st * kv_stage16);
#pragma unroll
    for (int kk = 0; kk < AW_BKV / 16; ++kk)
      Wgmma<AW_DO / 2>::rs(o, pa[kk], dv + (uint64_t)(kk * ((16 * 32) >> 4)), 1u);
    wgmma_commit();
  };
  auto wait_pv = [&]() {
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    wgmma_fence_regs_u32(pa);
  };
  auto release = [&](int st) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);
  };
  // S of tile t -> exponentials in place; updates m, l and sets the O rescale factors a_lo / a_hi
  auto softmax = [&](int t) {
    if (ragged && t == n_tiles - 1) {
      const int valid = p.Nkv - t * AW_BKV;   // keys of this tile that exist (>= 1)
#pragma unroll
      for (int i = 0; i < AW_BKV / 2; ++i)
        if (8 * (i >> 2) + 2 * t4 + (i & 1) >= valid) s[i] = -INFINITY;
    }
    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int i = 0; i < AW_BKV / 2; i += 4) {
      mx_lo = fmaxf(mx_lo, fmaxf(s[i], s[i + 1]));
      mx_hi = fmaxf(mx_hi, fmaxf(s[i + 2], s[i + 3]));
    }
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
    mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
    mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
    // sc > 0, so the max of the scaled logits is the scaled max
    const float mn_lo = fmaxf(m_lo, mx_lo * sc), mn_hi = fmaxf(m_hi, mx_hi * sc);
    a_lo = mufu_ex2(m_lo - mn_lo);   // 0 on the first tile
    a_hi = mufu_ex2(m_hi - mn_hi);
    m_lo = mn_lo;
    m_hi = mn_hi;
    float sum_lo = 0.f, sum_hi = 0.f;
#pragma unroll
    for (int i = 0; i < AW_BKV / 2; i += 4) {
      s[i] = mufu_ex2(fmaf(s[i], sc, -mn_lo));
      s[i + 1] = mufu_ex2(fmaf(s[i + 1], sc, -mn_lo));
      s[i + 2] = mufu_ex2(fmaf(s[i + 2], sc, -mn_hi));
      s[i + 3] = mufu_ex2(fmaf(s[i + 3], sc, -mn_hi));
      sum_lo += s[i] + s[i + 1];
      sum_hi += s[i + 2] + s[i + 3];
    }
    l_lo = fmaf(l_lo, a_lo, sum_lo);
    l_hi = fmaf(l_hi, a_hi, sum_hi);
  };
  auto rescale_and_pack = [&]() {
#pragma unroll
    for (int i = 0; i < AW_DO / 4; ++i) o[i] *= ((i >> 1) & 1) ? a_hi : a_lo;
#pragma unroll
    for (int kk = 0; kk < AW_BKV / 16; ++kk)
#pragma unroll
      for (int h = 0; h < 4; ++h) pa[kk][h] = ea_pack2(s[8 * kk + 2 * h], s[8 * kk + 2 * h + 1]);
  };

  mbar_wait(q_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  mbar_wait(&kv_full[0], 0);
  wgmma_fence();
  issue_s(0);
  wgmma_wait<0>();
  wgmma_fence_regs(s);
  softmax(0);
  rescale_and_pack();
  for (int j = 1; j < n_tiles; ++j) {
    const int prev = stage;
    if (++stage == p.stages) { stage = 0; phase ^= 1u; }
    mbar_wait(&kv_full[stage], phase);
    wgmma_fence();
    issue_s(stage);
    issue_pv(prev);
    wgmma_wait<1>();
    wgmma_fence_regs(s);
    softmax(j);
    wait_pv();
    release(prev);
    // tile j - 1 + stages goes where tile j - 1 was, once every warp has released it (the empty barrier's
    // ((j - 1) / stages)-th phase)
    if (threadIdx.x == 0 && j - 1 + p.stages < n_tiles) {
      mbar_wait(&kv_empty[prev], (uint32_t)(((j - 1) / p.stages) & 1));
      load_tile(j - 1 + p.stages);
    }
    __syncwarp();
    rescale_and_pack();
  }
  wgmma_fence();
  issue_pv(stage);
  wait_pv();

  // ---- epilogue: O / l
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
  l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
  l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
  const float inv_lo = 1.f / l_lo, inv_hi = 1.f / l_hi;
  ea_half* orow_lo = p.out + (long long)b * p.o_bs + (long long)q_lo * p.o_ns + (long long)head * p.d;
  ea_half* orow_hi = orow_lo + 8 * p.o_ns;
#pragma unroll
  for (int i = 0; i < AW_DO / 4; i += 4) {
    const int col = wg * (AW_DO / 2) + 8 * (i >> 2) + 2 * t4;
    if (col < p.d) {
      if (q_lo < p.Nq) *reinterpret_cast<uint32_t*>(orow_lo + col) = ea_pack2(o[i] * inv_lo, o[i + 1] * inv_lo);
      if (q_hi < p.Nq) *reinterpret_cast<uint32_t*>(orow_hi + col) = ea_pack2(o[i + 2] * inv_hi, o[i + 3] * inv_hi);
    }
  }
}

// [B, N, heads, d] with strides (bs, ns, d) elements; boxes of `box_cols` head-dim columns x `box_rows` rows
static int encode_qkv(CUtensorMap* m, const void* base, int d, int heads, int N, int B,
                      long long ns, long long bs, int box_cols, CUtensorMapSwizzle swizzle, int box_rows = 128) {
  cuuint64_t dims[4] = {(cuuint64_t)d, (cuuint64_t)heads, (cuuint64_t)N, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)d * 2, (cuuint64_t)ns * 2, (cuuint64_t)bs * 2};
  cuuint32_t box[4] = {(cuuint32_t)box_cols, 1, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = ea_tmap_encode()(m, EA_TMAP_DTYPE, 4, const_cast<void*>(base), dims, strides, box,
                                estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
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

template <int DO>
static int launch_attn_width(bool bias, const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                             const AttnKParams& p, dim3 grid, int smem_bytes, cudaStream_t stream) {
  return bias ? launch_attn<DO, true>(tq, tk, tv, p, grid, smem_bytes, stream)
              : launch_attn<DO, false>(tq, tk, tv, p, grid, smem_bytes, stream);
}

// P V accumulator width for head dim d: the head dims the UNets and SAM run (40, 64, 80, 160) rounded up to 16,
// and 192 for the rest of the ABI's range
static int attn_pv_width(int d) {
  return d <= 48 ? 48 : d <= 64 ? 64 : d <= 80 ? 80 : d <= 160 ? 160 : 192;
}

// 192 < d <= 512, no bias
static int launch_attn_wide(const ea_attn_args* a, AttnKParams& p, cudaStream_t stream) {
  const int budget = 227 * 1024 - 1024 - 256;
  const int q_bytes = p.nd * AW_QBOX;
  const int stage_bytes = p.nd * AW_KBOX + AW_NV * AW_VBOX;
  int stages = (budget - q_bytes) / stage_bytes;
  if (stages > AW_MAX_STAGES) stages = AW_MAX_STAGES;
  const int n_tiles = (a->Nkv + AW_BKV - 1) / AW_BKV;
  if (stages > n_tiles) stages = n_tiles;
  p.stages = stages;

  CUtensorMap tq, tk, tv;
  if (encode_qkv(&tq, a->q, a->d, a->heads, a->Nq, a->B, a->q_ns, a->q_bs, 64, CU_TENSOR_MAP_SWIZZLE_128B, AW_BQ))
    return EA_ERR_TMAP;
  if (encode_qkv(&tk, a->k, a->d, a->heads, a->Nkv, a->B, a->k_ns, a->k_bs, 64, CU_TENSOR_MAP_SWIZZLE_128B, AW_BKV))
    return EA_ERR_TMAP;
  if (encode_qkv(&tv, a->v, a->d, a->heads, a->Nkv, a->B, a->v_ns, a->v_bs, 16, CU_TENSOR_MAP_SWIZZLE_32B, AW_BKV))
    return EA_ERR_TMAP;

  const int smem_bytes = q_bytes + stages * stage_bytes + (1 + 2 * AW_MAX_STAGES) * 8 + 1024;
  static int max_set_dev[EA_MAX_DEV];
  int& max_set = max_set_dev[ea_dev()];
  if (smem_bytes > max_set) {
    const cudaError_t e = cudaFuncSetAttribute(ea_attn_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               smem_bytes);
    if (e != cudaSuccess) return ea_cuda_fail(e, "ea_attention: cudaFuncSetAttribute(MaxDynamicSharedMemorySize)");
    max_set = smem_bytes;
  }
  dim3 grid((unsigned)((a->Nq + AW_BQ - 1) / AW_BQ), (unsigned)a->heads, (unsigned)a->B);
  const cudaError_t e = ea_launch(ea_attn_wide_kernel, grid, dim3(AW_THREADS), (size_t)smem_bytes, stream,
                                  tq, tk, tv, p);
  return e == cudaSuccess ? 0 : ea_cuda_fail(e, "ea_attention: kernel launch");
}

}  // namespace ea

using namespace ea;

extern "C" int ea_attention(const ea_attn_args* a, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!a || !a->q || !a->k || !a->v || !a->out) return EA_ERR_ARG;
  if (a->d % 8 != 0 || a->d < 8 || a->d > AW_DO) return EA_ERR_SHAPE;
  if (a->Nq <= 0 || a->Nkv <= 0 || a->B <= 0 || a->heads <= 0) return EA_ERR_SHAPE;
  if (a->q_ns % 8 || a->k_ns % 8 || a->v_ns % 8 || a->q_bs % 8 || a->k_bs % 8 || a->v_bs % 8 ||
      a->o_ns % 8 || a->o_bs % 8)
    return EA_ERR_SHAPE;
  if (!(a->scale > 0.f) || isinf(a->scale)) return EA_ERR_ARG;   // the kernel scales the row max, not every logit
  if ((a->rel_h != nullptr) != (a->rel_w != nullptr)) return EA_ERR_ARG;
  if (a->rel_h && a->rel_s <= 0) return EA_ERR_ARG;
  // bias[q, kk] is defined for kk < rel_s^2 only (the kernel clamps kk / rel_s, which masked keys need)
  if (a->rel_h && (long long)a->rel_s * a->rel_s < a->Nkv) return EA_ERR_SHAPE;

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
  if (a->d > 192) {
    if (bias) return EA_ERR_SHAPE;   // the wide kernel has no rel-pos bias terms
    const int st = launch_attn_wide(a, p, stream);
    if (st) return st;
    ea_count_launch();
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : ea_cuda_fail(e, "ea_attention: after the kernel launch");
  }
  const int dv = attn_pv_width(a->d);
  const int budget = 227 * 1024 - 1024 - 256;
  // 64-bit: rel_w rows of a huge rel_s must not wrap around and pass as a small shared-memory footprint
  const long long bias_ll = bias ? ((AT_BQ * ((long long)a->rel_s + 1) + 3) & ~3LL) * 4 : 0;
  const int stage_bytes = p.nd * AT_ATOM + dv / 16 * AT_VBOX;
  const long long stages_ll = (budget - p.nd * AT_ATOM - bias_ll) / stage_bytes;
  if (stages_ll < 1) return EA_ERR_SHAPE;
  const int bias_bytes = (int)bias_ll;
  int stages = stages_ll > AT_MAX_STAGES ? AT_MAX_STAGES : (int)stages_ll;
  const int n_tiles = (a->Nkv + AT_BKV - 1) / AT_BKV;
  if (stages > n_tiles) stages = n_tiles;
  p.stages = stages;

  CUtensorMap tq, tk, tv;
  if (encode_qkv(&tq, a->q, a->d, a->heads, a->Nq, a->B, a->q_ns, a->q_bs, 64, CU_TENSOR_MAP_SWIZZLE_128B))
    return EA_ERR_TMAP;
  if (encode_qkv(&tk, a->k, a->d, a->heads, a->Nkv, a->B, a->k_ns, a->k_bs, 64, CU_TENSOR_MAP_SWIZZLE_128B))
    return EA_ERR_TMAP;
  if (encode_qkv(&tv, a->v, a->d, a->heads, a->Nkv, a->B, a->v_ns, a->v_bs, 16, CU_TENSOR_MAP_SWIZZLE_32B))
    return EA_ERR_TMAP;

  const int smem_bytes = p.nd * AT_ATOM + stages * stage_bytes + bias_bytes + (1 + 2 * AT_MAX_STAGES) * 8 + 1024;
  dim3 grid((unsigned)((a->Nq + AT_BQ - 1) / AT_BQ), (unsigned)a->heads, (unsigned)a->B);
  int st;
  switch (dv) {
    case 48: st = launch_attn_width<48>(bias, tq, tk, tv, p, grid, smem_bytes, stream); break;
    case 64: st = launch_attn_width<64>(bias, tq, tk, tv, p, grid, smem_bytes, stream); break;
    case 80: st = launch_attn_width<80>(bias, tq, tk, tv, p, grid, smem_bytes, stream); break;
    case 160: st = launch_attn_width<160>(bias, tq, tk, tv, p, grid, smem_bytes, stream); break;
    default: st = launch_attn_width<192>(bias, tq, tk, tv, p, grid, smem_bytes, stream); break;
  }
  if (st) return st;
  ea_count_launch();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : ea_cuda_fail(e, "ea_attention: after the kernel launch");
}
