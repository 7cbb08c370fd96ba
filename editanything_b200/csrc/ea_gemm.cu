// ea_gemm.cu — the wgmma GEMM / implicit-GEMM convolution kernel (sm_90a).
//
// One kernel serves every dense contraction of the UNet / ControlNet / SAM hot path
// (SURVEY.md §8a rows R1, R7, R9-R12):
//   * Linear layers and 1x1 convolutions            (mode LINEAR)
//   * 3x3 stride-1 pad-1 convolutions on NHWC data  (mode CONV_S1), optionally with the
//     ResBlock's 1x1 skip convolution folded in as extra K-blocks (openaimodel.py:233-240,274)
//   * 3x3 stride-2 pad-1 convolutions (Downsample, openaimodel.py:133-159) (mode CONV_S2)
//
// ea_gemm_kernel<BN, NG, RP>: a CTA computes RP vertically adjacent 128 x BN output tiles (row tiles RP t ..
// RP t + RP - 1, "sub-tiles") that share every W stage, one work item per CTA, or walking a list of items
// (persistent launches: one CTA per SM).  RP = 2 loads 2 x 16 KB of A and one W box per 64-deep K-block for twice the
// MMA work of RP = 1 (85 instead of 64 FLOP per byte of L2 traffic at BN = 128) and pays the per-item fixed costs once
// per two tiles.  Roles (384 threads = three warp-groups, one CTA per SM, launched at 168 registers per thread;
// setmaxnreg moves registers from the producer warp-group, 56 per thread, to the consumers, 224 per thread):
//   TMA producer (warp-group 2; warp 8 lane 0 issues TMA, lanes 2-31 of warp 8 walk the L2 prefetch hint, warps
//                  9-11 exit): the A box of every valid sub-tile (128 rows x 64 halves, SWIZZLE_128B) and the W box
//                  (BN x 64) into a `stages`-deep shared-memory ring, mbarrier-signalled.  For convolutions the A box
//                  of filter tap (kh,kw) is a 4-D box {64ch, bw, bh, bn} of the NHWC tensor shifted by (kh-1, kw-1);
//                  the zero padding is TMA out-of-bounds fill, no im2col buffer exists.  W-operand loads carry an L2
//                  evict-first hint (see gemm_fill_group).
//   consumers    (warp-groups 0-1): per stage, RP = 1: warp-group g issues wgmma m64nBNk16 x4 for tile rows
//                  64g .. 64g+63; RP = 2: warp-group g owns sub-tile g and issues two m64nBNk16 x4 (its rows 0-63 and
//                  64-127), BN accumulator registers per thread at most (BN <= 128).  Stages are released as soon as
//                  the next one's MMAs are in flight.  The finished accumulators are staged row-major in shared memory
//                  (over the drained ring) and the same 256 threads run the fused epilogue with one thread per
//                  sub-tile row: RP = 1 with the two warp-groups on alternating 64-column groups of the one tile,
//                  RP = 2 with warp-group g over all BN columns of sub-tile g.  Epilogue: bias / time-embedding row
//                  vector / LayerNorm fold / SiLU|GELU|GEGLU / scale / residual add / accumulate-into-destination
//                  (ControlNet zero-conv residual, cldm/cldm.py:34-41) / dual store, rows written as coalesced
//                  128-byte pieces through shared memory.
#include "ea_common.cuh"
#include "ea_internal.h"

namespace ea {

static constexpr int BM = 128;
static constexpr int BK = 64;
// Warp roles: consumer warps 0-7 (warp-groups 0-1), producer warp-group 2 (warps 8-11).  A CTA is launched with
// 384 x 168 registers (__launch_bounds__(384, 1)); setmaxnreg then re-divides exactly that pool: 224 per consumer
// thread, which holds the RP = 2 accumulator at BN = 128 (2 x 64 per thread) without spills, and 56 per producer
// thread (the grouped two-sub-tile convolution producer spills at 40).
static constexpr int GEMM_THREADS = 384;
static constexpr int W_TMA = 8;
static constexpr int EPI_WARPS = 8, EPI_THREADS = 256;
static constexpr int PRODUCER_REGS = 56, CONSUMER_REGS = 224;
static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= GEMM_THREADS * 168,
              "setmaxnreg.inc can only take what .dec released from the CTA's launch allocation");
// Shared memory: the stage ring (RP A boxes + one W box per stage), which after an item's last MMA also holds the
// staged fp32 accumulators ([RP * BM][BN + 4]: the pad keeps the row-per-thread reads conflict-free) and 2 x 4 KB of
// store / residual staging per consumer warp; then the barriers and the per-column vectors.
static constexpr int GEMM_SMEM_RING = 216 * 1024;
__host__ __device__ constexpr int gemm_stage_bytes(int bn, int rp) { return rp * BM * BK * 2 + bn * BK * 2; }
__host__ __device__ constexpr int gemm_epi_bytes(int bn, int rp) {
  return rp * BM * (bn + 4) * 4 + 2 * 4096 * EPI_WARPS;
}
__host__ __device__ constexpr int gemm_region_bytes(int bn, int stages, int rp) {
  return stages * gemm_stage_bytes(bn, rp) > gemm_epi_bytes(bn, rp) ? stages * gemm_stage_bytes(bn, rp)
                                                                    : gemm_epi_bytes(bn, rp);
}
static_assert(4 * gemm_stage_bytes(128, 2) <= GEMM_SMEM_RING, "RP = 2, BN = 128: four 48 KB stages fill the ring");
static_assert(gemm_epi_bytes(128, 2) <= GEMM_SMEM_RING, "the staged accumulators and the store staging fit the ring");
// per-column epilogue vectors: [2 item parities][RP sub-tiles][2][256] fp32
__host__ __device__ constexpr int gemm_cb_bytes(int rp) { return 2 * rp * 2 * 256 * 4; }

struct GemmKParams {
  int M, N;
  int mode;
  int nkb_main;   // K-blocks from the main A source
  int nkb_extra;  // K-blocks from the extra (1x1 skip) A source
  int cin_blocks; // Cin / 64 (conv): K-blocks per filter tap
  int BN, stages;
  // conv geometry (output space)
  int H, W, Bsz;
  int bw, bh, bn;
  int tiles_w, tiles_h;
  // epilogue
  const float* bias;
  const float* rowvec;
  int rows_per_batch;
  int rowvec_ld;
  const ea_half* residual;
  long long ldr;
  ea_half* out;
  long long ldo;
  ea_half* out2;
  long long ldo2;
  float* out_f32;  // optional fp32 output (same ldo) instead of half
  int act;
  float out_scale;
  int accumulate;
  // split-K: blockIdx.z = split index; partial tiles go through `ws`, arrival counters in `cnt`
  int splits;
  int kb_per_split;
  float* ws;   // [items][splits][RP * 128][BN] fp32
  int* cnt;    // [items][2]: arrived, done (zero between launches)
  // LayerNorm fold (see ea_gemm_args): producer side / consumer side
  float2* rowstats_out;     // [N/32][M] (sum, M2 about the chunk mean) of the stored values per 32-column chunk
  const float2* ln_stats;   // [ln_parts][M] partials of this GEMM's A rows
  const float* ln_g;        // [N]
  int ln_parts;
  float ln_inv_c, ln_eps;
  const float* row_scale;   // [M] fp32 per-row output factor (general / split-K epilogues only) or null
  const char* pf[EA_GEMM_MAX_PREFETCH];   // L2 prefetch hints (a later launch's weights) or null; pf_ctas CTAs share each range
  long long pf_bytes[EA_GEMM_MAX_PREFETCH];
  int pf_ctas;
  unsigned long long b_policy;   // L2 eviction hint of the W operand's TMA loads (0 = none)
};

// One launch can run up to GEMM_MAX_GROUPS independent problems of the SAME shape and launch plan (ea_gemm_grouped):
// the UNet encoder and the ControlNets are the same network with different weights reading the same latent
// (cldm/cldm.py:22-45,284-305), so every one of their layers is one grouped launch.  Each group has its own tensor
// maps and parameter block (any pointers), selected by blockIdx.z / splits (tile index / tiles for the persistent
// kernel); with NG = 1 the selection is a compile-time constant and the code is the ungrouped kernel.
static constexpr int GEMM_MAX_GROUPS = 3;
struct GemmGroup {
  CUtensorMap tmA0, tmA1, tmA2, tmA3, tmAx, tmB;
  GemmKParams p;
};
template <int NG>
struct GemmLaunch {
  GemmGroup g[NG];
};

__device__ __forceinline__ void tile_origin(const GemmKParams& p, int tm, int& n0, int& h0,
                                            int& w0) {
  // tiles enumerate (image block, tile row, tile col); an image block is bn images
  int per_blk = p.tiles_w * p.tiles_h;
  int nb = tm / per_blk;
  int r = tm - nb * per_blk;
  int th = r / p.tiles_w;
  n0 = nb * p.bn;
  h0 = th * p.bh;
  w0 = (r - th * p.tiles_w) * p.bw;
}

// Whether row tile tm holds any output row: the second sub-tile of the last RP = 2 item lies past the problem when the
// number of row tiles is odd (its loads and stores are skipped).
__device__ __forceinline__ bool tile_valid(const GemmKParams& p, int tm) {
  if (p.mode == EA_GEMM_LINEAR) return (long long)tm * BM < p.M;
  return tm / (p.tiles_w * p.tiles_h) * p.bn < p.Bsz;
}

struct RowInfo {
  long long m;   // global output row
  bool ok;
  int batch;
};

__device__ __forceinline__ RowInfo row_info(const GemmKParams& p, int tm, int r) {
  RowInfo ri;
  if (p.mode == EA_GEMM_LINEAR) {
    ri.m = (long long)tm * BM + r;
    ri.ok = ri.m < p.M;
    ri.batch = p.rows_per_batch > 0 ? (int)(ri.m / p.rows_per_batch) : 0;
  } else {
    int n0, h0, w0;
    tile_origin(p, tm, n0, h0, w0);
    int dn = r / (p.bw * p.bh);
    int rr = r - dn * (p.bw * p.bh);
    int dh = rr / p.bw;
    int dw = rr - dh * p.bw;
    int n = n0 + dn, h = h0 + dh, w = w0 + dw;
    ri.ok = (n < p.Bsz) && (h < p.H) && (w < p.W);
    ri.m = ((long long)n * p.H + h) * p.W + w;
    ri.batch = n;
  }
  return ri;
}

// named barrier over the 256 consumer threads (warps 0-7); barrier 0 is __syncthreads
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// LayerNorm fold, consumer side (ln_row_stats below): one row's mean / rstd from the producer's per-32-column partial
// (sum, M2) pairs.  The loads of a batch of 16 partials are all issued before the first merge, so they are in flight
// together instead of one dependent L2 round trip per partial (10 for C = 320, 40 for C = 1280).  The merges keep
// their fixed order, so the result stays deterministic.
// L2 prefetch of a later launch's weights (ea_gemm_args.prefetch): lanes `lane0 .. 31` of one warp in each of the first
// pf_ctas CTAs walk the range line by line.  Issued before the dependency wait - weights are never produced by a
// predecessor kernel - so HBM works on the next layer while this one computes from L2.
__device__ __forceinline__ void l2_prefetch_hint(const GemmKParams& p, int cta, int lane, int lane0) {
  if (cta >= p.pf_ctas || lane < lane0) return;
  // One 128-byte line per instruction through the load/store path (prefetch.global.L2), not cp.async.bulk.prefetch:
  // bulk prefetches queue in the SM's TMA unit in front of the launch's own operand loads.
  const int nl = 32 - lane0;
#pragma unroll 1
  for (int i = 0; i < EA_GEMM_MAX_PREFETCH; ++i) {
    if (p.pf[i] == nullptr) continue;
    const long long nlines = p.pf_bytes[i] >> 7;
    const char* base = p.pf[i];
#pragma unroll 4
    for (long long c = (long long)cta * nl + (lane - lane0); c < nlines; c += (long long)p.pf_ctas * nl)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(base + (c << 7)));
  }
}

__device__ __forceinline__ void ln_row_stats(const GemmKParams& p, long long m, float& ln_r, float& ln_nm) {
  // Chunk j has mean m_j = s_j / 32 and M2_j about it, so over the P = ln_parts chunks
  //   mean = m_0 + sum d_j / P,  M2 = sum M2_j + 32 (sum d_j^2 - (sum d_j)^2 / P),  d_j = m_j - m_0.
  // Shifting by the first chunk's mean keeps every term on the scale of the spread, whatever |mean| / std, and the
  // three sums are independent add chains (no divisions in the loop).
  float m0 = 0.f, d1 = 0.f, d2 = 0.f, s2 = 0.f;
  const float2* base = p.ln_stats + m;
  for (int j0 = 0; j0 < p.ln_parts; j0 += 16) {
    float2 v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u)
      v[u] = (j0 + u < p.ln_parts) ? __ldcg(base + (size_t)(j0 + u) * p.M) : make_float2(0.f, 0.f);
    if (j0 == 0) m0 = v[0].x * (1.f / 32.f);
    // the slots past ln_parts are zeroed by a factor, not skipped by a branch: a branch per slot lets the compiler
    // move each load next to its use, one dependent L2 round trip per partial again
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const float d = fmaf(v[u].x, 1.f / 32.f, -m0) * (j0 + u < p.ln_parts ? 1.f : 0.f);
      d1 += d;
      d2 = fmaf(d, d, d2);
      s2 += v[u].y;
    }
  }
  const float ip = 32.f * p.ln_inv_c;   // 1 / ln_parts
  const float m2 = fmaf(32.f, fmaxf(fmaf(-d1 * ip, d1, d2), 0.f), s2);
  ln_r = rsqrtf(m2 * p.ln_inv_c + p.ln_eps);
  ln_nm = -ln_r * fmaf(d1, ip, m0);
}

// Out-of-line activation for the rarely taken paths (general / split-K epilogues, SiLU): one copy of
// the code instead of 32 inlined ones per site keeps the kernel image small (instruction cache).
__device__ __noinline__ float act_call(float x, int act) {
  return act == EA_ACT_SILU ? silu_f(x) : gelu_erf_f(x);
}

// Coalesced tile stores.  A thread owns one accumulator row, so a direct store instruction would touch 32
// different rows (32 half-written sectors per instruction).  Instead every epilogue warp transposes its
// 32 rows x 64 columns through a private 4 KB staging block in shared memory, XOR-swizzled in 16-byte pieces,
// and writes each row's 128 bytes with 8 consecutive lanes.
__device__ __forceinline__ void stage_put32(uint4* stg, int lane, int half, const uint4 (&o)[4]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) stg[lane * 8 + ((half * 4 + q) ^ (lane & 7))] = o[q];
}
__device__ __forceinline__ void stage_flush(const uint4* stg, int lane, ea_half* out, long long ldo,
                                            ea_half* out2, long long ldo2, long long m_mine, bool ok_mine,
                                            int col0, int pieces, int n_limit, long long lin_m0, int M) {
  __syncwarp();
  // Straight-line on purpose: the eight 16-byte pieces of a lane are loaded from the staging block first (8 LDS in
  // flight) and stored with addresses advanced by a constant row stride (a rolled loop spends its instructions on
  // 64-bit multiplies, shuffle-or-linear branches and reconvergence barriers per 16-byte store).
  const int piece = lane & 7, rsub = lane >> 3;
  const int col = col0 + piece * 8;
  const bool col_ok = piece < pieces && col < n_limit;
  uint4 val[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int row = i * 4 + rsub;
    val[i] = stg[row * 8 + (piece ^ (row & 7))];
  }
  if (lin_m0 >= 0) {   // linear GEMM: the warp's rows are consecutive
    const long long m0 = lin_m0 + rsub;
    ea_half* ptr = out + m0 * ldo + col;
    ea_half* ptr2 = out2 ? out2 + m0 * ldo2 + col : nullptr;
    const long long step = 4 * ldo, step2 = 4 * ldo2;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (col_ok && m0 + 4 * i < M) {
        *reinterpret_cast<uint4*>(ptr) = val[i];
        if (ptr2) *reinterpret_cast<uint4*>(ptr2) = val[i];
      }
      ptr += step;
      if (ptr2) ptr2 += step2;
    }
  } else {             // convolution tiles: a row's pixel comes from the lane that owns it
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int row = i * 4 + rsub;
      const long long m_r = __shfl_sync(0xffffffffu, m_mine, row);
      const int ok_r = __shfl_sync(0xffffffffu, (int)ok_mine, row);
      if (ok_r && col_ok) {
        *reinterpret_cast<uint4*>(out + m_r * ldo + col) = val[i];
        if (out2) *reinterpret_cast<uint4*>(out2 + m_r * ldo2 + col) = val[i];
      }
    }
  }
  __syncwarp();
}

// The same for a 32-column group (64 bytes per row): four lanes per row, eight rows per pass, four passes - the 64-column
// mapping would leave half of the lanes idle for twice as many passes (the GEGLU epilogue of the 8-warp persistent
// kernel flushes 32 output columns per warp-group chunk).  Linear GEMMs only.
__device__ __forceinline__ void stage_flush32(const uint4* stg, int lane, ea_half* out, long long ldo, int col0,
                                              int n_limit, long long lin_m0, int M) {
  __syncwarp();
  const int piece = lane & 3, rsub = lane >> 2;
  const int col = col0 + piece * 8;
  const bool col_ok = col < n_limit;
  uint4 val[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = i * 8 + rsub;
    val[i] = stg[row * 8 + (piece ^ (row & 7))];
  }
  const long long m0 = lin_m0 + rsub;
  ea_half* ptr = out + m0 * ldo + col;
  const long long step = 8 * ldo;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (col_ok && m0 + 8 * i < M) *reinterpret_cast<uint4*>(ptr) = val[i];
    ptr += step;
  }
  __syncwarp();
}

// Coalesced load of a 32-row x 64-column group of the residual: lane -> (row 4i + lane/8, 16-byte piece
// lane%8), so 8 consecutive lanes read one row's 128 bytes.  Rows come from the owning lanes by shuffle.
__device__ __forceinline__ void residual_load64(uint4 (&rr)[8], const ea_half* residual, long long ldr,
                                                int lane, long long m_mine, bool ok_mine, int col0,
                                                int cols_left, int n_limit, long long lin_m0, int M) {
  const int piece = lane & 7, rsub = lane >> 3;
  const int col = col0 + piece * 8;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int row = i * 4 + rsub;
    long long m_r;
    int ok_r;
    if (lin_m0 >= 0) {
      m_r = lin_m0 + row;
      ok_r = m_r < M;
    } else {
      m_r = __shfl_sync(0xffffffffu, m_mine, row);
      ok_r = __shfl_sync(0xffffffffu, (int)ok_mine, row);
    }
    rr[i] = (ok_r && piece * 8 < cols_left && col < n_limit)
                ? __ldg(reinterpret_cast<const uint4*>(residual + m_r * ldr + col))
                : make_uint4(0, 0, 0, 0);
  }
}

// GEGLU: value chunk fx (tile columns c..c+31), gate chunk fg (tile columns BN/2+c..): out = x*gelu(g)
// ln: the LayerNorm fold - acc * rstd[m] - rstd[m] * mean[m] * g[n] + c[n], g staged at cb + 256
__device__ __forceinline__ void epilogue_geglu32(const float* cb, int half_bn, int c, float (&fx)[32],
                                                 float (&fg)[32], uint4 (&o)[4], bool ln, float ln_r,
                                                 float ln_nm) {
  uint32_t packed[16];
#pragma unroll
  for (int j = 0; j < 32; j += 4) {     // 16-byte shared-memory loads: the per-column vectors are warp broadcasts
    float4 bx = *reinterpret_cast<const float4*>(cb + c + j);
    float4 bg = *reinterpret_cast<const float4*>(cb + half_bn + c + j);
    if (ln) {
      const float4 gx = *reinterpret_cast<const float4*>(cb + 256 + c + j);
      const float4 gg = *reinterpret_cast<const float4*>(cb + 256 + half_bn + c + j);
      bx.x = fmaf(ln_nm, gx.x, bx.x); bx.y = fmaf(ln_nm, gx.y, bx.y); bx.z = fmaf(ln_nm, gx.z, bx.z); bx.w = fmaf(ln_nm, gx.w, bx.w);
      bg.x = fmaf(ln_nm, gg.x, bg.x); bg.y = fmaf(ln_nm, gg.y, bg.y); bg.z = fmaf(ln_nm, gg.z, bg.z); bg.w = fmaf(ln_nm, gg.w, bg.w);
    }
    const float x0 = fmaf(fx[j], ln_r, bx.x), x1 = fmaf(fx[j + 1], ln_r, bx.y);
    const float x2 = fmaf(fx[j + 2], ln_r, bx.z), x3 = fmaf(fx[j + 3], ln_r, bx.w);
    const float g0 = fmaf(fg[j], ln_r, bg.x), g1 = fmaf(fg[j + 1], ln_r, bg.y);
    const float g2 = fmaf(fg[j + 2], ln_r, bg.z), g3 = fmaf(fg[j + 3], ln_r, bg.w);
    packed[j >> 1] = ea_pack2(x0 * gelu_erf_f(g0), x1 * gelu_erf_f(g1));
    packed[(j >> 1) + 1] = ea_pack2(x2 * gelu_erf_f(g2), x3 * gelu_erf_f(g3));
  }
#pragma unroll
  for (int q = 0; q < 4; ++q)
    o[q] = make_uint4(packed[4 * q], packed[4 * q + 1], packed[4 * q + 2], packed[4 * q + 3]);
}

// split-K reduce path: one thread = one (row, 32-column) unit, bias from global, direct stores
__device__ __forceinline__ void epilogue_geglu32_direct(const GemmKParams& p, const RowInfo& ri, int ncol0,
                                                        int half_bn, int c, float (&fx)[32],
                                                        float (&fg)[32]) {
  const int nout0 = (ncol0 >> 1) + c;  // output column of element 0
  if (!(ri.ok && nout0 < (p.N >> 1))) return;
  uint32_t packed[16];
#pragma unroll
  for (int j = 0; j < 32; j += 2) {
    float x0 = fx[j], x1 = fx[j + 1], g0 = fg[j], g1 = fg[j + 1];
    if (p.bias) {
      x0 += __ldg(p.bias + ncol0 + c + j);
      x1 += __ldg(p.bias + ncol0 + c + j + 1);
      g0 += __ldg(p.bias + ncol0 + half_bn + c + j);
      g1 += __ldg(p.bias + ncol0 + half_bn + c + j + 1);
    }
    packed[j >> 1] = ea_pack2(x0 * act_call(g0, EA_ACT_GELU), x1 * act_call(g1, EA_ACT_GELU));
  }
  uint4* dst = reinterpret_cast<uint4*>(p.out + ri.m * p.ldo + nout0);
#pragma unroll
  for (int q = 0; q < 4; ++q)
    dst[q] = make_uint4(packed[4 * q], packed[4 * q + 1], packed[4 * q + 2], packed[4 * q + 3]);
}

// +bias -> +rowvec -> act -> *scale -> +residual -> (+= out) -> store (and out2); 32 columns
__device__ __forceinline__ void epilogue_chunk32(const GemmKParams& p, const RowInfo& ri,
                                                 int n_first, float (&f)[32]) {
  if (!(ri.ok && n_first < p.N)) return;
  const long long m = ri.m;
  if (p.bias) {
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      if (n_first + j < p.N) {
        float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + n_first + j));
        f[j] += b.x; f[j + 1] += b.y; f[j + 2] += b.z; f[j + 3] += b.w;
      }
    }
  }
  if (p.rowvec) {
    const float* rv = p.rowvec + (long long)ri.batch * p.rowvec_ld + n_first;
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      if (n_first + j < p.N) {
        float4 b = __ldg(reinterpret_cast<const float4*>(rv + j));
        f[j] += b.x; f[j + 1] += b.y; f[j + 2] += b.z; f[j + 3] += b.w;
      }
    }
  }
  if (p.act == EA_ACT_SILU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = act_call(f[j], EA_ACT_SILU);
  } else if (p.act == EA_ACT_GELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = act_call(f[j], EA_ACT_GELU);
  }
  if (p.out_scale != 1.0f) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] *= p.out_scale;
  }
  if (p.row_scale) {   // spatial conditioning-scale map (utils/stable_diffusion_controlnet.py:789-802): one factor per row
    const float rs = __ldg(p.row_scale + m);
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] *= rs;
  }
  if (p.residual) {
    const uint4* rp = reinterpret_cast<const uint4*>(p.residual + m * p.ldr + n_first);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (n_first + q * 8 < p.N) {
        uint4 u = __ldg(rp + q);
        float2 a = ea_unpack2(u.x), b = ea_unpack2(u.y), cc = ea_unpack2(u.z), d = ea_unpack2(u.w);
        f[q * 8 + 0] += a.x; f[q * 8 + 1] += a.y; f[q * 8 + 2] += b.x; f[q * 8 + 3] += b.y;
        f[q * 8 + 4] += cc.x; f[q * 8 + 5] += cc.y; f[q * 8 + 6] += d.x; f[q * 8 + 7] += d.y;
      }
    }
  }
  if (p.out_f32) {
    float* dst = p.out_f32 + m * p.ldo + n_first;
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      if (n_first + j < p.N) {
        float4 o = make_float4(f[j], f[j + 1], f[j + 2], f[j + 3]);
        if (p.accumulate) {
          float4 old = *reinterpret_cast<float4*>(dst + j);
          o.x += old.x; o.y += old.y; o.z += old.z; o.w += old.w;
        }
        *reinterpret_cast<float4*>(dst + j) = o;
      }
    }
    return;
  }
  uint4* dst = reinterpret_cast<uint4*>(p.out + m * p.ldo + n_first);
  if (p.accumulate) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (n_first + q * 8 < p.N) {
        uint4 u = dst[q];
        float2 a = ea_unpack2(u.x), b = ea_unpack2(u.y), cc = ea_unpack2(u.z), d = ea_unpack2(u.w);
        f[q * 8 + 0] += a.x; f[q * 8 + 1] += a.y; f[q * 8 + 2] += b.x; f[q * 8 + 3] += b.y;
        f[q * 8 + 4] += cc.x; f[q * 8 + 5] += cc.y; f[q * 8 + 6] += d.x; f[q * 8 + 7] += d.y;
      }
    }
  }
  uint4* dst2 = p.out2 ? reinterpret_cast<uint4*>(p.out2 + m * p.ldo2 + n_first) : nullptr;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (n_first + q * 8 < p.N) {
      uint4 o = make_uint4(ea_pack2(f[q * 8 + 0], f[q * 8 + 1]), ea_pack2(f[q * 8 + 2], f[q * 8 + 3]),
                           ea_pack2(f[q * 8 + 4], f[q * 8 + 5]), ea_pack2(f[q * 8 + 6], f[q * 8 + 7]));
      dst[q] = o;
      if (dst2) dst2[q] = o;
    }
  }
}

// ------------------------------- host side ---------------------------------

static int encode_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer,
                     uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer) {
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = ea_tmap_encode()(m, EA_TMAP_DTYPE, 2, const_cast<void*>(base), dims, strides, box,
                                estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

static int encode_4d(CUtensorMap* m, const void* base, const uint64_t dims_[4],
                     const uint64_t strides_bytes[3], const uint32_t box_[4]) {
  cuuint64_t dims[4] = {dims_[0], dims_[1], dims_[2], dims_[3]};
  cuuint64_t strides[3] = {strides_bytes[0], strides_bytes[1], strides_bytes[2]};
  cuuint32_t box[4] = {box_[0], box_[1], box_[2], box_[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = ea_tmap_encode()(m, EA_TMAP_DTYPE, 4, const_cast<void*>(base), dims, strides, box,
                                estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

// Tile box geometry for an output of H x W per image: bw*bh*bn == 128, powers of two.
static void conv_geometry(int H, int W, int& bw, int& bh, int& bn) {
  bw = 1;
  while (bw * 2 <= W && bw * 2 <= 128 && (W % (bw * 2)) == 0) bw *= 2;
  bh = 1;
  while (bh * 2 <= H && bw * bh * 2 <= 128 && (H % (bh * 2)) == 0) bh *= 2;
  bn = 128 / (bw * bh);
}

// 32 staged accumulator values of tile row r, columns [c, c + 32)
__device__ __forceinline__ void acc_ld32(const float* accs, int ld, int r, int c, uint32_t (&v)[32]) {
  const float4* src = reinterpret_cast<const float4*>(accs + (size_t)r * ld + c);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 f = src[j];
    v[4 * j] = __float_as_uint(f.x); v[4 * j + 1] = __float_as_uint(f.y);
    v[4 * j + 2] = __float_as_uint(f.z); v[4 * j + 3] = __float_as_uint(f.w);
  }
}

// The work list runs over (group, split, tn, item) with the item (RP row tiles) fastest, so CTAs working side by side
// share their weight tile in L2; every group has the same shape and plan.  `p` below = the shared fields (group 0),
// each item re-binds `p` / the tensor maps to its own group.  tm0 = the item's first row tile.
#define EA_GEMM_TILE()                                                             \
  const int gi = NG == 1 ? 0 : tile / tiles_per_group;                             \
  const int gtile = NG == 1 ? tile : tile - gi * tiles_per_group;                  \
  const int zsplit = gtile / mn_items;                                             \
  const int mn = gtile - zsplit * mn_items;                                        \
  const GemmGroup& GG = L.g[gi];                                                   \
  const GemmKParams& p = GG.p;                                                     \
  const int tp = mn % m_items, tn = mn / m_items;                                  \
  const int tm0 = tp * RP;                                                         \
  const int kb0 = zsplit * p.kb_per_split;                                         \
  const int kb1 = min(nkb, kb0 + p.kb_per_split);

template <int BN, int NG, int RP>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
ea_gemm_kernel(const __grid_constant__ GemmLaunch<NG> L, const int tiles_per_group, const int m_items,
               const int n_groups) {
  const GemmKParams& p0 = L.g[0].p;
  const int n_tiles = (p0.N + BN - 1) / BN;
  const int mn_items = m_items * n_tiles;
  const int num_tiles = tiles_per_group * (NG == 1 ? 1 : n_groups);
  const int nkb = p0.nkb_main + p0.nkb_extra;
  constexpr int a_bytes = BM * BK * 2;
  constexpr int stage_bytes = gemm_stage_bytes(BN, RP);
  constexpr int ACC_LD = BN + 4;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~uintptr_t(1023));
  float* accs = reinterpret_cast<float*>(smem);
  uint8_t* stg_base = smem + RP * BM * ACC_LD * 4;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + gemm_region_bytes(BN, p0.stages, RP));
  uint64_t* empty_bar = full_bar + p0.stages;
  uint64_t* epi_done = empty_bar + p0.stages;       // the staged accumulator has been consumed: the ring is free
  float* cb = reinterpret_cast<float*>(epi_done + 2);   // [2 item parities][RP][2][256] per-column vectors

  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == W_TMA && lane == 0) {
    const int g0 = NG == 1 ? 0 : min((int)blockIdx.x / tiles_per_group, n_groups - 1);
    tma_prefetch_desc(&L.g[g0].tmA0);
    tma_prefetch_desc(&L.g[g0].tmB);
    if (p0.mode == EA_GEMM_CONV_S2 || p0.mode == EA_GEMM_CONV_S2A) {
      tma_prefetch_desc(&L.g[g0].tmA1);
      tma_prefetch_desc(&L.g[g0].tmA2);
      tma_prefetch_desc(&L.g[g0].tmA3);
    }
    if (p0.nkb_extra > 0) tma_prefetch_desc(&L.g[g0].tmAx);
  }
  if (warp == W_TMA) {   // lanes 2..31: every group's L2 prefetch hint, shared by the launch's first CTAs
    for (int g = 0; g < (NG == 1 ? 1 : n_groups); ++g) l2_prefetch_hint(L.g[g].p, (int)blockIdx.x, lane, 2);
  }
  if (warp == W_TMA && lane == 1) {
    for (int s = 0; s < p0.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], EPI_WARPS);
    }
    mbar_init(epi_done, EPI_WARPS);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= EPI_WARPS) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp != W_TMA || lane != 0) return;
    pdl_wait();
    // ============================ TMA producer ============================
    // One thread; the loop body is kept to a handful of scalar instructions (no divisions: the filter-tap /
    // channel-block position advances incrementally).
    int stage = 0;
    uint32_t phase = 0;
    uint8_t* sa = smem;
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      EA_GEMM_TILE()
      const CUtensorMap& tmA0 = GG.tmA0;
      const CUtensorMap& tmAx = GG.tmAx;
      const CUtensorMap& tmB = GG.tmB;
      if (it > 0) mbar_wait(epi_done, (uint32_t)((it - 1) & 1));   // the previous item's accumulator is read
      const int bcol = tn * BN;
      // sub-tile 0 always holds rows; sub-tile 1 (RP = 2) not in the last item of an odd number of row tiles
      const bool second = RP == 2 && tile_valid(p, tm0 + 1);
      const uint32_t tx_bytes = (uint32_t)((second ? 2 : 1) * a_bytes + BN * BK * 2);
      if (p.mode == EA_GEMM_LINEAR) {
        const int arow = tm0 * BM;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          mbar_expect_tx(&full_bar[stage], tx_bytes);
          tma_load_2d(sa, &tmA0, &full_bar[stage], kb * BK, arow);
          if (second) tma_load_2d(sa + a_bytes, &tmA0, &full_bar[stage], kb * BK, arow + BM);
          tma_load_2d_hint(sa + RP * a_bytes, &tmB, &full_bar[stage], kb * BK, bcol, p.b_policy);
          sa += stage_bytes;
          if (++stage == p.stages) { stage = 0; phase ^= 1u; sa = smem; }
        }
      } else {
        int n0, h0, w0, n1 = 0, h1 = 0, w1 = 0;
        tile_origin(p, tm0, n0, h0, w0);
        if (second) tile_origin(p, tm0 + 1, n1, h1, w1);
        // position of kb0: tap (kh, kw) and channel block c0 of the main source
        int tap = kb0 / p.cin_blocks;
        int c0 = (kb0 - tap * p.cin_blocks) * BK;
        int kh = tap / 3, kw = tap - kh * 3;
        const int cin = p.cin_blocks * BK;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          mbar_expect_tx(&full_bar[stage], tx_bytes);
          if (kb >= p.nkb_main) {
            // fused 1x1 skip convolution: centre tap of the raw block input
            tma_load_4d(sa, &tmAx, &full_bar[stage], (kb - p.nkb_main) * BK, w0, h0, n0);
            if (second) tma_load_4d(sa + a_bytes, &tmAx, &full_bar[stage], (kb - p.nkb_main) * BK, w1, h1, n1);
          } else if (p.mode == EA_GEMM_CONV_S1) {
            tma_load_4d(sa, &tmA0, &full_bar[stage], c0, w0 + kw - 1, h0 + kh - 1, n0);
            if (second) tma_load_4d(sa + a_bytes, &tmA0, &full_bar[stage], c0, w1 + kw - 1, h1 + kh - 1, n1);
          } else {
            // stride 2, pad 1: input row 2*oh + kh - 1 lives in phase ph = (kh != 1) at index oh + dh.
            // stride 2, pad (0,1,0,1) (CONV_S2A, the VAE encoder's Downsample): input row 2*oh + kh lives in
            // phase ph = (kh == 1) at index oh + (kh == 2); the bottom / right padding is TMA zero fill.
            const bool asym = p.mode == EA_GEMM_CONV_S2A;
            const int ph = asym ? (kh == 1 ? 1 : 0) : (kh == 1 ? 0 : 1);
            const int dh = asym ? (kh == 2 ? 1 : 0) : (kh == 0 ? -1 : 0);
            const int pw = asym ? (kw == 1 ? 1 : 0) : (kw == 1 ? 0 : 1);
            const int dw = asym ? (kw == 2 ? 1 : 0) : (kw == 0 ? -1 : 0);
            const int sel = ph * 2 + pw;
            const CUtensorMap* m = &tmA0 + sel;   // tmA0 .. tmA3 are consecutive members of GemmGroup
            tma_load_4d(sa, m, &full_bar[stage], c0, w0 + dw, h0 + dh, n0);
            if (second) tma_load_4d(sa + a_bytes, m, &full_bar[stage], c0, w1 + dw, h1 + dh, n1);
          }
          tma_load_2d_hint(sa + RP * a_bytes, &tmB, &full_bar[stage], kb * BK, bcol, p.b_policy);
          c0 += BK;
          if (c0 == cin) { c0 = 0; if (++kw == 3) { kw = 0; ++kh; } }
          sa += stage_bytes;
          if (++stage == p.stages) { stage = 0; phase ^= 1u; sa = smem; }
        }
      }
    }
    return;
  }

  // ================================ consumers =================================
  setmaxnreg_inc<CONSUMER_REGS>();
  pdl_wait();
  const int wg = warp >> 2;
  const int wq = warp & 3;
  const int r = wq * 32 + lane;        // epilogue: sub-tile row owned by this thread
  const int et = threadIdx.x;          // 0 .. EPI_THREADS-1
  // RP = 1: both warp-groups share the tile's rows (MMA: rows 64 wg ..) and take alternating 64-column groups of the
  // epilogue.  RP = 2: warp-group wg owns sub-tile wg, all of its rows and columns.
  const int sub = RP == 2 ? wg : 0;
  const int ar = sub * BM + r;                       // row of the staged accumulators
  constexpr int SUB_THREADS = EPI_THREADS / RP;      // epilogue threads of one sub-tile
  const int st_i = RP == 2 ? et & (SUB_THREADS - 1) : et;
  const int c64 = RP == 2 ? 0 : wg * 64;             // first 64-column group of this warp-group
  constexpr int GSTEP = RP == 2 ? 64 : 128;          // distance between two 64-column groups of one warp-group
  const int c32 = RP == 2 ? 0 : wg * 32;             // first 32-column chunk (general / split-K epilogues)
  constexpr int CSTEP = RP == 2 ? 32 : 64;
  uint4* stg = reinterpret_cast<uint4*>(stg_base + warp * 4096);
  uint4* stg2 = reinterpret_cast<uint4*>(stg_base + 4096 * EPI_WARPS + warp * 4096);
  const uint32_t smem0 = smem_u32(smem);
  int stage = 0;
  uint32_t phase = 0;
  int it = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
    EA_GEMM_TILE()
    const int tm = tm0 + sub;                        // this thread's row tile
    const bool sub_ok = RP == 1 || tile_valid(p, tm);
    const bool geglu = p.act == EA_ACT_GEGLU;
    const int half_bn = BN >> 1;
    const bool has_res = p.residual != nullptr;
    const RowInfo ri = row_info(p, tm, r);
    const int ncol0 = tn * BN;
    float* cbt = cb + ((it & 1) * RP + sub) * 512;
    const long long lin_m0 = p.mode == EA_GEMM_LINEAR ? (long long)tm * BM + wq * 32 : -1;
    const int b_first = row_info(p, tm, 0).batch, b_end = row_info(p, tm, BM - 1).batch;
    // rowvec has rows for the problem's batches only; the tile's last row lies past them in a partly empty image
    // block or in the last partial tile of a LINEAR problem, so the second staged row is that of the last valid row.
    // The epilogue is still chosen from the tile's full span b_first .. b_end: it decides the rounding order of
    // bias + rowvec, which must not depend on how many image slots hold data.
    const int b_last = min(b_end, p.mode != EA_GEMM_LINEAR ? p.Bsz - 1
                                  : p.rows_per_batch > 0 ? (p.M - 1) / p.rows_per_batch : 0);
    // Fast path (the common case): before the main loop, bias (+ the per-image time-embedding row vector) for the
    // tile's columns is staged in shared memory and the first residual chunk is pulled into registers, so that the
    // per-chunk work after the main loop is load -> FMA -> 16-byte stores with the NEXT chunk's residual in flight.
    const bool fast = sub_ok && p.splits == 1 && !geglu && !p.out_f32 && !p.accumulate && !p.row_scale &&
                      (b_end - b_first) <= 1;
    uint4 rres[8];   // next 64-column group of the residual (coalesced layout)
    // LayerNorm fold, consumer side: this row's mean / rstd from the producer's per-chunk partials (fixed
    // summation order: deterministic).  out = acc * ln_r + ln_nm * g[n] + c[n].
    const bool ln = p.ln_stats != nullptr;
    float ln_r = 1.f, ln_nm = 0.f;
    if (ln && ri.ok) ln_row_stats(p, ri.m, ln_r, ln_nm);
    if (fast) {
      for (int i = st_i; i < BN; i += SUB_THREADS) {
        const int col = ncol0 + i;
        float v0 = 0.f, v1 = 0.f;
        if (col < p.N) {
          const float bsum = p.bias ? __ldg(p.bias + col) : 0.f;
          v0 = bsum + (p.rowvec ? __ldg(p.rowvec + (long long)b_first * p.rowvec_ld + col) : 0.f);
          v1 = ln ? __ldg(p.ln_g + col)       // no row vector with the fold: the second slot carries g[n]
                  : bsum + (p.rowvec ? __ldg(p.rowvec + (long long)b_last * p.rowvec_ld + col) : 0.f);
        }
        cbt[i] = v0;
        cbt[256 + i] = v1;
      }
      if (has_res && c64 < BN)
        residual_load64(rres, p.residual, p.ldr, lane, ri.m, ri.ok, ncol0 + c64, BN - c64, p.N, lin_m0, p.M);
    } else if (geglu && p.splits == 1) {
      for (int i = st_i; i < BN; i += SUB_THREADS) {
        const bool in = ncol0 + i < p.N;
        cbt[i] = (p.bias && in) ? __ldg(p.bias + ncol0 + i) : 0.f;
        if (ln) cbt[256 + i] = in ? __ldg(p.ln_g + ncol0 + i) : 0.f;
      }
    }

    // ---- main loop: the stage of K-block kb is released once the MMAs of kb + 1 are in flight
    //      (a warp-group whose sub-tile lies past the problem multiplies whatever its A slot holds; nothing of it is
    //      stored)
    {
      float acc[RP][BN / 2];
#pragma unroll
      for (int h = 0; h < RP; ++h)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
      // A rows of this warp-group's 64-row MMA block h: RP = 1 -> tile rows 64 wg ..; RP = 2 -> sub-tile wg, rows 64 h ..
      const uint32_t a_off = RP == 2 ? (uint32_t)(wg * a_bytes) : (uint32_t)(wg * 64 * 128);
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem0 + (uint32_t)(stage * stage_bytes);
        const uint64_t db = gmma_desc_k_sw128(sa + (uint32_t)(RP * a_bytes), 1024);
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < RP; ++h) {
          const uint64_t da = gmma_desc_k_sw128(sa + a_off + (uint32_t)(h * 64 * 128), 1024);
#pragma unroll
          for (int k = 0; k < 4; ++k) Wgmma<BN>::ss(acc[h], da + 2 * k, db + 2 * k, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < RP; ++h) wgmma_fence_regs(acc[h]);
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      // every TMA load of this item has landed and, once both warp-groups are here, every MMA has retired: the ring
      // is free for the accumulators
      epi_bar_sync();
#pragma unroll
      for (int h = 0; h < RP; ++h) {
        const int r0 = (RP == 2 ? wg * BM + h * 64 : wg * 64) + wq * 16 + (lane >> 2);
        float* d0 = accs + (size_t)r0 * ACC_LD + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          *reinterpret_cast<float2*>(d0 + 8 * j) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
          *reinterpret_cast<float2*>(d0 + 8 * ACC_LD + 8 * j) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
        }
      }
    }
    epi_bar_sync();

    if (fast) {
      const float* cbr = cbt + ((!ln && ri.batch != b_first) ? 256 : 0);
      // this warp-group's chunks: both halves of the 64-column groups c64, c64 + GSTEP, ...
      auto next_chunk = [&](int c) { return ((c & 32) == 0 && c + 32 < BN) ? c + 32 : (c & ~63) + GSTEP; };
      for (int c = c64; c < BN; c = next_chunk(c)) {
        uint32_t v[32];
        acc_ld32(accs, ACC_LD, ar, c, v);
        const int n_first = ncol0 + c;
        const int half = (c >> 5) & 1;
        if (has_res && half == 0) {
          // hand the prefetched group to its rows through the second staging block, then put the next group's
          // loads in flight
          const int piece = lane & 7, rsub = lane >> 3;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int row = i * 4 + rsub;
            stg2[row * 8 + (piece ^ (row & 7))] = rres[i];
          }
          __syncwarp();
          if (c + GSTEP < BN)
            residual_load64(rres, p.residual, p.ldr, lane, ri.m, ri.ok, n_first + GSTEP, BN - c - GSTEP, p.N, lin_m0, p.M);
        }
        float f[32];
        if (ln) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const float4 b4 = *reinterpret_cast<const float4*>(cbt + c + j);
            const float4 g4 = *reinterpret_cast<const float4*>(cbt + 256 + c + j);
            f[j] = fmaf(__uint_as_float(v[j]), ln_r, fmaf(ln_nm, g4.x, b4.x));
            f[j + 1] = fmaf(__uint_as_float(v[j + 1]), ln_r, fmaf(ln_nm, g4.y, b4.y));
            f[j + 2] = fmaf(__uint_as_float(v[j + 2]), ln_r, fmaf(ln_nm, g4.z, b4.z));
            f[j + 3] = fmaf(__uint_as_float(v[j + 3]), ln_r, fmaf(ln_nm, g4.w, b4.w));
          }
        } else {
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const float4 b4 = *reinterpret_cast<const float4*>(cbr + c + j);
            f[j] = __uint_as_float(v[j]) + b4.x;
            f[j + 1] = __uint_as_float(v[j + 1]) + b4.y;
            f[j + 2] = __uint_as_float(v[j + 2]) + b4.z;
            f[j + 3] = __uint_as_float(v[j + 3]) + b4.w;
          }
        }
        if (p.act == EA_ACT_SILU) {
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] = act_call(f[j], EA_ACT_SILU);
        } else if (p.act == EA_ACT_GELU) {
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] = gelu_erf_f(f[j]);
        }
        if (p.out_scale != 1.0f) {
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] *= p.out_scale;
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int slot = lane * 8 + ((half * 4 + q) ^ (lane & 7));
          if (has_res) {
            const uint4 rc = stg2[slot];
            const float2 a = ea_unpack2(rc.x), b = ea_unpack2(rc.y), cc = ea_unpack2(rc.z), d = ea_unpack2(rc.w);
            f[q * 8 + 0] += a.x; f[q * 8 + 1] += a.y; f[q * 8 + 2] += b.x; f[q * 8 + 3] += b.y;
            f[q * 8 + 4] += cc.x; f[q * 8 + 5] += cc.y; f[q * 8 + 6] += d.x; f[q * 8 + 7] += d.y;
          }
          const uint4 o = make_uint4(ea_pack2(f[q * 8 + 0], f[q * 8 + 1]), ea_pack2(f[q * 8 + 2], f[q * 8 + 3]),
                                     ea_pack2(f[q * 8 + 4], f[q * 8 + 5]), ea_pack2(f[q * 8 + 6], f[q * 8 + 7]));
          stg[slot] = o;
          if (p.rowstats_out) {   // the statistics describe the rounded values the consumer will read
            const float2 a = ea_unpack2(o.x), b = ea_unpack2(o.y), cc = ea_unpack2(o.z), d = ea_unpack2(o.w);
            f[q * 8 + 0] = a.x; f[q * 8 + 1] = a.y; f[q * 8 + 2] = b.x; f[q * 8 + 3] = b.y;
            f[q * 8 + 4] = cc.x; f[q * 8 + 5] = cc.y; f[q * 8 + 6] = d.x; f[q * 8 + 7] = d.y;
          }
        }
        if (p.rowstats_out) {
          // LayerNorm fold, producer side: this row's (sum, sum of squared deviations from the chunk mean) over the
          // chunk's 32 stored values.  Centring on the chunk mean keeps M2 exact to a few ulps whatever |mean| / std.
          float s0 = 0.f, s1 = 0.f;
#pragma unroll
          for (int j = 0; j < 32; j += 2) { s0 += f[j]; s1 += f[j + 1]; }
          const float s = s0 + s1, mc = s * (1.f / 32.f);
          float q0 = 0.f, q1 = 0.f;
#pragma unroll
          for (int j = 0; j < 32; j += 2) {
            const float d0 = f[j] - mc, d1 = f[j + 1] - mc;
            q0 = fmaf(d0, d0, q0);
            q1 = fmaf(d1, d1, q1);
          }
          if (ri.ok && n_first < p.N) p.rowstats_out[(size_t)(n_first >> 5) * p.M + ri.m] = make_float2(s, q0 + q1);
        }
        if (half == 1 || c + 32 >= BN)
          stage_flush(stg, lane, p.out, p.ldo, p.out2, p.ldo2, ri.m, ri.ok, n_first - half * 32,
                      half == 1 ? 8 : 4, p.N, lin_m0, p.M);
      }
    } else if (p.splits == 1) {
      if (geglu) {
        // tile columns: [0, BN/2) = value half, [BN/2, BN) = gate half (weights pre-interleaved); RP = 1: the
        // 32-column output chunks alternate between the two warp-groups, each flushed on its own
        for (int c = c32; c < half_bn; c += CSTEP) {
          uint32_t xv[32], gv[32];
          acc_ld32(accs, ACC_LD, ar, c, xv);
          acc_ld32(accs, ACC_LD, ar, half_bn + c, gv);
          float fx[32], fg[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) { fx[j] = __uint_as_float(xv[j]); fg[j] = __uint_as_float(gv[j]); }
          uint4 o[4];
          epilogue_geglu32(cbt, half_bn, c, fx, fg, o, ln, ln_r, ln_nm);
          stage_put32(stg, lane, 0, o);
          if (lin_m0 >= 0)
            stage_flush32(stg, lane, p.out, p.ldo, (ncol0 >> 1) + c, p.N >> 1, lin_m0, p.M);
          else
            stage_flush(stg, lane, p.out, p.ldo, nullptr, 0, ri.m, ri.ok, (ncol0 >> 1) + c, 4, p.N >> 1, lin_m0, p.M);
        }
      } else {
        for (int c = c32; c < BN; c += CSTEP) {
          uint32_t v[32];
          acc_ld32(accs, ACC_LD, ar, c, v);
          float f[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(v[j]);
          epilogue_chunk32(p, ri, ncol0 + c, f);
          __syncwarp();
        }
      }
    } else {
      // ---- split-K: publish the fp32 partial item (RP sub-tiles), wait for the sibling splits, then every
      //      split CTA reduces and finishes a 1/splits share of the item's (row, 32-col) units.
      constexpr int RB = RP * BM;                    // rows of one item
      const int tile_id = tn * m_items + tp;
      float* wtile = p.ws + (size_t)tile_id * p.splits * (RB * BN);
      float* mine = wtile + (size_t)zsplit * (RB * BN);
      for (int c = c32; c < BN; c += CSTEP) {
        uint32_t v[32];
        acc_ld32(accs, ACC_LD, ar, c, v);
        float4* dst = reinterpret_cast<float4*>(mine + (size_t)ar * BN + c);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          __stcg(dst + j, make_float4(__uint_as_float(v[4 * j]), __uint_as_float(v[4 * j + 1]),
                                      __uint_as_float(v[4 * j + 2]), __uint_as_float(v[4 * j + 3])));
      }
      __threadfence();
      epi_bar_sync();
      int* cnt = p.cnt + 2 * tile_id;
      if (et == 0) {
        atomicAdd(cnt, 1);
        uint32_t spins = 0;
        while (ld_acquire_gpu(cnt) < p.splits) {
          __nanosleep(40);
          if (++spins > (1u << 24)) { asm volatile("trap;"); }
        }
      }
      epi_bar_sync();
      __threadfence();
      {
        const int chunks = geglu ? (half_bn >> 5) : (BN >> 5);
        const int units = RB * chunks;
        const int u0 = (int)(((long long)units * zsplit) / p.splits);
        const int u1 = (int)(((long long)units * (zsplit + 1)) / p.splits);
        // Stage 1 (all consumer threads, float4 granularity, loads of the sibling partials unrolled for
        // memory-level parallelism) sums this CTA's share into the (published, now dead) accumulator staging;
        // stage 2 runs the fused epilogue on whole 32-column units, one per thread.
        const int segs = geglu ? 2 : 1;                 // 32-float segments per unit (value | gate)
        const int ustride = segs * 32 + 4;              // padded floats per unit in smem
        float* stage_f = accs;
        const size_t split_stride = (size_t)RB * BN;
        for (int ub = u0; ub < u1; ub += EPI_THREADS) {
          const int nu = min(EPI_THREADS, u1 - ub);
          const int nvec4 = nu * segs * 8;
          for (int idx = et; idx < nvec4; idx += EPI_THREADS) {
            const int ul = idx / (segs * 8);
            const int rem = idx - ul * (segs * 8);
            const int seg = rem >> 3, q = rem & 7;
            const int u = ub + ul;
            const int rr = u & (RB - 1);
            const int c = ((u / RB) << 5) + seg * half_bn * (geglu ? 1 : 0);
            const float4* src = reinterpret_cast<const float4*>(wtile + (size_t)rr * BN + c) + q;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            int sidx = 0;
            for (; sidx + 4 <= p.splits; sidx += 4) {
              float4 v0 = __ldcg(src + (size_t)(sidx + 0) * (split_stride >> 2));
              float4 v1 = __ldcg(src + (size_t)(sidx + 1) * (split_stride >> 2));
              float4 v2 = __ldcg(src + (size_t)(sidx + 2) * (split_stride >> 2));
              float4 v3 = __ldcg(src + (size_t)(sidx + 3) * (split_stride >> 2));
              acc.x += v0.x; acc.y += v0.y; acc.z += v0.z; acc.w += v0.w;
              acc.x += v1.x; acc.y += v1.y; acc.z += v1.z; acc.w += v1.w;
              acc.x += v2.x; acc.y += v2.y; acc.z += v2.z; acc.w += v2.w;
              acc.x += v3.x; acc.y += v3.y; acc.z += v3.z; acc.w += v3.w;
            }
            for (; sidx < p.splits; ++sidx) {
              float4 v0 = __ldcg(src + (size_t)sidx * (split_stride >> 2));
              acc.x += v0.x; acc.y += v0.y; acc.z += v0.z; acc.w += v0.w;
            }
            *reinterpret_cast<float4*>(stage_f + ul * ustride + seg * 32 + q * 4) = acc;
          }
          epi_bar_sync();
          if (et < nu) {
            const int u = ub + et;
            const int rr = u & (RB - 1);
            const int c = (u / RB) << 5;
            RowInfo r2 = row_info(p, tm0 + rr / BM, rr & (BM - 1));
            const float4* sp = reinterpret_cast<const float4*>(stage_f + et * ustride);
            float f[32];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              float4 v = sp[j];
              f[4 * j] = v.x; f[4 * j + 1] = v.y; f[4 * j + 2] = v.z; f[4 * j + 3] = v.w;
            }
            if (geglu) {
              float fg[32];
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                float4 v = sp[8 + j];
                fg[4 * j] = v.x; fg[4 * j + 1] = v.y; fg[4 * j + 2] = v.z; fg[4 * j + 3] = v.w;
              }
              epilogue_geglu32_direct(p, r2, ncol0, half_bn, c, f, fg);
            } else {
              epilogue_chunk32(p, r2, ncol0 + c, f);
            }
          }
          epi_bar_sync();
        }
        epi_bar_sync();
        if (et == 0) {
          int old = atomicAdd(cnt + 1, 1);
          if (old == p.splits - 1) {  // last finisher: re-arm the counters for the next launch
            cnt[0] = 0;
            cnt[1] = 0;
          }
        }
      }
    }
    // the staged accumulator has been read: hand the ring back to the producer (its next loads are async-proxy
    // writes over what this thread wrote and read through the generic proxy)
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) mbar_arrive(epi_done);
  }
}
#undef EA_GEMM_TILE

// ---- launch planner -------------------------------------------------------------------
// Picks (BN, row tiles per CTA, stages, split-K) for one problem from a small cycle model: per K-block a CTA needs
// max(MMA time, its share of chip bandwidth, TMA latency / stages in flight); small-M layers (8x8 / 16x16 latents:
// M = 128 / 512) are weight-streaming bound, so K is split across CTAs until every SM has one deep pipeline, and the
// partial tiles are combined in-kernel (see the epilogue).  Two row tiles per CTA (rp = 2) share each W box: per
// K-block the A bytes and the MMA time double, the W bytes do not, and the fixed costs are paid once per pair.  They
// are never combined with split-K, which exists because there are fewer tiles than SMs.
struct GemmPlan { int BN, stages, splits, kbps, rp; double cost; };

// Per-SM and chip rates in bytes per SM clock, from the H100 SXM data sheet (3.35 TB/s HBM3; fp16 wgmma at
// 989 TFLOP/s over 132 SMs = 2048 MAC / clk / SM, so a 128 x BN x 64 K-block takes 4 BN clk) and L2 at about 1.6x
// HBM; the fixed costs (pipeline start ~3800 clk, ~50 clk per accumulator column of epilogue) are not measured
// per shape.  tools/gemm_rowpair_ab.py times every GEMM shape of the bench step both ways; on an H100 SXM at a
// 400 W power limit no single-wave shape reached the MMA rate (120 CTAs of 512 x 1280 x 5120: ~1190 clk per
// 512-clk K-block), so these constants rank layouts rather than predict times.
static constexpr double PL_LAT = 2100.0, PL_SM_CAP = 57.0, PL_L2 = 3000.0, PL_HBM = 1900.0;
static constexpr double PL_SPLIT_COL = 8.0, PL_SPLIT_FIX = 7000.0;
static constexpr double PL_START = 3800.0, PL_EPI = 50.0, PL_EPI_RES = 21.0;
static constexpr int GEMM_BN[3] = {128, 64, 32};   // the tile widths the planner picks from (see GEMM_THREADS)

// groups: identical problems run by the same launch - they multiply the CTAs (waves, what is left to split K
// over) but not the reuse of one weight tile across its M-tiles.  force_rp: 0 = either, 1 / 2 = only that.
static GemmPlan plan_gemm(int mt, int N, int nkb, int act, long long ws_floats, int n_sm, bool has_res = false,
                          int groups = 1, int force_rp = 0) {
  const double epi_col = (PL_EPI + (has_res ? PL_EPI_RES : 0.0)) * (act == EA_ACT_GEGLU ? 0.84 : 1.0);
  GemmPlan best = {0, 0, 1, nkb, 1, 1e30};
  for (int rp = 1; rp <= 2; ++rp) {
    if (force_rp > 0 && rp != force_rp) continue;
    if (force_rp == 0 && rp == 2 && mt < 2) continue;
    const int mi = (mt + rp - 1) / rp;              // row items (CTAs along M)
    for (int BN : GEMM_BN) {
      if (act == EA_ACT_GEGLU && BN != 128) continue;  // weights are interleaved per 128-row block
      if (BN > 32 && N <= BN - 32) continue;            // a narrower tile covers N just as well
      const int nt = (N + BN - 1) / BN;
      const long long tiles = (long long)mi * nt * groups;
      const int stage_bytes = gemm_stage_bytes(BN, rp);
      int st = GEMM_SMEM_RING / stage_bytes;
      if (st > 8) st = 8;
      if (st > nkb) st = nkb < 2 ? 2 : nkb;
      const long long slots = n_sm;                   // one CTA per SM
      // Pairs only pay once one tile per CTA needs more than one wave: below that they halve the SMs at work, and
      // on H100 (tools/gemm_rowpair_ab.py) every such step shape ran slower paired, e.g. 120 tiles of 512 x 1280 x
      // 5120: 54 us single, 74 us paired.
      if (force_rp == 0 && rp == 2 && (long long)mt * nt * groups <= slots) continue;
      for (int pass = 0; pass < (rp == 1 ? 2 : 1); ++pass) {
        int splits = 1, kbps = nkb;
        if (pass == 1) {
          if (tiles >= slots || nkb < 8) break;
          int s_max = (int)(slots / tiles);
          if (s_max > nkb / 4) s_max = nkb / 4;
          if (s_max < 2) break;
          kbps = (nkb + s_max - 1) / s_max;
          splits = (nkb + kbps - 1) / kbps;  // every split owns at least one K-block
          if (splits < 2) break;
          if (tiles > 2048 || tiles * splits * (long long)(BM * BN) > ws_floats) break;
        }
        const long long ctas = tiles * splits;
        const long long waves = (ctas + slots - 1) / slots;
        const long long conc = ctas < slots ? ctas : slots;
        const double t_mma = 4.0 * BN * rp;
        const double t_sm = (double)stage_bytes / PL_SM_CAP;               // per-SM TMA fill cap
        const double a_bytes = rp * BM * BK * 2.0, b_bytes = BN * BK * 2.0;
        const double hbm_frac = 1.0 / (double)mi;                         // weights: HBM once, then L2
        const double t_chip = (double)conc * (a_bytes / PL_L2 + b_bytes * hbm_frac / PL_HBM +
                                              b_bytes * (1.0 - hbm_frac) / PL_L2);
        const double t_lat = PL_LAT / st;
        double t_kb = t_mma;
        if (t_sm > t_kb) t_kb = t_sm;
        if (t_chip > t_kb) t_kb = t_chip;
        if (t_lat > t_kb) t_kb = t_lat;
        double cost;
        if (splits == 1) {
          cost = (double)waves * (PL_START + kbps * t_kb + epi_col * BN * rp);
        } else {
          // fp32 partial store, arrival counter, distributed reduce + fused epilogue
          cost = (double)waves * (PL_START + kbps * t_kb + PL_SPLIT_COL * BN) + PL_SPLIT_FIX +
                 3.0 * (BM * BN * 4.0) / 25.0 + 150.0 * splits;
        }
        if (cost < best.cost) best = {BN, st, splits, kbps, rp, cost};
      }
    }
  }
  return best;
}

static int sm_count() { return ea_sm_count(); }

}  // namespace ea

using namespace ea;

extern "C" int ea_gemm_plan(int m_tiles, int N, int k_blocks, int act, long long workspace_bytes,
                            int n_sm, int* out5) {
  if (!out5 || m_tiles <= 0 || N <= 0 || k_blocks <= 0) return EA_ERR_ARG;
  const long long ws_floats = workspace_bytes > 65536 ? (workspace_bytes - 65536) / 4 : 0;
  GemmPlan pl = plan_gemm(m_tiles, N, k_blocks, act, ws_floats, n_sm > 0 ? n_sm : 132);
  out5[0] = pl.BN; out5[1] = pl.stages; out5[2] = pl.splits; out5[3] = pl.kbps;
  out5[4] = 1;   // CTAs per SM
  return pl.BN ? EA_OK : EA_ERR_SHAPE;
}

// Everything of one problem that does not depend on the launch plan: validation, the parameter block, the A maps.
struct GemmShape {
  int m_tiles, nkb;
  long long Ktot;
  bool ln_any;
};

static int gemm_fill_group(const ea_gemm_args* a, GemmGroup& G, GemmShape& sh) {
  if (!a || !a->a || !a->w || (!a->out && !a->out_f32)) return EA_ERR_ARG;
  if (a->mode < 0 || a->mode > EA_GEMM_CONV_S2A) return EA_ERR_ARG;
  if (a->N <= 0 || a->M <= 0) return EA_ERR_ARG;
  if (a->N % 8 != 0) return EA_ERR_SHAPE;
  GemmKParams& p = G.p;
  memset(&p, 0, sizeof(p));
  p.M = a->M;
  p.N = a->N;
  p.mode = a->mode;
  p.bias = a->bias;
  p.rowvec = a->rowvec;
  p.rows_per_batch = a->rows_per_batch;
  p.rowvec_ld = a->rowvec_ld;
  p.residual = reinterpret_cast<const ea_half*>(a->residual);
  p.ldr = a->ldr;
  p.out = reinterpret_cast<ea_half*>(a->out);
  p.ldo = a->ldo;
  p.out2 = reinterpret_cast<ea_half*>(a->out2);
  p.ldo2 = a->ldo2;
  p.out_f32 = a->out_f32;
  p.act = a->act;
  p.out_scale = a->out_scale;
  p.accumulate = a->accumulate;
  p.row_scale = a->row_scale;
  for (int i = 0; i < EA_GEMM_MAX_PREFETCH; ++i) {
    p.pf[i] = reinterpret_cast<const char*>(a->prefetch[i]);
    p.pf_bytes[i] = a->prefetch[i] ? (a->prefetch_bytes[i] & ~15LL) : 0;
  }
  p.pf_ctas = 0;   // set with the grid
  // W operand: streamed once per step (3.16 GB through a 50 MB L2) - marked evict-first so that it displaces itself
  // rather than the activations and skip tensors the following launches read.
  p.b_policy = 0x12F0000000000000ull;
  if (a->row_scale && (a->act == EA_ACT_GEGLU || a->rowstats_out || a->ln_stats)) return EA_ERR_ARG;
  // The GEGLU epilogues apply the bias and the LayerNorm fold only
  if (a->act == EA_ACT_GEGLU &&
      (a->rowvec || a->residual || a->out2 || a->out_f32 || a->accumulate || a->out_scale != 1.0f))
    return EA_ERR_ARG;
  sh.ln_any = a->rowstats_out || a->ln_stats;
  if (sh.ln_any) {
    // rows_per_batch could make a tile span more than two batches, whose (general) epilogue has no fold
    if (a->mode != EA_GEMM_LINEAR || a->rowvec || a->rows_per_batch != 0 || a->out_f32 || a->accumulate)
      return EA_ERR_ARG;
    if (a->rowstats_out && (a->N % 32 != 0 || a->act == EA_ACT_GEGLU)) return EA_ERR_SHAPE;
    if (a->ln_stats && (!a->ln_g || a->ln_parts <= 0 || a->K != a->ln_parts * 32)) return EA_ERR_ARG;
    p.rowstats_out = reinterpret_cast<float2*>(a->rowstats_out);
    p.ln_stats = reinterpret_cast<const float2*>(a->ln_stats);
    p.ln_g = a->ln_g;
    p.ln_parts = a->ln_parts;
    p.ln_inv_c = a->ln_stats ? 1.0f / (float)a->K : 0.f;
    p.ln_eps = a->ln_eps;
  }
  // a leading dimension narrower than the row it strides over makes rows overlap (0 writes every row onto row 0)
  const long long n_out = a->act == EA_ACT_GEGLU ? a->N / 2 : a->N;
  if (p.ldo % 8 != 0 || p.ldo < n_out || (p.residual && (p.ldr % 8 != 0 || p.ldr < n_out)) ||
      (p.out2 && (p.ldo2 % 8 != 0 || p.ldo2 < n_out)))
    return EA_ERR_SHAPE;

  CUtensorMap* tmA[4] = {&G.tmA0, &G.tmA1, &G.tmA2, &G.tmA3};
  if (a->mode == EA_GEMM_LINEAR) {
    if (a->K % 8 != 0 || a->lda % 8 != 0 || a->lda < a->K) return EA_ERR_SHAPE;
    p.nkb_main = (a->K + BK - 1) / BK;
    p.nkb_extra = 0;
    p.cin_blocks = 1;
    sh.m_tiles = (a->M + BM - 1) / BM;
    sh.Ktot = a->K;
    if (encode_2d(tmA[0], a->a, (uint64_t)a->K, (uint64_t)a->M, (uint64_t)a->lda * 2, BK, BM))
      return EA_ERR_TMAP;
    G.tmA1 = G.tmA2 = G.tmA3 = G.tmA0;
    G.tmAx = G.tmA0;
  } else {
    const int H = a->H, W = a->W, B = a->Bsz, C = a->Cin;
    if (C % 64 != 0 || H <= 0 || W <= 0 || B <= 0) return EA_ERR_SHAPE;
    if ((long long)B * H * W != a->M) return EA_ERR_SHAPE;
    if (a->lda != 0 && (a->lda < C || a->lda % 8 != 0)) return EA_ERR_SHAPE;
    p.H = H; p.W = W; p.Bsz = B;
    conv_geometry(H, W, p.bw, p.bh, p.bn);
    p.tiles_w = W / p.bw;
    p.tiles_h = H / p.bh;
    p.cin_blocks = C / 64;
    p.nkb_main = 9 * p.cin_blocks;
    p.nkb_extra = 0;
    sh.m_tiles = ((B + p.bn - 1) / p.bn) * p.tiles_w * p.tiles_h;
    sh.Ktot = 9LL * C;
    const long long lda = a->lda > 0 ? a->lda : C;  // channel stride of one pixel (elements)
    uint32_t box[4] = {64, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
    if (a->mode == EA_GEMM_CONV_S1) {
      uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
      uint64_t st[3] = {(uint64_t)lda * 2, (uint64_t)lda * W * 2, (uint64_t)lda * W * H * 2};
      if (encode_4d(tmA[0], a->a, dims, st, box)) return EA_ERR_TMAP;
      G.tmA1 = G.tmA2 = G.tmA3 = G.tmA0;
    } else {
      // input is (2H x 2W); four phase views (ph, pw) each of H x W
      const int Hin = 2 * H, Win = 2 * W;
      for (int ph = 0; ph < 2; ++ph)
        for (int pw = 0; pw < 2; ++pw) {
          const ea_half* base =
              reinterpret_cast<const ea_half*>(a->a) + ((long long)ph * Win + pw) * lda;
          uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
          uint64_t st[3] = {(uint64_t)lda * 2 * 2, (uint64_t)lda * Win * 2 * 2,
                            (uint64_t)lda * Win * Hin * 2};
          if (encode_4d(tmA[ph * 2 + pw], base, dims, st, box)) return EA_ERR_TMAP;
        }
    }
    G.tmAx = G.tmA0;
    if (a->a_extra) {
      if (a->mode != EA_GEMM_CONV_S1 || a->Cin_extra % 64 != 0) return EA_ERR_SHAPE;
      if (a->ld_extra != 0 && (a->ld_extra < a->Cin_extra || a->ld_extra % 8 != 0)) return EA_ERR_SHAPE;
      const long long ldx = a->ld_extra > 0 ? a->ld_extra : a->Cin_extra;
      uint64_t dims[4] = {(uint64_t)a->Cin_extra, (uint64_t)W, (uint64_t)H, (uint64_t)B};
      uint64_t st[3] = {(uint64_t)ldx * 2, (uint64_t)ldx * W * 2, (uint64_t)ldx * W * H * 2};
      if (encode_4d(&G.tmAx, a->a_extra, dims, st, box)) return EA_ERR_TMAP;
      p.nkb_extra = a->Cin_extra / 64;
      sh.Ktot += a->Cin_extra;
    }
  }
  sh.nkb = p.nkb_main + p.nkb_extra;
  if (a->ldw > 0 && (a->ldw % 8 != 0 || a->ldw < sh.Ktot)) return EA_ERR_SHAPE;
  return EA_OK;
}

// groups of one launch must be the same problem with different pointers
static bool gemm_same_problem(const ea_gemm_args* a, const ea_gemm_args* b) {
  return a->mode == b->mode && a->M == b->M && a->N == b->N && a->K == b->K && a->Bsz == b->Bsz && a->H == b->H &&
         a->W == b->W && a->Cin == b->Cin && a->Cin_extra == b->Cin_extra && (!a->a_extra) == (!b->a_extra) &&
         a->act == b->act && a->accumulate == b->accumulate && (!a->out_f32) == (!b->out_f32) &&
         (!a->row_scale) == (!b->row_scale) &&
         (!a->rowvec) == (!b->rowvec) && a->rows_per_batch == b->rows_per_batch &&
         (!a->rowstats_out) == (!b->rowstats_out) && (!a->ln_stats) == (!b->ln_stats) && a->ln_parts == b->ln_parts &&
         a->force_bn == b->force_bn && a->force_splits == b->force_splits && a->force_2cta == b->force_2cta &&
         a->force_persistent == b->force_persistent;
}

template <typename K>
static int set_max_smem(K kernel, int bytes, int& cached) {
  if (bytes > cached) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return ea_cuda_fail(e, "ea_gemm: cudaFuncSetAttribute(MaxDynamicSharedMemorySize)");
    cached = bytes;
  }
  return EA_OK;
}

template <int BN, int NG, int RP>
static cudaError_t launch_gemm(const GemmLaunch<NG>& L, int grid, int smem_bytes, int tiles_per_group, int m_items,
                               int n_groups, cudaStream_t stream, int& rc) {
  static int cache[EA_MAX_DEV];   // zero-initialised; per device (see ea_internal.h)
  if ((rc = set_max_smem(ea_gemm_kernel<BN, NG, RP>, smem_bytes, cache[ea_dev()]))) return cudaSuccess;
  return ea_launch(ea_gemm_kernel<BN, NG, RP>, dim3((unsigned)grid), dim3(GEMM_THREADS), (size_t)smem_bytes, stream,
                   L, tiles_per_group, m_items, n_groups);
}

template <int NG>
static cudaError_t launch_gemm_bn(int BN, int rp, const GemmLaunch<NG>& L, int grid, int smem_bytes,
                                  int tiles_per_group, int m_items, int n_groups, cudaStream_t stream, int& rc) {
  if (rp == 2) {
    switch (BN) {
      case 32: return launch_gemm<32, NG, 2>(L, grid, smem_bytes, tiles_per_group, m_items, n_groups, stream, rc);
      case 64: return launch_gemm<64, NG, 2>(L, grid, smem_bytes, tiles_per_group, m_items, n_groups, stream, rc);
      case 128: return launch_gemm<128, NG, 2>(L, grid, smem_bytes, tiles_per_group, m_items, n_groups, stream, rc);
      default: return cudaErrorInvalidValue;   // ea_gemm_grouped admits 32 / 64 / 128 only
    }
  }
  switch (BN) {
    case 32: return launch_gemm<32, NG, 1>(L, grid, smem_bytes, tiles_per_group, m_items, n_groups, stream, rc);
    case 64: return launch_gemm<64, NG, 1>(L, grid, smem_bytes, tiles_per_group, m_items, n_groups, stream, rc);
    case 128: return launch_gemm<128, NG, 1>(L, grid, smem_bytes, tiles_per_group, m_items, n_groups, stream, rc);
    default: return cudaErrorInvalidValue;
  }
}

extern "C" int ea_gemm_grouped(const ea_gemm_args* args, int n_groups, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!args || n_groups < 1 || n_groups > GEMM_MAX_GROUPS) return EA_ERR_ARG;
  const ea_gemm_args* a = &args[0];          // shape, flags and plan come from group 0
  static GemmLaunch<GEMM_MAX_GROUPS> L;      // host-side staging (ea_gemm is not re-entrant per process, see header)
  GemmShape sh0;
  memset(&L, 0, sizeof(L));
  for (int g = 0; g < n_groups; ++g) {
    GemmShape shg;
    if (g > 0 && !gemm_same_problem(a, &args[g])) return EA_ERR_ARG;
    const int rc = gemm_fill_group(&args[g], L.g[g], g == 0 ? sh0 : shg);
    if (rc != EA_OK) return rc;
  }
  const int m_tiles = sh0.m_tiles, nkb = sh0.nkb;
  const bool ln_any = sh0.ln_any;
  const int G = n_groups;
  // workspace: [0, 64 KB) arrival counters (int, zero between launches), then fp32 partial tiles
  const long long ws_floats =      // the LayerNorm fold lives in the unsplit epilogues only
      (a->workspace && a->workspace_bytes > 65536 && !ln_any) ? (a->workspace_bytes - 65536) / 4 : 0;
  // force_persistent > 0: one CTA per SM walking the tile list (no split-K); otherwise one tile per CTA
  const bool persist = a->force_persistent > 0;
  const bool has_res = a->residual != nullptr;
  // force_2cta: 1 = two row tiles per CTA, -1 = one, 0 = the planner's choice
  const int force_rp = a->force_2cta > 0 ? 2 : a->force_2cta < 0 ? 1 : 0;
  GemmPlan plan =
      plan_gemm(m_tiles, a->N, nkb, a->act, persist ? 0 : ws_floats, sm_count(), has_res, G, force_rp);
  if (a->force_bn > 0) plan.BN = a->force_bn;
  if (plan.BN != 32 && plan.BN != 64 && plan.BN != 128) return EA_ERR_SHAPE;
  if (a->force_bn > 0 || a->force_splits > 0) {
    const int sb = gemm_stage_bytes(plan.BN, plan.rp);
    if (a->force_bn > 0) plan.stages = 3;
    if (plan.stages * sb > GEMM_SMEM_RING) plan.stages = GEMM_SMEM_RING / sb;
    if (plan.stages > nkb) plan.stages = nkb < 2 ? 2 : nkb;
    plan.splits = 1;
    plan.kbps = nkb;
    if (a->force_splits > 1 && !persist) {
      plan.kbps = (nkb + a->force_splits - 1) / a->force_splits;
      plan.splits = (nkb + plan.kbps - 1) / plan.kbps;
    }
  }
  if (ln_any && plan.splits > 1) return EA_ERR_ARG;
  const int BN = plan.BN, RP = plan.rp;
  if (a->act == EA_ACT_GEGLU && (a->N % 128 != 0 || BN != 128)) return EA_ERR_SHAPE;
  const int n_tiles = (a->N + BN - 1) / BN;
  const int m_items = (m_tiles + RP - 1) / RP;
  const long long tiles = (long long)m_items * n_tiles;      // work items (CTAs without split-K) per group
  if (plan.splits > 1 &&
      (!ws_floats || tiles * G > 8192 || tiles * G * plan.splits * (long long)(RP * BM * BN) > ws_floats))
    return EA_ERR_SHAPE;
  // the spinning split-K fix-up makes split CTAs wait for their siblings: every CTA of the grid must be resident at
  // once (one per SM; the planner guarantees it, forced test configurations are checked here instead of deadlocking)
  if (plan.splits > 1 && tiles * G * plan.splits > (long long)sm_count()) return EA_ERR_SHAPE;

  int stages = plan.stages;
  if (stages > 8) stages = 8;
  if (stages < 2) stages = 2;
  const int smem_bytes = gemm_region_bytes(BN, stages, RP) + (2 * stages + 2) * 8 + gemm_cb_bytes(RP) + 1024;
  const long long tiles_per_group = tiles * plan.splits;
  for (int g = 0; g < G; ++g) {
    GemmKParams& p = L.g[g].p;
    const ea_gemm_args* ag = &args[g];
    p.BN = BN;
    p.stages = stages;
    p.splits = plan.splits;
    p.kb_per_split = plan.kbps;
    if (p.splits > 1) {   // every group has its own counters and partial tiles in the (shared) workspace
      p.cnt = reinterpret_cast<int*>(a->workspace) + 2 * g * tiles;
      p.ws = reinterpret_cast<float*>(reinterpret_cast<char*>(a->workspace) + 65536) +
             (size_t)g * tiles * p.splits * (RP * BM * BN);
    }
    const long long ldw = ag->ldw > 0 ? ag->ldw : sh0.Ktot;
    if (encode_2d(&L.g[g].tmB, ag->w, (uint64_t)sh0.Ktot, (uint64_t)ag->N, (uint64_t)ldw * 2, BK, (uint32_t)BN))
      return EA_ERR_TMAP;
  }
  // The evict-first hint on W pays where a weight tile is used within about one wave (<= 64 row tiles per network: the
  // step at 1 image / GPU, SAM).  With thousands of row tiles (VAE: M up to 262144; 4 images / GPU at 64x64) the same
  // weight tile is re-read wave after wave: plain loads there.
  if (m_tiles > 64)
    for (int g = 0; g < G; ++g) L.g[g].p.b_policy = 0ull;
  const long long total = tiles_per_group * G;
  const int grid = (int)(persist && total > sm_count() ? sm_count() : total);
  for (int g = 0; g < G; ++g)   // L2 prefetch hints: the launch's first CTAs share each group's range
    L.g[g].p.pf_ctas = grid < sm_count() ? grid : sm_count();

  cudaError_t le;
  int rc = EA_OK;
  if (G == 1) {
    GemmLaunch<1> L1;
    L1.g[0] = L.g[0];
    le = launch_gemm_bn<1>(BN, RP, L1, grid, smem_bytes, (int)tiles_per_group, m_items, G, stream, rc);
  } else {
    le = launch_gemm_bn<GEMM_MAX_GROUPS>(BN, RP, L, grid, smem_bytes, (int)tiles_per_group, m_items, G, stream, rc);
  }
  if (rc) return rc;
  ea_count_launch();
  if (le != cudaSuccess) return ea_cuda_fail(le, "ea_gemm: kernel launch");
  const cudaError_t ke = cudaGetLastError();
  return ke == cudaSuccess ? 0 : ea_cuda_fail(ke, "ea_gemm: after the kernel launch");
}

extern "C" int ea_gemm(const ea_gemm_args* a, void* stream) { return ea_gemm_grouped(a, 1, stream); }
