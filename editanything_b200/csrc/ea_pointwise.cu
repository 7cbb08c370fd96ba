// ea_pointwise.cu — the HBM/L2-bound operators around the tensor-core kernels (sm_90a).
// GroupNorm(+SiLU), LayerNorm, small direct convolutions, nearest upsample, the tiny
// time-embedding linears, the fused out-conv + CFG + DDIM step, and the SAM window helpers.
// All use 16-byte vector accesses on channels-last data and warp-shuffle reductions.
#include "ea_common.cuh"
#include "ea_internal.h"

namespace ea {

// ------------------------------- GroupNorm ---------------------------------
// ONE launch: every CTA owns a run of pixels of one image, keeps it in shared memory, reduces its
// per-group sum / sum-of-squares in registers (thread <-> fixed 8-channel vector, so no atomics in
// the loop), publishes its 2*groups partials (plain stores, one slot per CTA), waits on a per-image arrival counter
// (all CTAs are resident: grid <= #SMs), then normalises + affine (+SiLU) straight out of shared
// memory.  The tensor is read from HBM/L2 once and written once.  Workspace layout per image b:
// ws[b*(2G+2) + 0..2G) = {sum, sumsq} per group, then two int counters {arrived, done}; it must be
// zero before the first launch and is left zero by the last CTA of each image.
__device__ __forceinline__ int gn_ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Affine parameters per network group: images [g * ipg, (g + 1) * ipg) use gamma[g] / beta[g] (the UNet encoder and the
// ControlNets run the same layer on stacked activations with their own weights); ipg = 0 -> one set for all images.
struct GnAffine {
  const float* gamma[3];
  const float* beta[3];
  int ipg;
};

__global__ void __launch_bounds__(512, 1)
gn_fused_kernel(const ea_half* __restrict__ x, long long ldx, int C1,
                const ea_half* __restrict__ x2, long long ldx2,
                const GnAffine aff,
                ea_half* __restrict__ out, long long ldo, int HW, int C, int groups, float eps,
                int silu, int chunks, int ppc, int cached, int part_bytes, int phase,
                float* __restrict__ ws) {
  pdl_launch_dependents();
  const int net = aff.ipg > 0 ? (int)blockIdx.y / aff.ipg : 0;
  const float* __restrict__ gamma = net == 0 ? aff.gamma[0] : net == 1 ? aff.gamma[1] : aff.gamma[2];
  const float* __restrict__ beta = net == 0 ? aff.beta[0] : net == 1 ? aff.beta[1] : aff.beta[2];
  // the affine parameters are weights, not the previous kernel's output: fetch them before the dependency wait
  float4 ga = make_float4(0.f, 0.f, 0.f, 0.f), gb = ga, ba = ga, bb = ga;
  {
    const int nvec0 = C >> 3, v0 = threadIdx.x % nvec0;
    if ((int)threadIdx.x / nvec0 < (int)blockDim.x / nvec0) {
      ga = __ldg(reinterpret_cast<const float4*>(gamma + (v0 << 3)));
      gb = __ldg(reinterpret_cast<const float4*>(gamma + (v0 << 3) + 4));
      ba = __ldg(reinterpret_cast<const float4*>(beta + (v0 << 3)));
      bb = __ldg(reinterpret_cast<const float4*>(beta + (v0 << 3) + 4));
    }
  }
  pdl_wait();
  extern __shared__ __align__(16) uint8_t gn_smem[];
  float* sh = reinterpret_cast<float*>(gn_smem);                  // [2*groups]
  float* part = reinterpret_cast<float*>(gn_smem + 512);          // [lanes][2][C] per-lane partials
  uint4* cache = reinterpret_cast<uint4*>(gn_smem + 512 + part_bytes);  // [ppc][nvec] (if cached)
  const int b = blockIdx.y;
  const int p0 = blockIdx.x * ppc;
  const int p1 = min(HW, p0 + ppc);
  const int nvec = C >> 3;
  const int cpg = C / groups;
  const int lanes = blockDim.x / nvec;       // pixel lanes
  const int v = threadIdx.x % nvec;
  const int pl = threadIdx.x / nvec;
  const bool active = pl < lanes;
  const int c = v << 3;
  // workspace: [B][2] int counters {arrived, done}, then one slot of 2*groups partial sums per (image, CTA): every
  // CTA publishes its partials with plain stores and every CTA sums them back in the same fixed order - no
  // floating-point atomics, so the statistics (and everything downstream) are bit-reproducible run to run
  int* cnt = reinterpret_cast<int*>(ws) + 2 * b;
  float* pws_b = ws + 2 * gridDim.y + (size_t)b * chunks * (2 * groups);
  // phase 0: fused (pass 1, image-wide spin barrier, pass 2).  phases 1 / 2: the two passes as
  // SEPARATE launches without any inter-CTA wait - used when several streams run concurrently and
  // a spinning, partially resident grid could starve another one (no co-residency guarantee then).
  for (int i = threadIdx.x; i < groups * 2; i += blockDim.x) sh[i] = 0.f;
  __syncthreads();
  const ea_half* src;
  long long lds;
  if (c < C1) { src = x + c; lds = ldx; } else { src = x2 + (c - C1); lds = ldx2; }
  // Shifted statistics: the sums are of (x - k_g), with k_g the value of group g's first channel at the image's first
  // pixel (the same element for every CTA, so the result stays deterministic).  The one-pass variance
  // E[(x-k)^2] - E[x-k]^2 then loses precision with (mean - k)^2 / var instead of mean^2 / var, which is large for
  // groups whose mean sits far from zero relative to their spread.
  float shift[8];
  {
    int gprev = -1;
    float kv = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int g = (c + j) / cpg;
      if (g != gprev) {
        const int ch = g * cpg;
        kv = ea_h2f(ch < C1 ? x[(long long)b * HW * ldx + ch] : x2[(long long)b * HW * ldx2 + (ch - C1)]);
        gprev = g;
      }
      shift[j] = kv;
    }
  }
  if (phase != 2) {
  // ---- pass 1: load (cache) + per-thread, per-channel partial sums (the thread's 8 channels
  //      are fixed, so their groups are too: shared-memory atomics only once, after the loop)
  float cs[8], cq[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { cs[j] = 0.f; cq[j] = 0.f; }
  if (active) {
#ifndef EA_GN_NO_ASYNC
    if (cached) {
      // every pixel of this thread goes global -> shared memory asynchronously: all of its loads are in flight at
      // once (ONE L2 round trip) instead of four at a time through registers (a chain of ~8 round trips whatever the
      // tensor size)
      for (int pp = p0 + pl; pp < p1; pp += lanes) {
        const uint32_t dst = (uint32_t)__cvta_generic_to_shared(&cache[(pp - p0) * nvec + v]);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src + ((long long)b * HW + pp) * lds) : "memory");
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 0;" ::: "memory");
#pragma unroll 4
      for (int pp = p0 + pl; pp < p1; pp += lanes) {
        const uint4 u = cache[(pp - p0) * nvec + v];
        float2 f0 = ea_unpack2(u.x), f1 = ea_unpack2(u.y), f2 = ea_unpack2(u.z), f3 = ea_unpack2(u.w);
        float vals[8] = {f0.x, f0.y, f1.x, f1.y, f2.x, f2.y, f3.x, f3.y};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = vals[j] - shift[j];
          cs[j] += d;
          cq[j] += d * d;
        }
      }
    } else
#endif
    {
#pragma unroll 8
    for (int pp = p0 + pl; pp < p1; pp += lanes) {
      uint4 u = __ldg(reinterpret_cast<const uint4*>(src + ((long long)b * HW + pp) * lds));
      if (cached) cache[(pp - p0) * nvec + v] = u;
      float2 f0 = ea_unpack2(u.x), f1 = ea_unpack2(u.y), f2 = ea_unpack2(u.z), f3 = ea_unpack2(u.w);
      float vals[8] = {f0.x, f0.y, f1.x, f1.y, f2.x, f2.y, f3.x, f3.y};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = vals[j] - shift[j];
        cs[j] += d;
        cq[j] += d * d;
      }
    }
    }
    // per-(pixel lane, channel) partials -> shared memory (no atomics: 480 threads x 16 contended
    // shared atomics per launch)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      part[(pl * 2 + 0) * C + c + j] = cs[j];
      part[(pl * 2 + 1) * C + c + j] = cq[j];
    }
  }
  __syncthreads();
  if (threadIdx.x < groups * 2) {   // one thread per (group, sum | sumsq): lanes x cpg adds
    const int g = threadIdx.x >> 1, which = threadIdx.x & 1;
    float acc = 0.f;
    for (int l = 0; l < lanes; ++l) {
      const float* pp = part + (l * 2 + which) * C + g * cpg;
      for (int j = 0; j < cpg; ++j) acc += pp[j];
    }
    sh[threadIdx.x] = acc;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < groups * 2; i += blockDim.x) __stcg(&pws_b[(size_t)blockIdx.x * (2 * groups) + i], sh[i]);
  __threadfence();
  __syncthreads();
  if (phase == 1) return;
  // ---- image-wide barrier
  if (threadIdx.x == 0) {
    atomicAdd(cnt, 1);
    uint32_t spins = 0;
    while (gn_ld_acquire(cnt) < chunks) {
      __nanosleep(32);
      if (++spins > (1u << 24)) { asm volatile("trap;"); }
    }
  }
  __syncthreads();
  __threadfence();
  }  // phase != 2
  // ---- pass 2: y = x * a + b with a = rstd*gamma, b = beta - mean*a (per channel of this thread)
  // the image's 2*groups statistics come back in ONE L2 round trip (per-thread dependent loads of
  // "its" groups cost several serialized round trips)
  __syncthreads();
  {
    // sum of the image's per-CTA partials in a fixed order: `parts` threads per statistic take every parts-th CTA
    // (independent loads: one or two L2 round trips), then one thread per statistic adds the parts in order
    const int g2 = 2 * groups;
    int parts = (int)blockDim.x / g2;
    const int cap = part_bytes / (g2 * (int)sizeof(float));
    if (parts > cap) parts = cap;
    if (parts < 1) parts = 1;
    const int i = threadIdx.x % g2, pidx = threadIdx.x / g2;
    if (pidx < parts) {
      float acc = 0.f;
      for (int cidx = pidx; cidx < chunks; cidx += parts) acc += __ldcg(&pws_b[(size_t)cidx * g2 + i]);
      part[pidx * g2 + i] = acc;
    }
    __syncthreads();
    if (threadIdx.x < g2) {
      float acc = 0.f;
      for (int q = 0; q < parts; ++q) acc += part[q * g2 + threadIdx.x];
      sh[threadIdx.x] = acc;
    }
  }
  __syncthreads();
  if (active) {
    const float inv_n = 1.0f / ((float)HW * (float)cpg);
    float av[8], bv[8];
    {
      float gm[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
      float bt[8] = {ba.x, ba.y, ba.z, ba.w, bb.x, bb.y, bb.z, bb.w};
      int gprev = -1;
      float mean = 0.f, rstd = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int g = (c + j) / cpg;
        if (g != gprev) {
          const float s = sh[g * 2], q = sh[g * 2 + 1];
          const float dm = s * inv_n;                  // mean of (x - k_g)
          mean = shift[j] + dm;
          rstd = rsqrtf(fmaxf(q * inv_n - dm * dm, 0.f) + eps);
          gprev = g;
        }
        av[j] = rstd * gm[j];
        bv[j] = bt[j] - mean * av[j];
      }
    }
    for (int pp = p0 + pl; pp < p1; pp += lanes) {
      uint4 u = cached ? cache[(pp - p0) * nvec + v]
                       : __ldg(reinterpret_cast<const uint4*>(src + ((long long)b * HW + pp) * lds));
      float2 f0 = ea_unpack2(u.x), f1 = ea_unpack2(u.y), f2 = ea_unpack2(u.z), f3 = ea_unpack2(u.w);
      float vals[8] = {f0.x, f0.y, f1.x, f1.y, f2.x, f2.y, f3.x, f3.y};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float y = fmaf(vals[j], av[j], bv[j]);
        vals[j] = silu ? silu_f(y) : y;
      }
      *reinterpret_cast<uint4*>(out + ((long long)b * HW + pp) * ldo + c) =
          make_uint4(ea_pack2(vals[0], vals[1]), ea_pack2(vals[2], vals[3]),
                     ea_pack2(vals[4], vals[5]), ea_pack2(vals[6], vals[7]));
    }
  }
  // ---- leave the counters zero for the next launch (the partial slots are simply overwritten)
  __syncthreads();
  if (phase == 0 && threadIdx.x == 0) {
    int old = atomicAdd(cnt + 1, 1);
    if (old == chunks - 1) {
      cnt[0] = 0;
      cnt[1] = 0;
    }
  }
}

// ------------------------------- LayerNorm ---------------------------------
static constexpr int LN_MAXV = 8;  // C <= 8 * 32 * 8 = 2048
__global__ void layernorm_kernel(const ea_half* __restrict__ x, long long ldx,
                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                 ea_half* __restrict__ out, long long ldo, int M, int C,
                                 float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int warps_per_cta = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * warps_per_cta + (threadIdx.x >> 5);
  if (row >= M) return;
  const int nvec = C >> 3;
  uint4 regs[LN_MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    int v = lane + i * 32;
    if (v < nvec) {
      regs[i] = __ldg(reinterpret_cast<const uint4*>(x + row * ldx + (v << 3)));
      float2 a = ea_unpack2(regs[i].x), b = ea_unpack2(regs[i].y), c = ea_unpack2(regs[i].z),
             d = ea_unpack2(regs[i].w);
      s += a.x + a.y + b.x + b.y + c.x + c.y + d.x + d.y;
    }
  }
  s = warp_sum(s);
  const float mean = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    int v = lane + i * 32;
    if (v < nvec) {
      float2 a = ea_unpack2(regs[i].x), b = ea_unpack2(regs[i].y), c = ea_unpack2(regs[i].z),
             d = ea_unpack2(regs[i].w);
      float t;
      t = a.x - mean; q += t * t; t = a.y - mean; q += t * t;
      t = b.x - mean; q += t * t; t = b.y - mean; q += t * t;
      t = c.x - mean; q += t * t; t = c.y - mean; q += t * t;
      t = d.x - mean; q += t * t; t = d.y - mean; q += t * t;
    }
  }
  q = warp_sum(q);
  const float rstd = rsqrtf(q / (float)C + eps);
#pragma unroll
  for (int i = 0; i < LN_MAXV; ++i) {
    int v = lane + i * 32;
    if (v < nvec) {
      int c0 = v << 3;
      float2 a = ea_unpack2(regs[i].x), b = ea_unpack2(regs[i].y), c = ea_unpack2(regs[i].z),
             d = ea_unpack2(regs[i].w);
      float vals[8] = {a.x, a.y, b.x, b.y, c.x, c.y, d.x, d.y};
      float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c0));
      float4 gb = __ldg(reinterpret_cast<const float4*>(gamma + c0 + 4));
      float4 ba = __ldg(reinterpret_cast<const float4*>(beta + c0));
      float4 bb = __ldg(reinterpret_cast<const float4*>(beta + c0 + 4));
      float gm[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
      float bt[8] = {ba.x, ba.y, ba.z, ba.w, bb.x, bb.y, bb.z, bb.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) vals[j] = (vals[j] - mean) * rstd * gm[j] + bt[j];
      uint4 o = make_uint4(ea_pack2(vals[0], vals[1]), ea_pack2(vals[2], vals[3]),
                           ea_pack2(vals[4], vals[5]), ea_pack2(vals[6], vals[7]));
      *reinterpret_cast<uint4*>(out + row * ldo + c0) = o;
    }
  }
}

// ---------------------------- direct small conv ----------------------------
// thread <-> (pixel, cout); weights [k,k,Cin,Cout] fp32 so a warp (consecutive cout) reads them
// coalesced while the input pixel values are warp-broadcast.
__global__ void conv_direct_kernel(const ea_half* __restrict__ x, const float* __restrict__ w,
                                   const float* __restrict__ bias, ea_half* __restrict__ out,
                                   int B, int Hin, int Win, int Cin, int Cout, int ks, int stride,
                                   int silu, const ea_half* __restrict__ add, long long ldo) {
  pdl_launch_dependents();
  pdl_wait();
  const int Ho = (Hin + stride - 1) / stride, Wo = (Win + stride - 1) / stride;
  const long long total = (long long)B * Ho * Wo * Cout;
  const int pad = ks / 2;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int co = (int)(idx % Cout);
    long long pix = idx / Cout;
    int wo = (int)(pix % Wo);
    int ho = (int)((pix / Wo) % Ho);
    int b = (int)(pix / ((long long)Wo * Ho));
    float acc = bias ? __ldg(bias + co) : 0.f;
    for (int kh = 0; kh < ks; ++kh) {
      int hi = ho * stride + kh - pad;
      if (hi < 0 || hi >= Hin) continue;
      for (int kw = 0; kw < ks; ++kw) {
        int wi = wo * stride + kw - pad;
        if (wi < 0 || wi >= Win) continue;
        const ea_half* xp = x + (((long long)b * Hin + hi) * Win + wi) * Cin;
        const float* wp = w + ((long long)(kh * ks + kw) * Cin) * Cout + co;
        for (int c = 0; c < Cin; ++c) acc += ea_h2f(xp[c]) * __ldg(wp + (long long)c * Cout);
      }
    }
    if (silu) acc = silu_f(acc);
    if (add) acc += ea_h2f(add[idx]);
    out[pix * ldo + co] = ea_f2h(acc);
  }
}

__global__ void upsample2x_kernel(const ea_half* __restrict__ x, ea_half* __restrict__ out, int B,
                                  int H, int W, int C) {
  pdl_launch_dependents();
  pdl_wait();
  const int nvec = C >> 3;
  const long long total = (long long)B * (2 * H) * (2 * W) * nvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int v = (int)(idx % nvec);
    long long pix = idx / nvec;
    int wo = (int)(pix % (2 * W));
    int ho = (int)((pix / (2 * W)) % (2 * H));
    int b = (int)(pix / ((long long)4 * W * H));
    const uint4* src = reinterpret_cast<const uint4*>(
        x + (((long long)b * H + (ho >> 1)) * W + (wo >> 1)) * C + (v << 3));
    *reinterpret_cast<uint4*>(out + pix * C + (v << 3)) = __ldg(src);
  }
}

// y[M,N] = act_out(W[N,K] x act_in(x[M,K]) + b); one warp per output column n, M <= 16.
__global__ void small_linear_kernel(const float* __restrict__ x, const ea_half* __restrict__ w,
                                    const float* __restrict__ bias, float* __restrict__ y, int M,
                                    int N, int K, int silu_in, int silu_out) {
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  float acc[16];
#pragma unroll
  for (int m = 0; m < 16; ++m) acc[m] = 0.f;
  const ea_half* wr = w + (long long)n * K;
  for (int k = lane * 8; k < K; k += 32 * 8) {
    uint4 u = __ldg(reinterpret_cast<const uint4*>(wr + k));
    float2 a = ea_unpack2(u.x), b = ea_unpack2(u.y), c = ea_unpack2(u.z), d = ea_unpack2(u.w);
    float wv[8] = {a.x, a.y, b.x, b.y, c.x, c.y, d.x, d.y};
#pragma unroll
    for (int m = 0; m < 16; ++m) {
      if (m < M) {
        const float* xr = x + (long long)m * K + k;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float xv = __ldg(xr + j);
          if (silu_in) xv = silu_f(xv);
          acc[m] += wv[j] * xv;
        }
      }
    }
  }
#pragma unroll
  for (int m = 0; m < 16; ++m) {
    if (m < M) {
      float s = warp_sum(acc[m]);
      if (lane == 0) {
        s += bias ? __ldg(bias + n) : 0.f;
        if (silu_out) s = silu_f(s);
        y[(long long)m * N + n] = s;
      }
    }
  }
}

// util.py:154-174: freqs = exp(-ln(10000) * i / half), emb = [cos(t f) | sin(t f)]
__global__ void timestep_embedding_kernel(const float* __restrict__ t, float* __restrict__ out,
                                          int B, int dim) {
  pdl_launch_dependents();
  pdl_wait();
  const int half = dim / 2;
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * half) return;
  int b = idx / half, i = idx - b * half;
  float f = expf(-9.210340371976184f * (float)i / (float)half);
  float a = t[b] * f;
  out[(long long)b * dim + i] = cosf(a);
  out[(long long)b * dim + half + i] = sinf(a);
}

// ---------------- out conv (C -> 4) + CFG + DDIM + inpaint blend -------------
// One warp per (image, pixel).  kCfg: xn, eps_out and lat_half hold 2*Nimg rows (unconditional first) and both
// halves are reduced by the same warp, so the guidance combine and the DDIM update happen in registers.  !kCfg:
// they hold the Nimg rows alone and the update reads their eps directly (sampling without guidance).
// kV: the network predicts v = sqrt(a) eps - sqrt(1-a) x0 (v-prediction base models such as SD2.1-768); the update
// converts the (guidance-combined) output to x0 and eps first.  eps_out stays the raw network output either way.
template <bool kCfg, bool kV>
__global__ void out_ddim_kernel(const ea_half* __restrict__ xn, const float* __restrict__ w,
                                    const float* __restrict__ bias, float* __restrict__ latents,
                                    float* __restrict__ eps_out, const float* __restrict__ coef,
                                    float guidance, const float* __restrict__ known,
                                    const float* __restrict__ noise,
                                    const float* __restrict__ mask, ea_half* __restrict__ lat_half,
                                    int* __restrict__ step_ctr, float* __restrict__ hist, int Nimg, int H, int W,
                                    int C) {
  pdl_launch_dependents();
  pdl_wait();
  // device-side step counter of the captured loop: the first kernel of the step (step_gather_kernel) read it,
  // this last one advances it - stream order makes that race-free
  if (step_ctr && blockIdx.x == 0 && threadIdx.x == 0) *step_ctr = *step_ctr + 1;
  const int lane = threadIdx.x & 31;
  const long long gw = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long npix = (long long)Nimg * H * W;
  if (gw >= npix) return;
  const int img = (int)(gw / ((long long)H * W));
  const int rem = (int)(gw - (long long)img * H * W);
  const int h = rem / W, wq = rem - h * W;
  float au[4] = {0.f, 0.f, 0.f, 0.f}, ac[4] = {0.f, 0.f, 0.f, 0.f};
  for (int kh = 0; kh < 3; ++kh) {
    int hi = h + kh - 1;
    if (hi < 0 || hi >= H) continue;
    for (int kw = 0; kw < 3; ++kw) {
      int wi = wq + kw - 1;
      if (wi < 0 || wi >= W) continue;
      const ea_half* pu = xn + (((long long)img * H + hi) * W + wi) * C;
      const ea_half* pc = kCfg ? xn + (((long long)(img + Nimg) * H + hi) * W + wi) * C : nullptr;
      const float* wt = w + (kh * 3 + kw) * C;  // + o*9*C
      for (int c = lane * 8; c < C; c += 256) {
        uint4 uu = __ldg(reinterpret_cast<const uint4*>(pu + c));
        float2 a0 = ea_unpack2(uu.x), a1 = ea_unpack2(uu.y), a2 = ea_unpack2(uu.z),
               a3 = ea_unpack2(uu.w);
        float xu[8] = {a0.x, a0.y, a1.x, a1.y, a2.x, a2.y, a3.x, a3.y};
        float xc[8];
        if constexpr (kCfg) {
          uint4 uc = __ldg(reinterpret_cast<const uint4*>(pc + c));
          float2 b0 = ea_unpack2(uc.x), b1 = ea_unpack2(uc.y), b2 = ea_unpack2(uc.z),
                 b3 = ea_unpack2(uc.w);
          xc[0] = b0.x; xc[1] = b0.y; xc[2] = b1.x; xc[3] = b1.y;
          xc[4] = b2.x; xc[5] = b2.y; xc[6] = b3.x; xc[7] = b3.y;
        }
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          const float* wo = wt + (long long)o * 9 * C + c;
          float4 w0 = __ldg(reinterpret_cast<const float4*>(wo));
          float4 w1 = __ldg(reinterpret_cast<const float4*>(wo + 4));
          float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            au[o] += wv[j] * xu[j];
            if constexpr (kCfg) ac[o] += wv[j] * xc[j];
          }
        }
      }
    }
  }
#pragma unroll
  for (int o = 0; o < 4; ++o) {
    au[o] = warp_sum(au[o]);
    if constexpr (kCfg) ac[o] = warp_sum(ac[o]);
  }
  if (lane < 4) {
    const int o = lane;
    float eu = (o == 0 ? au[0] : o == 1 ? au[1] : o == 2 ? au[2] : au[3]) + bias[o];
    float ec = 0.f;
    if constexpr (kCfg) ec = (o == 0 ? ac[0] : o == 1 ? ac[1] : o == 2 ? ac[2] : ac[3]) + bias[o];
    if (eps_out) {
      eps_out[gw * 4 + o] = eu;
      if constexpr (kCfg) eps_out[(gw + npix) * 4 + o] = ec;
    }
    if (latents) {
      // cldm/ddim_hacked.py:192 (applied to v as well, :190-192); without guidance the network output itself
      // (:187-188)
      float m = kCfg ? eu + guidance * (ec - eu) : eu;
      float sa = coef[0], s1a = coef[1], sap = coef[2], s1ap = coef[3];
      float xt = latents[gw * 4 + o];
      float x0, e;
      if constexpr (kV) {
        x0 = sa * xt - s1a * m;             // :217, ddpm.py:290-296 (predict_start_from_z_and_v)
        e = sa * m + s1a * xt;              // :195, ddpm.py:298-302 (predict_eps_from_z_and_v)
      } else {
        e = m;
        x0 = (xt - s1a * e) / sa;           // :215
      }
      float xp = sap * x0 + s1ap * e;       // :226-230 (eta = 0)
      if (hist && coef[7] != 0.f) {
        // Linear multistep predictor-corrector (UniPC, the scheduler every reference entry point installs:
        // editany_lora.py:383,418) - all coefficients are functions of the timestep table, precomputed per step:
        //   xc = kx x + kl last + k1 m1 + k2 m2 + k0 x0    (corrector; identity on the first step)
        //   x' = px xc + p0 x0 + p1 m1                     (predictor for the next timestep)
        //   m2 <- m1, m1 <- x0, last <- xc                 (history of x0 predictions / corrected samples)
        const long long n4 = npix * 4, idx = gw * 4 + o;
        const float m1 = hist[idx], m2 = hist[n4 + idx], last = hist[2 * n4 + idx];
        const float xc = coef[8] * xt + coef[9] * last + coef[10] * m1 + coef[11] * m2 + coef[12] * x0;
        xp = coef[13] * xc + coef[14] * x0 + coef[15] * m1;
        hist[n4 + idx] = m1;
        hist[idx] = x0;
        hist[2 * n4 + idx] = xc;
      }
      if (known) {
        // inpaint blend (utils/stable_diffusion_controlnet_inpaint.py:1647-1656).  With `noise` the kept
        // region is re-noised here: add_noise(init, noise, t_next) = coef[4] * init + coef[5] * noise, and
        // coef[6] switches the blend per step (alignment_ratio window) without touching the launch.
        float mk = mask[gw];
        float kn = known[gw * 4 + o];
        if (noise) {
          kn = coef[4] * kn + coef[5] * noise[gw * 4 + o];
          mk *= coef[6];
        }
        xp = kn * mk + xp * (1.f - mk);
      }
      latents[gw * 4 + o] = xp;
      if (lat_half) {
        lat_half[gw * 4 + o] = ea_f2h(xp);
        if constexpr (kCfg) lat_half[(gw + npix) * 4 + o] = ea_f2h(xp);
      }
    }
  }
}

// ---------------- alpha-mixing of the latents (last kernel of a mixing pipeline's step) -------------
// utils/stable_diffusion_controlnet_inpaint.py:2039-2051, after the scheduler update of step r = *ctr - 1 (the
// epilogue before this kernel has advanced the counter).  One thread per latent pixel (4 fp32 channels).
//   p = k_init * known + k_noise * noise[r]                    (add_noise(init, randn, t_{r+1}))
//   x = m * (in_window ? p : x) + (1 - m) * ((1 - alpha) x + alpha p)
// Rows with active == 0 (the last step) and counters outside [1, n_rows] leave everything untouched.
__global__ void latent_mix_kernel(float* __restrict__ latents, const float* __restrict__ known,
                                  const float* __restrict__ mask, const float* __restrict__ noise,
                                  const float* __restrict__ mix, float alpha, const int* __restrict__ ctr,
                                  int n_rows, ea_half* __restrict__ lat_half, int copies, long long npix) {
  pdl_launch_dependents();
  pdl_wait();
  const int r = *ctr - 1;
  if (r < 0 || r >= n_rows) return;
  const float k_init = mix[r * 4 + 0], k_noise = mix[r * 4 + 1], in_window = mix[r * 4 + 2];
  if (mix[r * 4 + 3] == 0.f) return;
  const float* z = noise + (long long)r * npix * 4;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += stride) {
    const float m = mask[p];
    const float4 x = reinterpret_cast<const float4*>(latents)[p];
    const float4 k = __ldg(reinterpret_cast<const float4*>(known) + p);
    const float4 n = __ldg(reinterpret_cast<const float4*>(z) + p);
    float xv[4] = {x.x, x.y, x.z, x.w};
    const float kv[4] = {k.x, k.y, k.z, k.w}, nv[4] = {n.x, n.y, n.z, n.w};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float pv = k_init * kv[c] + k_noise * nv[c];
      const float keep = in_window != 0.f ? pv : xv[c];
      xv[c] = keep * m + ((1.f - alpha) * xv[c] + alpha * pv) * (1.f - m);
    }
    reinterpret_cast<float4*>(latents)[p] = make_float4(xv[0], xv[1], xv[2], xv[3]);
    if (lat_half) {
      ea_half h4[4] = {ea_f2h(xv[0]), ea_f2h(xv[1]), ea_f2h(xv[2]), ea_f2h(xv[3])};
      const uint2 hv = *reinterpret_cast<const uint2*>(h4);
      for (int c = 0; c < copies; ++c) reinterpret_cast<uint2*>(lat_half)[c * npix + p] = hv;
    }
  }
}

// ---------------- per-step table gather (first kernel of a captured denoising step) -------------
// Everything that changes from step to step (the scheduler coefficients and every net's time-embedding rows)
// lives in device tables with one row per step; this kernel copies row min(*ctr, n_rows - 1) of each table into
// the fixed buffers the captured step reads, so the host's per-step work is ONE graph launch.
struct StepTables {
  int n;
  const float* src[EA_STEP_MAX_TABLES];
  float* dst[EA_STEP_MAX_TABLES];
  long long row_elems[EA_STEP_MAX_TABLES];
};
__global__ void step_gather_kernel(const int* __restrict__ ctr, int n_rows, const StepTables tb) {
  pdl_launch_dependents();
  pdl_wait();
  int row = *ctr;
  row = row < 0 ? 0 : (row >= n_rows ? n_rows - 1 : row);
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (int k = 0; k < tb.n; ++k) {
    const float* s = tb.src[k] + (long long)row * tb.row_elems[k];
    float* d = tb.dst[k];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < tb.row_elems[k]; i += stride) d[i] = __ldg(s + i);
  }
}

// ------------------------------ SAM helpers --------------------------------
// Decomposed relative-position terms (HF modeling_sam.py:789-801):
//   rel_h[bh, (qh,qw), kh] = sum_c q[b,(qh,qw),h,c] * Rh[qh, kh, c]      (blockIdx.z = 0, CTA <-> fixed qh)
//   rel_w[bh, (qh,qw), kw] = sum_c q[b,(qh,qw),h,c] * Rw[qw, kw, c]      (blockIdx.z = 1, CTA <-> fixed qw)
// One CTA = one (fixed coordinate f, batch*head): the S query rows that share R[f] and the S x d
// table slice live in shared memory (row stride d+1 floats: conflict-free), thread <-> output
// column k, looping over the S rows (q[row][c] is a warp broadcast).
__global__ void sam_relpos_kernel(const ea_half* __restrict__ q, long long q_bs, long long q_ns,
                                  const float* __restrict__ Rh, const float* __restrict__ Rw,
                                  float* __restrict__ rel_h, float* __restrict__ rel_w, int B,
                                  int heads, int S, int d) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float rp_sm[];
  const int f = blockIdx.x;              // fixed coordinate: qh (z = 0) or qw (z = 1)
  const int bh = blockIdx.y;
  const bool is_h = blockIdx.z == 0;
  const int b = bh / heads, hd = bh - b * heads;
  const int ld = d + 1;
  float* qs = rp_sm;                     // [S][d+1]
  float* rs = rp_sm + S * ld;            // [S][d+1]
  const float* R = (is_h ? Rh : Rw) + (long long)f * S * d;
  for (int i = threadIdx.x; i < S * d; i += blockDim.x) {
    const int row = i / d, c = i - row * d;
    rs[row * ld + c] = __ldg(R + i);
    const int qi = is_h ? f * S + row : row * S + f;   // the S queries that share R[f]
    qs[row * ld + c] = ea_h2f(q[(long long)b * q_bs + (long long)qi * q_ns + (long long)hd * d + c]);
  }
  __syncthreads();
  float* dst = is_h ? rel_h : rel_w;
  for (int o = threadIdx.x; o < S * S; o += blockDim.x) {
    const int row = o / S, k = o - row * S;
    const float* qr = qs + row * ld;
    const float* rr = rs + k * ld;
    float acc = 0.f;
#pragma unroll 8
    for (int c = 0; c < d; ++c) acc = fmaf(qr[c], rr[c], acc);
    const int qi = is_h ? f * S + row : row * S + f;
    dst[((long long)bh * S * S + qi) * S + k] = acc;
  }
}

__global__ void window_partition_kernel(const ea_half* __restrict__ x, ea_half* __restrict__ out,
                                        int B, int H, int W, int C, int ws, int nWh, int nWw) {
  pdl_launch_dependents();
  pdl_wait();
  const int nvec = C >> 3;
  const long long total = (long long)B * nWh * nWw * ws * ws * nvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int v = (int)(idx % nvec);
    long long t = idx / nvec;
    int j = (int)(t % ws); t /= ws;
    int i = (int)(t % ws); t /= ws;
    int ww = (int)(t % nWw); t /= nWw;
    int wh = (int)(t % nWh);
    int b = (int)(t / nWh);
    int h = wh * ws + i, w = ww * ws + j;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (h < H && w < W)
      val = __ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + h) * W + w) * C + (v << 3)));
    *reinterpret_cast<uint4*>(out + (idx / nvec) * C + (v << 3)) = val;
  }
}

__global__ void window_unpartition_kernel(const ea_half* __restrict__ xw,
                                          const ea_half* __restrict__ residual,
                                          ea_half* __restrict__ out, int B, int H, int W, int C,
                                          int ws, int nWh, int nWw) {
  pdl_launch_dependents();
  pdl_wait();
  const int nvec = C >> 3;
  const long long total = (long long)B * H * W * nvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int v = (int)(idx % nvec);
    long long pix = idx / nvec;
    int w = (int)(pix % W);
    int h = (int)((pix / W) % H);
    int b = (int)(pix / ((long long)W * H));
    int wh = h / ws, i = h - wh * ws, ww = w / ws, j = w - ww * ws;
    long long src = ((((long long)b * nWh + wh) * nWw + ww) * ws + i) * ws + j;
    uint4 u = __ldg(reinterpret_cast<const uint4*>(xw + src * C + (v << 3)));
    if (residual) {
      uint4 r = __ldg(reinterpret_cast<const uint4*>(residual + pix * C + (v << 3)));
      float2 a, b2;
      a = ea_unpack2(u.x); b2 = ea_unpack2(r.x); u.x = ea_pack2(a.x + b2.x, a.y + b2.y);
      a = ea_unpack2(u.y); b2 = ea_unpack2(r.y); u.y = ea_pack2(a.x + b2.x, a.y + b2.y);
      a = ea_unpack2(u.z); b2 = ea_unpack2(r.z); u.z = ea_pack2(a.x + b2.x, a.y + b2.y);
      a = ea_unpack2(u.w); b2 = ea_unpack2(r.w); u.w = ea_pack2(a.x + b2.x, a.y + b2.y);
    }
    *reinterpret_cast<uint4*>(out + pix * C + (v << 3)) = u;
  }
}

// Patch embedding im2col (SAM PatchEmbed: Conv2d(3, C, k=16, s=16)): fp32 NCHW image ->
// half [B*gh*gw, Cin*ps*ps] with K index = (c*ps + kh)*ps + kw, i.e. the flattened conv weight
// order, so the convolution is one ea_gemm.  Thread <-> 8 consecutive kw.
__global__ void patchify_kernel(const float* __restrict__ img, ea_half* __restrict__ out, int B,
                                int Cin, int H, int W, int ps) {
  pdl_launch_dependents();
  pdl_wait();
  const int gh = H / ps, gw = W / ps;
  const int K = Cin * ps * ps;
  const int kvec = K >> 3;
  const long long total = (long long)B * gh * gw * kvec;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    int kv = (int)(idx % kvec);
    long long patch = idx / kvec;
    int pw = (int)(patch % gw);
    int ph = (int)((patch / gw) % gh);
    int b = (int)(patch / ((long long)gw * gh));
    int k = kv << 3;
    int kw = k % ps;
    int kh = (k / ps) % ps;
    int c = k / (ps * ps);
    const float* src = img + (((long long)b * Cin + c) * H + (ph * ps + kh)) * W + pw * ps + kw;
    float4 a = __ldg(reinterpret_cast<const float4*>(src));
    float4 b4 = __ldg(reinterpret_cast<const float4*>(src + 4));
    uint4 o = make_uint4(ea_pack2(a.x, a.y), ea_pack2(a.z, a.w), ea_pack2(b4.x, b4.y),
                         ea_pack2(b4.z, b4.w));
    *reinterpret_cast<uint4*>(out + patch * K + k) = o;
  }
}

// NHWC half -> NCHW fp32 (the layout/precision the reference hands to the prompt/mask decoder).
__global__ void nhwc_to_nchw_f32_kernel(const ea_half* __restrict__ x, float* __restrict__ out,
                                        int B, int HW, int C) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + threadIdx.x;
    if (p < HW && c < C) tile[i][threadIdx.x] = ea_h2f(x[((long long)b * HW + p) * C + c]);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + threadIdx.x;
    if (p < HW && c < C) out[((long long)b * C + c) * HW + p] = tile[threadIdx.x][i];
  }
}

// Row softmax of fp32 logits -> half probabilities (VAE AttnBlock: one head, d = 512, so the logits
// go through two plain GEMMs instead of the flash kernel; ldm/modules/diffusionmodules/model.py:193-201).
// One CTA per row, three passes over a row that stays in L1/L2 (<= 64 KB).
__global__ void softmax_rows_kernel(const float* __restrict__ s, long long lds, ea_half* __restrict__ p,
                                    long long ldp, int cols) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[32];
  const float* row = s + (long long)blockIdx.x * lds;
  ea_half* prow = p + (long long)blockIdx.x * ldp;
  const int tid = threadIdx.x, nw = blockDim.x >> 5;
  float m = -INFINITY;
  for (int i = tid * 4; i < cols; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(row + i);
    m = fmaxf(fmaxf(m, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((tid & 31) == 0) red[tid >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int i = 1; i < nw; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = tid * 4; i < cols; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(row + i);
    sum += (__expf(v.x - m) + __expf(v.y - m)) + (__expf(v.z - m) + __expf(v.w - m));
  }
  sum = warp_sum(sum);
  if ((tid & 31) == 0) red[tid >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < nw; ++i) sum += red[i];
  const float inv = 1.0f / sum;
  for (int i = tid * 4; i < cols; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(row + i);
    uint2 o;
    o.x = ea_pack2(__expf(v.x - m) * inv, __expf(v.y - m) * inv);
    o.y = ea_pack2(__expf(v.z - m) * inv, __expf(v.w - m) * inv);
    *reinterpret_cast<uint2*>(prow + i) = o;
  }
}

// Decoded image: NHWC half (first C channels of rows `ldx` wide) -> fp32 NCHW, out = clamp(x*scale +
// shift, lo, hi): decode_latents' (image / 2 + 0.5).clamp(0, 1) (utils/stable_diffusion_controlnet_
// inpaint.py:718-724) fused with the layout change.  One thread per pixel, planes written coalesced.
__global__ void image_out_kernel(const ea_half* __restrict__ x, long long ldx, float* __restrict__ out,
                                 int B, long long HW, int C, float scale, float shift, float lo, float hi) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * HW) return;
  const long long b = i / HW, pix = i - b * HW;
  const ea_half* px = x + i * ldx;
  for (int c = 0; c < C; ++c) {
    const float v = fminf(fmaxf(fmaf(ea_h2f(px[c]), scale, shift), lo), hi);
    out[(b * C + c) * HW + pix] = v;
  }
}

// 3x3 stride-1 pad-1 convolution with a tiny input depth (conv_in: 4 -> 320, openaimodel.py:533-539,
// and ControlNet `h = conv_in(x) + guided_hint`, cldm/cldm.py:293-297).  K = 9*Cin is far too small for
// the tensor-core path; the whole filter bank lives in shared memory, a thread owns one pixel and 8
// consecutive output channels (16-byte stores), the 9*Cin input taps sit in registers.
template <int CIN>
__global__ void __launch_bounds__(256)
conv_smallcin_kernel(const ea_half* __restrict__ x, const float* __restrict__ w,
                     const float* __restrict__ bias, ea_half* __restrict__ out,
                     long long ldo, ea_half* __restrict__ out2, long long ldo2,
                     const ea_half* __restrict__ add, int B, int H, int W, int Cout) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float wsm[];  // [9*CIN][Cout] + bias[Cout]
  const int nw = 9 * CIN * Cout;
  {  // filter bank -> shared memory, 16-byte loads, all issued before the first use (Cout % 8 == 0)
    const float4* w4 = reinterpret_cast<const float4*>(w);
    float4* s4 = reinterpret_cast<float4*>(wsm);
    for (int i = threadIdx.x; i < (nw >> 2); i += blockDim.x) s4[i] = __ldg(w4 + i);
  }
  for (int i = threadIdx.x; i < Cout; i += blockDim.x) wsm[nw + i] = bias ? bias[i] : 0.f;
  __syncthreads();
  // A thread owns 8 consecutive output channels of PX = 4 horizontally adjacent pixels: every weight read from
  // shared memory feeds 4 FMAs (one pixel per thread makes the kernel shared-memory-bandwidth bound), and a
  // persistent grid loads the 46 KB filter
  // bank once per CTA instead of once per 256 outputs.
  constexpr int PX = 4;
  const int ngrp = Cout >> 3;
  const int wq_n = (W + PX - 1) / PX;
  const long long total = (long long)B * H * wq_n * ngrp;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int g = (int)(idx % ngrp);
    const long long q = idx / ngrp;
    const int wo0 = (int)(q % wq_n) * PX;
    const int ho = (int)((q / wq_n) % H);
    const int b = (int)(q / ((long long)wq_n * H));
    float acc[PX][8];
#pragma unroll
    for (int p = 0; p < PX; ++p)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[p][j] = wsm[nw + g * 8 + j];
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hi = ho + kh - 1;
      if (hi < 0 || hi >= H) continue;
      float xin[PX + 2][CIN];          // input columns wo0 - 1 .. wo0 + PX of row hi (zero outside the image)
#pragma unroll
      for (int cidx = 0; cidx < PX + 2; ++cidx) {
        const int wi = wo0 + cidx - 1;
        const bool ok = wi >= 0 && wi < W;
        const ea_half* xp = x + (((long long)b * H + hi) * W + (ok ? wi : 0)) * CIN;
#pragma unroll
        for (int c = 0; c < CIN; ++c) xin[cidx][c] = ok ? ea_h2f(xp[c]) : 0.f;
      }
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
#pragma unroll
        for (int c = 0; c < CIN; ++c) {
          const float4* wr = reinterpret_cast<const float4*>(wsm + ((kh * 3 + kw) * CIN + c) * Cout + g * 8);
          const float4 w0 = wr[0], w1 = wr[1];
#pragma unroll
          for (int p = 0; p < PX; ++p) {
            const float xv = xin[p + kw][c];
            acc[p][0] = fmaf(xv, w0.x, acc[p][0]); acc[p][1] = fmaf(xv, w0.y, acc[p][1]);
            acc[p][2] = fmaf(xv, w0.z, acc[p][2]); acc[p][3] = fmaf(xv, w0.w, acc[p][3]);
            acc[p][4] = fmaf(xv, w1.x, acc[p][4]); acc[p][5] = fmaf(xv, w1.y, acc[p][5]);
            acc[p][6] = fmaf(xv, w1.z, acc[p][6]); acc[p][7] = fmaf(xv, w1.w, acc[p][7]);
          }
        }
      }
    }
#pragma unroll
    for (int p = 0; p < PX; ++p) {
      if (wo0 + p >= W) break;
      const long long pix = ((long long)b * H + ho) * W + wo0 + p;
      if (add) {
        uint4 u = __ldg(reinterpret_cast<const uint4*>(add + pix * Cout + g * 8));
        float2 a0 = ea_unpack2(u.x), a1 = ea_unpack2(u.y), a2 = ea_unpack2(u.z), a3 = ea_unpack2(u.w);
        acc[p][0] += a0.x; acc[p][1] += a0.y; acc[p][2] += a1.x; acc[p][3] += a1.y;
        acc[p][4] += a2.x; acc[p][5] += a2.y; acc[p][6] += a3.x; acc[p][7] += a3.y;
      }
      const uint4 o = make_uint4(ea_pack2(acc[p][0], acc[p][1]), ea_pack2(acc[p][2], acc[p][3]),
                                 ea_pack2(acc[p][4], acc[p][5]), ea_pack2(acc[p][6], acc[p][7]));
      *reinterpret_cast<uint4*>(out + pix * ldo + g * 8) = o;
      if (out2) *reinterpret_cast<uint4*>(out2 + pix * ldo2 + g * 8) = o;
    }
  }
}

static inline int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  long long cap = 148LL * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace ea

using namespace ea;
#define EA_STREAM(s) reinterpret_cast<cudaStream_t>(s)
#define EA_LAUNCH_OK() (ea_count_launch(), (cudaGetLastError() == cudaSuccess ? 0 : EA_ERR_CUDA))

extern "C" int ea_groupnorm(const ea_gn_args* a, void* stream) {
  if (!a || !a->x || !a->out || !a->gamma || !a->beta || !a->workspace) return EA_ERR_ARG;
  if (a->C % 8 != 0 || a->C % a->groups != 0 || a->ldx % 8 != 0 || a->ldo % 8 != 0 ||
      a->groups > 64 || a->C / 8 > 512)
    return EA_ERR_SHAPE;
  const int C1 = a->x2 ? a->C1 : a->C;
  if (a->x2 && (C1 % 8 != 0 || a->ldx2 % 8 != 0)) return EA_ERR_SHAPE;
  cudaStream_t st = EA_STREAM(stream);
  const int n_sm = ea_sm_count();
  if (a->B > n_sm) return EA_ERR_SHAPE;
  int chunks = n_sm / a->B;                 // all CTAs resident (they barrier on each other)
  if (chunks > a->HW) chunks = a->HW;
  int ppc = (a->HW + chunks - 1) / chunks;
  chunks = (a->HW + ppc - 1) / ppc;
  const int nvec = a->C / 8;
  int threads = (512 / nvec) * nvec;
  threads = ((threads + 31) / 32) * 32;
  if (threads > 512) threads = 512;
  const long long cache_bytes = (long long)ppc * nvec * 16;
  const int part_bytes = ((threads / nvec) * 2 * a->C * 4 + 15) & ~15;
  const int cached = cache_bytes + part_bytes <= 200 * 1024;
  const int smem = 512 + part_bytes + (cached ? (int)cache_bytes : 0);
  static int max_set_dev[EA_MAX_DEV];
  int& max_set = max_set_dev[ea_dev()];
  if (smem > max_set) {
    if (cudaFuncSetAttribute(gn_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) !=
        cudaSuccess)
      return EA_ERR_CUDA;
    max_set = smem;
  }
  GnAffine aff;
  aff.gamma[0] = a->gamma; aff.beta[0] = a->beta;
  aff.gamma[1] = aff.gamma[2] = a->gamma; aff.beta[1] = aff.beta[2] = a->beta;
  aff.ipg = 0;
  if (a->n_nets > 1) {
    if (a->n_nets > 3 || a->B % a->n_nets != 0) return EA_ERR_ARG;
    for (int g = 1; g < a->n_nets; ++g) {
      if (!a->gamma_more[g - 1] || !a->beta_more[g - 1]) return EA_ERR_ARG;
      aff.gamma[g] = a->gamma_more[g - 1];
      aff.beta[g] = a->beta_more[g - 1];
    }
    aff.ipg = a->B / a->n_nets;
  }
  dim3 grid(chunks, a->B);
  if (a->two_pass) {
    const int smem1 = 512 + part_bytes;
    for (int phase = 1; phase <= 2; ++phase)
      ea_launch(gn_fused_kernel, grid, dim3(threads), (size_t)smem1, st,
                reinterpret_cast<const ea_half*>(a->x), a->ldx, C1, reinterpret_cast<const ea_half*>(a->x2),
                a->ldx2, aff, reinterpret_cast<ea_half*>(a->out), a->ldo, a->HW, a->C,
                a->groups, a->eps, a->silu, chunks, ppc, 0, part_bytes, phase, a->workspace);
    ea_count_launch();
    return EA_LAUNCH_OK();
  }
  ea_launch(gn_fused_kernel, dim3(grid), dim3(threads), (size_t)(smem), st, reinterpret_cast<const ea_half*>(a->x), a->ldx, C1, reinterpret_cast<const ea_half*>(a->x2),
      a->ldx2, aff, reinterpret_cast<ea_half*>(a->out), a->ldo, a->HW, a->C,
      a->groups, a->eps, a->silu, chunks, ppc, cached, part_bytes, 0, a->workspace);
  return EA_LAUNCH_OK();
}

extern "C" int ea_layernorm(const void* x, long long ldx, const float* gamma, const float* beta,
                            void* out, long long ldo, int M, int C, float eps, void* stream) {
  if (!x || !out || !gamma || !beta) return EA_ERR_ARG;
  if (C % 8 != 0 || C > 8 * 32 * LN_MAXV || ldx % 8 != 0 || ldo % 8 != 0) return EA_ERR_SHAPE;
  const int wpc = 8;
  ea_launch(layernorm_kernel, dim3((M + wpc - 1) / wpc), dim3(wpc * 32), (size_t)(0), EA_STREAM(stream), reinterpret_cast<const ea_half*>(x), ldx, gamma, beta, reinterpret_cast<ea_half*>(out), ldo,
      M, C, eps);
  return EA_LAUNCH_OK();
}

extern "C" int ea_conv_direct(const void* x, const float* w, const float* bias, void* out, int B,
                              int Hin, int Win, int Cin, int Cout, int ksize, int stride, int silu,
                              const void* add, long long ldo, void* stream) {
  if (!x || !w || !out) return EA_ERR_ARG;
  if ((ksize != 1 && ksize != 3) || (stride != 1 && stride != 2)) return EA_ERR_SHAPE;
  int Ho = (Hin + stride - 1) / stride, Wo = (Win + stride - 1) / stride;
  long long total = (long long)B * Ho * Wo * Cout;
  ea_launch(conv_direct_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, EA_STREAM(stream), reinterpret_cast<const ea_half*>(x), w, bias, reinterpret_cast<ea_half*>(out), B, Hin, Win,
      Cin, Cout, ksize, stride, silu, reinterpret_cast<const ea_half*>(add), ldo > 0 ? ldo : Cout);
  return EA_LAUNCH_OK();
}

extern "C" int ea_upsample2x(const void* x, void* out, int B, int H, int W, int C, void* stream) {
  if (!x || !out) return EA_ERR_ARG;
  if (C % 8 != 0) return EA_ERR_SHAPE;
  long long total = (long long)B * 4 * H * W * (C / 8);
  ea_launch(upsample2x_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, EA_STREAM(stream), reinterpret_cast<const ea_half*>(x), reinterpret_cast<ea_half*>(out), B, H, W, C);
  return EA_LAUNCH_OK();
}

extern "C" int ea_small_linear(const float* x, const void* w, const float* bias, float* y, int M,
                               int N, int K, int silu_in, int silu_out, void* stream) {
  if (!x || !w || !y) return EA_ERR_ARG;
  if (M < 1 || M > 16 || K % 8 != 0) return EA_ERR_SHAPE;
  const int wpc = 8;
  ea_launch(small_linear_kernel, dim3((N + wpc - 1) / wpc), dim3(wpc * 32), (size_t)(0), EA_STREAM(stream), x, reinterpret_cast<const ea_half*>(w), bias, y, M, N, K, silu_in, silu_out);
  return EA_LAUNCH_OK();
}

extern "C" int ea_timestep_embedding(const float* t, float* out, int B, int dim, void* stream) {
  if (!t || !out) return EA_ERR_ARG;
  if (dim % 2 != 0) return EA_ERR_SHAPE;
  int total = B * dim / 2;
  ea_launch(timestep_embedding_kernel, dim3((total + 127) / 128), dim3(128), (size_t)(0), EA_STREAM(stream), t, out, B, dim);
  return EA_LAUNCH_OK();
}

template <bool kCfg, bool kV>
static int launch_out_ddim(const void* xn, const float* w, const float* bias, float* latents, float* eps_out,
                           const float* coef, float guidance, const float* known, const float* noise,
                           const float* mask, void* lat_half_out, int* step_counter, float* hist, int Nimg, int H,
                           int W, int C, void* stream) {
  if (!xn || !w || !bias || (!latents && !eps_out)) return EA_ERR_ARG;
  if (latents && !coef) return EA_ERR_ARG;
  if ((known && !mask) || (noise && !known)) return EA_ERR_ARG;
  if (C % 8 != 0 || Nimg < 1 || H < 1 || W < 1) return EA_ERR_SHAPE;
  long long npix = (long long)Nimg * H * W;
  const int wpc = 4;
  ea_launch(out_ddim_kernel<kCfg, kV>, dim3((unsigned)((npix + wpc - 1) / wpc)), dim3(wpc * 32), (size_t)(0), EA_STREAM(stream), reinterpret_cast<const ea_half*>(xn), w, bias, latents, eps_out, coef, guidance, known, noise, mask,
      reinterpret_cast<ea_half*>(lat_half_out), step_counter, hist, Nimg, H, W, C);
  return EA_LAUNCH_OK();
}

extern "C" int ea_out_cfg_ddim(const void* xn, const float* w, const float* bias, float* latents,
                               float* eps_out, const float* coef, float guidance,
                               const float* known, const float* noise, const float* mask, void* lat_half_out,
                               int* step_counter, float* hist, int Nimg, int H, int W, int C, void* stream) {
  return launch_out_ddim<true, false>(xn, w, bias, latents, eps_out, coef, guidance, known, noise, mask,
                                      lat_half_out, step_counter, hist, Nimg, H, W, C, stream);
}

extern "C" int ea_out_ddim(const void* xn, const float* w, const float* bias, float* latents, float* eps_out,
                           const float* coef, const float* known, const float* noise, const float* mask,
                           void* lat_half_out, int* step_counter, float* hist, int Nimg, int H, int W, int C,
                           void* stream) {
  return launch_out_ddim<false, false>(xn, w, bias, latents, eps_out, coef, 0.f, known, noise, mask, lat_half_out,
                                       step_counter, hist, Nimg, H, W, C, stream);
}

extern "C" int ea_out_cfg_vpred(const void* xn, const float* w, const float* bias, float* latents,
                                float* eps_out, const float* coef, float guidance,
                                const float* known, const float* noise, const float* mask, void* lat_half_out,
                                int* step_counter, float* hist, int Nimg, int H, int W, int C, void* stream) {
  return launch_out_ddim<true, true>(xn, w, bias, latents, eps_out, coef, guidance, known, noise, mask,
                                     lat_half_out, step_counter, hist, Nimg, H, W, C, stream);
}

extern "C" int ea_out_vpred(const void* xn, const float* w, const float* bias, float* latents, float* eps_out,
                            const float* coef, const float* known, const float* noise, const float* mask,
                            void* lat_half_out, int* step_counter, float* hist, int Nimg, int H, int W, int C,
                            void* stream) {
  return launch_out_ddim<false, true>(xn, w, bias, latents, eps_out, coef, 0.f, known, noise, mask, lat_half_out,
                                      step_counter, hist, Nimg, H, W, C, stream);
}

extern "C" int ea_latent_mix(float* latents, const float* known, const float* mask, const float* noise,
                             const float* mix, float alpha, const int* step_counter, int n_rows, void* lat_half_out,
                             int copies, int Nimg, int H, int W, void* stream) {
  if (!latents || !known || !mask || !noise || !mix || !step_counter) return EA_ERR_ARG;
  if (copies != 1 && copies != 2) return EA_ERR_ARG;
  if (Nimg < 1 || H < 1 || W < 1 || n_rows < 1) return EA_ERR_SHAPE;
  const uintptr_t a16 = (uintptr_t)latents | (uintptr_t)known | (uintptr_t)noise;
  if ((a16 & 15) != 0 || ((uintptr_t)lat_half_out & 7) != 0) return EA_ERR_SHAPE;
  const long long npix = (long long)Nimg * H * W;
  ea_launch(latent_mix_kernel, dim3(grid_for(npix, 256)), dim3(256), (size_t)0, EA_STREAM(stream), latents, known,
            mask, noise, mix, alpha, step_counter, n_rows, reinterpret_cast<ea_half*>(lat_half_out), copies, npix);
  return EA_LAUNCH_OK();
}

extern "C" int ea_step_gather(const int* step_counter, int n_rows, int n_tables, const float* const* src,
                              float* const* dst, const long long* row_elems, void* stream) {
  if (!step_counter || n_rows <= 0 || n_tables <= 0 || n_tables > EA_STEP_MAX_TABLES || !src || !dst || !row_elems)
    return EA_ERR_ARG;
  StepTables tb;
  memset(&tb, 0, sizeof(tb));
  tb.n = n_tables;
  long long total = 0;
  for (int k = 0; k < n_tables; ++k) {
    if (!src[k] || !dst[k] || row_elems[k] <= 0) return EA_ERR_ARG;
    tb.src[k] = src[k]; tb.dst[k] = dst[k]; tb.row_elems[k] = row_elems[k];
    total += row_elems[k];
  }
  ea_launch(step_gather_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, EA_STREAM(stream), step_counter, n_rows, tb);
  return EA_LAUNCH_OK();
}

extern "C" int ea_sam_relpos(const void* q, long long q_bs, long long q_ns, const float* Rh,
                             const float* Rw, float* rel_h, float* rel_w, int B, int heads, int S,
                             int d, void* stream) {
  if (!q || !Rh || !Rw || !rel_h || !rel_w) return EA_ERR_ARG;
  if (d % 2 != 0 || S <= 0 || S > 128) return EA_ERR_SHAPE;
  const int smem = 2 * S * (d + 1) * (int)sizeof(float);
  if (smem > 200 * 1024) return EA_ERR_SHAPE;
  static int max_set_dev[EA_MAX_DEV];
  int& max_set = max_set_dev[ea_dev()];
  if (smem > max_set) {
    if (cudaFuncSetAttribute(sam_relpos_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) !=
        cudaSuccess)
      return EA_ERR_CUDA;
    max_set = smem;
  }
  dim3 grid((unsigned)S, (unsigned)(B * heads), 2);
  int threads = S * S >= 1024 ? 256 : 128;
  ea_launch(sam_relpos_kernel, grid, dim3(threads), (size_t)smem, EA_STREAM(stream),
            reinterpret_cast<const ea_half*>(q), q_bs, q_ns, Rh, Rw, rel_h, rel_w, B, heads, S, d);
  return EA_LAUNCH_OK();
}

extern "C" int ea_window_partition(const void* x, void* out, int B, int H, int W, int C, int ws,
                                   void* stream) {
  if (!x || !out) return EA_ERR_ARG;
  if (C % 8 != 0 || ws <= 0) return EA_ERR_SHAPE;
  int nWh = (H + ws - 1) / ws, nWw = (W + ws - 1) / ws;
  long long total = (long long)B * nWh * nWw * ws * ws * (C / 8);
  ea_launch(window_partition_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, EA_STREAM(stream), reinterpret_cast<const ea_half*>(x), reinterpret_cast<ea_half*>(out), B, H, W, C, ws, nWh,
      nWw);
  return EA_LAUNCH_OK();
}

extern "C" int ea_window_unpartition(const void* xw, const void* residual, void* out, int B, int H,
                                     int W, int C, int ws, void* stream) {
  if (!xw || !out) return EA_ERR_ARG;
  if (C % 8 != 0 || ws <= 0) return EA_ERR_SHAPE;
  int nWh = (H + ws - 1) / ws, nWw = (W + ws - 1) / ws;
  long long total = (long long)B * H * W * (C / 8);
  ea_launch(window_unpartition_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, EA_STREAM(stream), reinterpret_cast<const ea_half*>(xw), reinterpret_cast<const ea_half*>(residual),
      reinterpret_cast<ea_half*>(out), B, H, W, C, ws, nWh, nWw);
  return EA_LAUNCH_OK();
}

extern "C" int ea_sam_patchify(const float* img, void* out, int B, int Cin, int H, int W, int ps,
                               void* stream) {
  if (!img || !out) return EA_ERR_ARG;
  if (ps % 8 != 0 || H % ps != 0 || W % ps != 0 || W % 4 != 0) return EA_ERR_SHAPE;
  long long total = (long long)B * (H / ps) * (W / ps) * (Cin * ps * ps / 8);
  ea_launch(patchify_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)0, EA_STREAM(stream), img, reinterpret_cast<ea_half*>(out), B, Cin, H, W, ps);
  return EA_LAUNCH_OK();
}

extern "C" int ea_nhwc_to_nchw_f32(const void* x, float* out, int B, int HW, int C, void* stream) {
  if (!x || !out) return EA_ERR_ARG;
  dim3 grid((HW + 31) / 32, (C + 31) / 32, B), block(32, 8);
  ea_launch(nhwc_to_nchw_f32_kernel, dim3(grid), dim3(block), (size_t)(0), EA_STREAM(stream), reinterpret_cast<const ea_half*>(x), out, B, HW, C);
  return EA_LAUNCH_OK();
}

extern "C" int ea_softmax_rows(const float* s, long long lds, void* p, long long ldp, int rows, int cols,
                               void* stream) {
  if (!s || !p) return EA_ERR_ARG;
  if (rows <= 0 || cols <= 0 || cols % 4 != 0 || lds % 4 != 0 || ldp % 4 != 0) return EA_ERR_SHAPE;
  ea_launch(softmax_rows_kernel, dim3((unsigned)rows), dim3(256), (size_t)0, EA_STREAM(stream), s, lds,
            reinterpret_cast<ea_half*>(p), ldp, cols);
  return EA_LAUNCH_OK();
}

extern "C" int ea_image_out(const void* x, long long ldx, float* out, int B, long long HW, int C, float scale,
                            float shift, float lo, float hi, void* stream) {
  if (!x || !out) return EA_ERR_ARG;
  if (B <= 0 || HW <= 0 || C <= 0 || ldx < C) return EA_ERR_SHAPE;
  const long long total = (long long)B * HW;
  ea_launch(image_out_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), (size_t)0, EA_STREAM(stream),
            reinterpret_cast<const ea_half*>(x), ldx, out, B, HW, C, scale, shift, lo, hi);
  return EA_LAUNCH_OK();
}

extern "C" int ea_conv_in(const void* x, const float* w, const float* bias, void* out, long long ldo,
                          void* out2, long long ldo2, const void* add, int B, int H, int W, int Cin,
                          int Cout, void* stream) {
  if (!x || !w || !out) return EA_ERR_ARG;
  if (Cout % 8 != 0 || (Cin != 4 && Cin != 8) || ldo % 8 != 0 || (out2 && ldo2 % 8 != 0))
    return EA_ERR_SHAPE;
  const int smem = (9 * Cin * Cout + Cout) * (int)sizeof(float);
  const long long total = (long long)B * H * ((W + 3) / 4) * (Cout / 8);   // a thread = 4 pixels x 8 channels
  int grid = (int)((total + 255) / 256);
  if (grid > 296) grid = 296;   // the filter bank (46 KB for 4 -> 320) is loaded once per CTA: two CTAs per SM
  if (grid < 1) grid = 1;
  cudaStream_t st = EA_STREAM(stream);
  const ea_half* xx = reinterpret_cast<const ea_half*>(x);
  ea_half* o1 = reinterpret_cast<ea_half*>(out);
  ea_half* o2 = reinterpret_cast<ea_half*>(out2);
  const ea_half* ad = reinterpret_cast<const ea_half*>(add);
  const long long l1 = ldo > 0 ? ldo : Cout, l2 = ldo2 > 0 ? ldo2 : Cout;
  if (Cin == 4) {
    static bool set4_dev[EA_MAX_DEV];
    bool& set4 = set4_dev[ea_dev()];
    if (!set4) {
      if (cudaFuncSetAttribute(conv_smallcin_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               96 * 1024) != cudaSuccess) return EA_ERR_CUDA;
      set4 = true;
    }
    if (smem > 96 * 1024) return EA_ERR_SHAPE;
    ea_launch(conv_smallcin_kernel<4>, dim3(grid), dim3(256), (size_t)(smem), st, xx, w, bias, o1, l1, o2, l2, ad, B, H, W, Cout);
  } else {
    static bool set8_dev[EA_MAX_DEV];
    bool& set8 = set8_dev[ea_dev()];
    if (!set8) {
      if (cudaFuncSetAttribute(conv_smallcin_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               192 * 1024) != cudaSuccess) return EA_ERR_CUDA;
      set8 = true;
    }
    if (smem > 192 * 1024) return EA_ERR_SHAPE;
    ea_launch(conv_smallcin_kernel<8>, dim3(grid), dim3(256), (size_t)(smem), st, xx, w, bias, o1, l1, o2, l2, ad, B, H, W, Cout);
  }
  return EA_LAUNCH_OK();
}
